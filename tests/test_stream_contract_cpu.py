"""CPU: the library's stream contract, read from its sources (include/tpq_b200.h: "never allocates, frees or keeps
caller memory, never synchronises the host, and launches only on the stream it is given").  Every kernel launch names
its stream, every async copy or memset takes one, and no allocating or synchronising runtime call appears outside the
debug-only ``tpq_profile_*`` hook.  tests/test_streams_gpu.py checks the same contract by capturing every entry point
into a CUDA graph; this file keeps it enforced where no GPU is available."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = sorted(glob.glob(os.path.join(ROOT, "torchpq_b200", "csrc", "*.cu*")))

# every asynchronous copy or memset of the runtime, and its argument count: the stream is the last argument
ASYNC_ARITY = {"cudaMemcpyAsync": 5, "cudaMemsetAsync": 4, "cudaMemcpy2DAsync": 8, "cudaMemset2DAsync": 6,
               "cudaMemcpy3DAsync": 2, "cudaMemset3DAsync": 4, "cudaMemcpyToSymbolAsync": 6,
               "cudaMemcpyFromSymbolAsync": 6, "cudaMemcpyPeerAsync": 6, "cudaMemcpy2DToArrayAsync": 9,
               "cudaMemcpy2DFromArrayAsync": 9}
# a synchronous copy or memset (any cudaMemcpy* / cudaMemset* without the Async suffix), an allocation or free, and a
# host wait on the device, a stream or an event
FORBIDDEN = re.compile(r"\b(cuda(?:Memcpy|Memset)\w*(?<!Async)|cuda(?:Malloc|Free)\w*|cuda(?:Device|Stream|Event)Synchronize)"
                       r"\s*\(")


def _strip(src):
    """`src` without comments and string literals (a launch written in a comment is not a launch)."""
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\])*"', lambda m: "" if m.group(0)[0] == "/" else '""', src,
                  flags=re.S)


def _code(path):
    return _strip(open(path).read())


def _top_level_args(text):
    """Split `text` at the commas outside any bracket."""
    args, depth, cur = [], 0, ""
    for ch in text:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
    return args + [cur.strip()]


def _call_args(code, start):
    """The top-level arguments of the call whose '(' is at code[start]."""
    depth = 0
    for end in range(start, len(code)):
        depth += {"(": 1, ")": -1}.get(code[end], 0)
        if depth == 0:
            return _top_level_args(code[start + 1:end])
    raise AssertionError("unbalanced call")


def _profile_spans(code):
    """[start, end) of every tpq_profile_* function body: the one place a global, synchronising hook is allowed."""
    spans = []
    for m in re.finditer(r'\bint\s+tpq_profile_\w+\s*\([^)]*\)\s*\{', code):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(code[i], 0)
            i += 1
        spans.append((m.start(), i))
    return spans


def test_sources_found():
    assert len(SOURCES) >= 10 and any(p.endswith("scan.cu") for p in SOURCES)


def test_every_launch_names_a_stream():
    n = 0
    for path in SOURCES:
        code = _code(path)
        for m in re.finditer(r"<<<(.*?)>>>", code, flags=re.S):
            cfg = _top_level_args(m.group(1))
            line = code[:m.start()].count("\n") + 1
            assert len(cfg) == 4 and cfg[3] not in ("0", "nullptr", "NULL", "cudaStreamLegacy", "cudaStreamPerThread"), \
                f"{os.path.basename(path)}:{line}: launch <<<{m.group(1)}>>> does not name the caller's stream"
            n += 1
    assert n >= 40                                                        # every kernel family was seen


def test_every_async_copy_and_memset_takes_a_stream():
    n = 0
    for path in SOURCES:
        code = _code(path)
        for m in re.finditer(r"\b(cuda(?:Memcpy|Memset)\w*Async)\s*\(", code):
            args = _call_args(code, m.end() - 1)
            line = code[:m.start()].count("\n") + 1
            assert m.group(1) in ASYNC_ARITY, f"{os.path.basename(path)}:{line}: add {m.group(1)} to ASYNC_ARITY"
            assert len(args) == ASYNC_ARITY[m.group(1)] and args[-1] not in ("0", "nullptr", "NULL"), \
                f"{os.path.basename(path)}:{line}: {m.group(1)} without the caller's stream"
            n += 1
    assert n >= 10                                                        # cudaMemcpy2DAsync of ivfflat.cu included


def test_no_allocation_or_host_sync_outside_the_profile_hook():
    for path in SOURCES:
        code = _code(path)
        spans = _profile_spans(code)
        for m in FORBIDDEN.finditer(code):
            line = code[:m.start()].count("\n") + 1
            assert any(a <= m.start() < b for a, b in spans), \
                f"{os.path.basename(path)}:{line}: {m.group(1)} outside tpq_profile_*"


def test_checker_sees_a_violation():
    """The parsers above would flag the forms they exist to catch."""
    assert len(_top_level_args("dim3((unsigned)((n + 255) / 256), (unsigned)l), 256, 0")) == 3
    assert len(_top_level_args("grid, 256, smem, st")) == 4
    code = "int f() { cudaMemsetAsync(p, 0, (size_t)n * 4); }"
    assert len(_call_args(code, code.index("(", code.index("cudaMemsetAsync")))) == 3
    assert _strip('x; // k<<<1, 1>>>();\n"cudaFree"') == 'x; \n""'
    code = _strip('extern "C" int tpq_profile_x(int a) { if (a) { cudaDeviceSynchronize(); } } int g() {}')
    (a, b), = _profile_spans(code)
    assert code[a:b].endswith("} }") and a < code.index("cudaDeviceSynchronize") < b
    caught = [m.group(1) for m in FORBIDDEN.finditer(
        "cudaMemcpy(a); cudaMemcpy2D(b); cudaMemcpyToSymbol(c); cudaMemset(d); cudaMallocAsync(e); cudaFreeHost(f); "
        "cudaEventSynchronize(g); cudaStreamSynchronize(h); cudaMemcpyAsync(i); cudaMemcpy2DAsync(j); cudaStreamWaitEvent(k)")]
    assert caught == ["cudaMemcpy", "cudaMemcpy2D", "cudaMemcpyToSymbol", "cudaMemset", "cudaMallocAsync", "cudaFreeHost",
                      "cudaEventSynchronize", "cudaStreamSynchronize"]


def test_every_python_entry_point_runs_on_its_data_device():
    """The library launches on the current device, so every Python entry point makes its data's device current
    (modules.on_device): an index on cuda:1 works while cuda:0 is current (test_streams_gpu.test_index_on_another_device
    runs it where two devices are visible)."""
    import torchpq_b200 as T
    entry = {T.FlatIndex: ("add", "remove", "search", "range_search"),
             T.IVFFlatIndex: ("train", "add", "remove", "search", "search_cells", "range_search"),
             T.IVFSQIndex: ("train", "add", "remove", "search", "search_cells", "range_search"),
             T.IVFPQIndex: ("train", "add", "remove", "search", "search_cells", "range_search", "layout", "encode",
                            "decode"),
             T.IVFPQRIndex: ("train", "add", "remove", "search", "rerank", "encode", "decode"),
             T.codec.SQCodec: ("encode", "decode"), T.fn.Topk: ("__call__",), T.fn.IVFPQTopk: ("topk",)}
    missing = [f"{cls.__name__}.{name}" for cls, names in entry.items() for name in names
               if not hasattr(getattr(cls, name), "__wrapped__")]
    fns = ("normalize", "coarse_probe", "precompute_adc", "max_sim", "kmeans_assign", "compute_centroids", "pq_decode",
           "merge_topk", "get_ioa", "empty_prefix", "get_write_address")
    missing += [f"fn.{name}" for name in fns if not hasattr(getattr(T.fn, name), "__wrapped__")]
    assert not missing, f"not run on their data's device: {missing}"
