"""Index build side (train / encode / add) -- the callers *before* the search hot path.

SURVEY.md section 8(f) rank 1-2 ("next" rows).  The two compute steps (assignment = tpq_max_sim,
centroid update = tpq_compute_centroids) are the library's CUDA kernels; the container bookkeeping
(index of appearance, expansion, write addresses) is expressed with PyTorch tensor ops on the index
device.  It is what builds the large synthetic indexes for the search benchmark; it is NOT the
measured path.  Semantics followed:

    IVFPQIndex.train        torchpq/index/IVFPQIndex.py:234-260  (VQ: <=15 Lloyd iters, PQ: <=25)
    KMeans / MultiKMeans    torchpq/clustering/KMeans.py:399-438, MultiKMeans.py:415-453
        assignment = arg-max of negative squared L2 (kernels/cuda/max_sim.cu:78-98)
        update     = member mean, empty cluster -> 0 (kernels/cuda/compute_centroids.cu:9-86)
    IVFPQIndex.add          torchpq/index/IVFPQIndex.py:316-364
    CellContainer.add       torchpq/container/CellContainer.py:313-367 (ioa, expand loop, write address
                            = ioa-th empty slot of the cell, get_write_address_v2.cu:9-41)
Unlike the reference (unseeded np.random.choice, MultiKMeans.py:277-283) initial centroids come
from a seeded torch.Generator: two runs start from the same centroids, and since every kernel of the loop sums in a fixed
order (no float atomics), two runs on the same GPU train the same codebooks bit for bit.
"""
from __future__ import annotations

import torch


def _assign(data: torch.Tensor, cent: torch.Tensor, exact: bool = True) -> torch.Tensor:
    """data [l, d, n], cent [l, d, k] -> labels [l, n] int64: tpq_max_sim.  exact=True: the reference's fp32
    arithmetic (used for encoding, so codes match the reference's); exact=False: TF32 tensor-core kernel where it
    applies (used inside the Lloyd iterations, where a label flip between near-equidistant centroids is harmless)."""
    from . import fn
    return fn.max_sim(data.contiguous(), cent.contiguous(), "euclidean", exact=exact, exact_values=False)[1]


def _init_centroids(data: torch.Tensor, k: int, seed: int) -> torch.Tensor:
    """MultiKMeans.initialize_centroids, init_mode="random" (MultiKMeans.py:271-283): k distinct data points, the same
    columns for every sub-quantizer -- from a seeded generator instead of the reference's unseeded np.random.choice."""
    l, d, n = data.shape
    gen = torch.Generator(device="cpu").manual_seed(seed)
    pick = torch.randperm(n, generator=gen)[:k].to(data.device)
    cent = data[:, :, pick].clone()
    if cent.shape[2] < k:                                              # fewer points than clusters
        cent = torch.cat([cent, torch.zeros(l, d, k - cent.shape[2], device=data.device)], dim=2)
    return cent


def fit(data: torch.Tensor, k: int, max_iter: int, tol: float = 1e-4, n_redo: int = 1, seed: int = 0,
        centroids: torch.Tensor | None = None, distance: str = "euclidean", exact: bool = False,
        kmeans_assign: bool = False, init=None):
    """MultiKMeans.fit (clustering/MultiKMeans.py:415-453; KMeans.fit, KMeans.py:399-438, is the l = 1 case):
    l independent k-means over data [l, d, n].  Per redo: Lloyd iterations until `error = sum((new - old)^2) <= tol`
    (calculate_error, :143-149 -- a SUM of squares over all l*d*k entries, not a mean shift) or max_iter; the redo
    with the lowest inertia = mean(-maxsims) (:151-152) wins.  -> (centroids [l, d, k], labels [l, n], inertia, n_iter).
    As in the reference the returned labels are those of the last assignment, i.e. relative to the centroids BEFORE
    the final update.  exact=True: the reference's fp32 assignment arithmetic bit for bit (max_sim.cu:78-98);
    exact=False: TF32 tensor-core assignment where the shape allows (labels can differ between near-equidistant
    centroids only).
    kmeans_assign=True (the Lloyd iterations of clustering.KMeans / MultiKMeans): the assignment is
    fn.kmeans_assign, i.e. TF32 tensor cores for every shape one of its kernels takes, cosine included, and distance
    may also be "manhattan" (exact kernel); `exact` is then ignored.  init(data, k, seed) -> centroids replaces the
    random initialisation (kmeans++)."""
    from . import fn
    assert data.dim() == 3 and data.is_contiguous(), "use .contiguous()"                  # MultiKMeans.py:421
    assert distance in (("euclidean", "cosine", "manhattan") if kmeans_assign else ("euclidean", "cosine"))
    init = init or _init_centroids
    best = None
    best_inertia = 1e32
    for redo in range(n_redo):
        cent = centroids if (centroids is not None and redo == 0) else init(data, k, seed + redo)
        n_iter = 0
        for _ in range(max_iter):
            if kmeans_assign:
                x, c = data, cent.contiguous()
                if distance == "cosine":                                # normalised out of place (the caller's tensors stay)
                    x = data / (data.norm(dim=-2, keepdim=True) + 1e-8)
                    c = cent / (cent.norm(dim=-2, keepdim=True) + 1e-8)
                maxsims, labels = fn.kmeans_assign(x, c.contiguous(), distance, exact_values=n_redo > 1)
            elif distance == "cosine":                                  # get_labels, MultiKMeans.py:314-333
                dn = data / (data.norm(dim=-2, keepdim=True) + 1e-8)
                cn = cent / (cent.norm(dim=-2, keepdim=True) + 1e-8)
                maxsims, labels = fn.max_sim(dn.contiguous(), cn.contiguous(), "cosine", exact=True)
            else:
                maxsims, labels = fn.max_sim(data, cent.contiguous(), "euclidean", exact=exact, exact_values=n_redo > 1)
            new = fn.compute_centroids(data, labels, k)
            error = (new - cent).pow(2).sum()
            cent = new
            n_iter += 1
            if float(error) <= tol:                                     # one host sync per iteration, as in the reference
                break
        inertia = float((-maxsims).mean())
        if inertia < best_inertia:
            best, best_inertia = (cent, labels, inertia, n_iter), inertia
    return best


def multi_kmeans(data: torch.Tensor, k: int, max_iter: int, tol: float = 1e-4, seed: int = 0,
                 distance: str = "euclidean") -> torch.Tensor:
    """l independent k-means over data [l, d, n] -> centroids [l, d, k] (fit with the reference's defaults)."""
    return fit(data, k, max_iter, tol=tol, n_redo=1, seed=seed, distance=distance)[0]


def train_coarse(index, x: torch.Tensor, seed: int = 0, vq_iters: int = 15):
    """The coarse half of IVFPQIndex.train: x [d, n] (normalised for cosine) -> (that x, the coarse codebook [d, n_cells]).
    IVFFlatIndex.train is this alone, so both indexes trained on the same data and seed probe the same cells."""
    assert x.dim() == 2 and x.shape[0] == index.d_vector
    from . import fn
    if index.distance == "cosine":
        x = fn.normalize(x.contiguous())
    return x, multi_kmeans(x[None].contiguous(), index.n_cells, vq_iters, seed=seed)[0].contiguous()


def train(index, x: torch.Tensor, seed: int = 0, vq_iters: int = 15, pq_iters: int = 25):
    """IVFPQIndex.train: fit the coarse quantizer and the M sub-quantizers on x [d, n]."""
    x, vq = train_coarse(index, x, seed, vq_iters)
    if getattr(index, "pq_use_residual", False):                       # IVFPQIndex.py:248-256: PQ learns x - vq(x)
        x = x - vq[:, _assign(x[None].contiguous(), vq[None])[0]]
    sub = x.reshape(index.n_subvectors, index.d_subvector, x.shape[1]).contiguous()
    pq = multi_kmeans(sub, 256, pq_iters, seed=seed + 1, distance=index.distance).contiguous()   # PQCodec.py:27-32
    index.vq_codec.set_codebook(vq)
    index.pq_codec.set_codebook(pq)
    index._state_changed()


def encode(index, x: torch.Tensor):
    """-> (cells [n] i64, codes [M, n] u8) for x [d, n] (already normalised for cosine)."""
    cells = _assign(x[None], index.vq_codec.codebook[None])[0]
    if getattr(index, "pq_use_residual", False):                       # IVFPQIndex.py:281-284
        x = x - index.vq_codec.codebook[:, cells]
    sub = x.reshape(index.n_subvectors, index.d_subvector, x.shape[1]).contiguous()
    codes = _assign(sub, index.pq_codec.codebook).to(torch.uint8)
    return cells, codes


def _expand(index, grow: torch.Tensor):
    """CellContainer.expand (CellContainer.py:249-311) for all cells with grow[c] > 0 in one pass: the per-cell tables
    are [n_cells] tensor arithmetic, the slot move is the library's tpq_expand_move kernel."""
    from ._lib import lib, check, ptr
    from . import _lib
    dev = index._storage.device
    shift = torch.cumsum(grow, 0) - grow                           # slots inserted before each cell
    old_cap = index.capacity
    new_cap = old_cap + int(grow.sum().item())
    if new_cap == old_cap:                                         # container_add would repeat this round forever
        raise RuntimeError("container expansion made no room: a short cell grew by 0 slots")
    storage = index._storage.new_zeros((index._storage.shape[0], new_cap, index._storage.shape[2]))   # u8 codes or f32
    a2i = torch.full((new_cap,), -1, dtype=torch.long, device=dev)
    emp = torch.ones(new_cap, dtype=torch.uint8, device=dev)
    if old_cap > 0:                                                # an empty store has no slot to move (and no pointers)
        check(lib.tpq_expand_move(ptr(index._storage), ptr(index._address2id), ptr(index._is_empty), ptr(index._cell_start),
                                  ptr(shift), index.n_cells, index.code_size, old_cap, new_cap,
                                  ptr(storage), ptr(a2i), ptr(emp), _lib.current_stream(dev)))
    for name, val in (("_storage", storage), ("_address2id", a2i), ("_is_empty", emp)):
        delattr(index, name)
        index.register_buffer(name, val)
    index._cell_start += shift
    index._cell_capacity += grow


def growth(capacity: torch.Tensor, short: torch.Tensor, expand_mode: str, expand_step_size: int) -> torch.Tensor:
    """Slots one expansion round adds to each cell (CellContainer.expand, CellContainer.py:249-311): 0 where the cell
    has room; for a short cell its capacity ("double") or expand_step_size ("step").  A cell of capacity 0 cannot
    double -- the reference's loop never ends on one -- so in "double" mode it grows by expand_step_size instead."""
    step = torch.full_like(capacity, expand_step_size)
    grow = torch.where(capacity > 0, capacity, step) if expand_mode == "double" else step
    return torch.where(short, grow, torch.zeros_like(capacity))


def container_add(index, codes: torch.Tensor, cells: torch.Tensor, ids=None, return_address=False):
    """CellContainer.add (CellContainer.py:313-367) on the library's placement kernels (csrc/place.cu): index of
    appearance, expansion test, write addresses, and one scatter into the reference layout AND the scan layout.
    An index without a scan layout (IVFFlatIndex: no ``_layout``, codes = the bytes of its fp32 columns) gets the
    reference layout only."""
    import ctypes as C
    from . import fn, _lib
    from ._lib import lib, check, ptr
    from .index import _fingerprint, _codebook_of
    assert codes.dtype == torch.uint8 and cells.dtype == torch.long
    assert codes.shape[0] == index.code_size and codes.shape[1] == cells.shape[0]
    assert index._storage is not None, "shard-only index: add to the full index and distribute again"
    dev = index._storage.device
    n = cells.shape[0]
    if ids is None:
        ids = torch.arange(n, device=dev, dtype=torch.long) + index.max_id + 1
    else:
        assert ids.dtype == torch.long and ids.shape[0] == n
        ids = ids.to(dev)
    if n == 0:
        return (ids, torch.empty(0, dtype=torch.long, device=dev)) if return_address else ids
    codes, cells = codes.contiguous(), cells.contiguous()
    assert int(cells.min().item()) >= 0 and int(cells.max().item()) < index.n_cells, "cell id out of range"
    lay = getattr(index, "_layout", None)
    fp = lambda: _fingerprint(index._storage, index._is_empty, index._cell_start, index._cell_size, index._address2id,
                              _codebook_of(index.vq_codec), _codebook_of(index.pq_codec))
    in_sync = lay is not None and lay.fingerprint == fp()
    ioa, counts = fn.get_ioa(cells, index.n_cells)
    prefix = None
    while True:
        # free slots of a cell = capacity - LIVE items.  Without holes live == _cell_size and this is the reference's
        # `capacity - cell_size - (ioa + 1) < 0` test (CellContainer.py:338-341) taken per cell: the largest ioa of a cell
        # is its count - 1.  With holes left by remove() the empty-slot prefix gives the live count.  A store of
        # capacity 0 (initial_size=0, or such a checkpoint loaded) holds nothing: every _cell_size is 0.
        if index._has_holes and index.capacity > 0:
            prefix = fn.empty_prefix(index._is_empty)
            p = prefix.to(torch.long) & 0xFFFFFFFF
            live = index._cell_capacity - (p[index._cell_start + index._cell_capacity] - p[index._cell_start])
        else:
            live = index._cell_size
        short = counts > index._cell_capacity - live
        if not bool(short.any().item()):
            break
        _expand(index, growth(index._cell_capacity, short, index.expand_mode, index.expand_step_size))
        in_sync = False                                              # addresses moved: the scan layout is rebuilt lazily
    write = fn.get_write_address(cells, ioa, index._cell_start, index._cell_size, index._cell_capacity, prefix)
    ix = lay.cindex if in_sync else _lib.TpqIndex()
    if not in_sync:
        # no scanned code without a scan layout: 4, the smallest n_subvectors tpq_store_codes takes (it then reads only
        # code_size), for any store, IVFPQ4Index's too, whose code_size is n_subvectors / 2
        ix.n_subvectors, ix.n_cells, ix.capacity = 4, index.n_cells, index.capacity
        ix.code_size = index.code_size
        ix.shard_world = 1
    ix.cell_start = index._cell_start.data_ptr()
    check(lib.tpq_store_codes(ptr(codes), ptr(cells), ptr(write), ptr(ids), n, C.byref(ix),
                              ptr(index._storage), ptr(index._address2id), ptr(index._is_empty), ptr(index._cell_size),
                              ptr(lay.codes_scan) if in_sync else None, ptr(lay.block_valid) if in_sync else None,
                              _lib.current_stream(dev)))
    index._ids_changed()                                             # the kernel wrote _address2id past its _version
    index._max_id = max(index._max_id, int(ids.max().item()))
    if in_sync:                                                      # the layout received the same items and stays valid
        rank, world = lay.shard                                      # (raw-pointer writes do not move the buffers' fingerprint);
        owned = n if world == 1 else int((cells % world == rank).sum().item())   # only the shard's cells reach block_valid
        lay.set_live(lay.n_live + owned)
    else:
        index._state_changed()
    return (ids, write) if return_address else ids


def add(index, x: torch.Tensor, ids=None, return_address=False, chunk: int = 1 << 20):
    """IVFPQIndex.add: encode x [d, n] and store it."""
    assert x.dim() == 2 and x.shape[0] == index.d_vector
    assert index._storage is not None, "shard-only / search-only index: add to the full index (reload the checkpoint)"
    from . import fn
    cells_l, codes_l = [], []
    for s in range(0, x.shape[1], chunk):
        xc = x[:, s:s + chunk].contiguous()
        if index.distance == "cosine":
            xc = fn.normalize(xc)
        c, q = encode(index, xc)
        cells_l.append(c)
        codes_l.append(q)
    return container_add(index, torch.cat(codes_l, 1), torch.cat(cells_l, 0), ids, return_address)


def container_remove(index, ids=None, address=None):
    """CellContainer.remove (CellContainer.py:369-393) as it is documented to behave (README.md:60-66: "virtually
    remove vectors ... ignores ids that don't exist"); see IVFPQIndex.remove.  Removed slots become holes (is_empty = 1,
    address2id = -1); ``_cell_size`` is not decremented."""
    if ids is not None:
        address = index.get_address_by_id(ids)
    elif address is not None:
        assert address.dtype == torch.int64
        address = address.to(index._address2id.device)
    else:
        raise RuntimeError("Need either ids or address")
    mask = (address >= 0) & (address < index.capacity)
    address = address[mask].unique(sorted=True)
    address = address[index._is_empty[address] == 0]
    if address.shape[0] == 0:
        return
    index._is_empty[address] = 1
    index._address2id[address] = -1
    index._has_holes = True
    index._state_changed()
