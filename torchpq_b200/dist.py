"""Cell-sharded multi-GPU search: one process per GPU, one NCCL all-gather of candidates per query batch.

The reference is single-GPU only (SURVEY.md section 2: no NCCL / torch.distributed anywhere).
Partitioning (SURVEY.md section 8e): the ``world`` ranks form a grid of ``cell_shards x query_groups``
(default ``world x 1``, the north-star's pure cell sharding).  Rank r owns the cells c with
``c % cell_shards == r % cell_shards`` and serves the queries of group ``r // cell_shards``.  Each rank holds
only ITS cells' codes (in scan layout); the two small codebooks, the per-cell tables and the address->id table
are replicated.  A rank runs the (deterministic) coarse probe, scans its own cells and emits its local top-k
as packed 64-bit (score, address) keys.  ONE ``all_gather_into_tensor`` of [nq / query_groups, k] keys
(8 B per candidate) follows, then the merge kernel picks the global top-k -- the union of per-shard top-k's
contains the global top-k, and keys carry GLOBAL addresses, so sharded == unsharded bit for bit, ties included.

``query_groups > 1`` trades memory for fixed cost: every (query, rank) pair pays one LUT build and one top-k
bootstrap whatever the shard holds, so at 8 GPUs a 4 x 2 grid halves that replicated work (each rank then
holds 1/4 of the codes instead of 1/8).
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import fn


def merge_gathered(keys_all: torch.Tensor, address2id: torch.Tensor):
    """keys_all [world, nq, k] -> (values, ids, address); CUDA kernel tpq_merge_topk."""
    return fn.merge_topk(keys_all.contiguous(), address2id)


def _gather_rows(t: torch.Tensor, world: int, group):
    out = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous(), group=group)
    return out


class PeerExchange:
    """Gather buffers in symmetric (peer-mapped) memory for the fused scan + exchange: rank r's scan kernel stores its
    keys straight into slot r of EVERY rank's buffer over NVLink (`tpq_ivfpq_scan_push`), a symmetric-memory barrier
    follows, and each rank merges its own copy.  Two buffers alternate: the barrier of step i+1 orders every rank's merge
    of step i before anybody's pushes of step i+2 into the same buffer."""

    def __init__(self, group, world, nq, k, device):
        import ctypes as C
        import torch.distributed._symmetric_memory as symm
        self.shape = (world, nq, k)
        self.bufs, self.hdls, self.ptrs = [], [], []
        for _ in range(2):
            t = symm.empty(world, nq, k, dtype=torch.int64, device=device)
            h = symm.rendezvous(t, group if group is not None else dist.group.WORLD)
            self.bufs.append(t)
            self.hdls.append(h)
            self.ptrs.append((C.c_void_p * world)(*[int(p) for p in h.buffer_ptrs]))
        self.step = 0

    def next(self):
        b = self.step & 1
        self.step += 1
        return self.bufs[b], self.hdls[b], self.ptrs[b]


_exchanges = {}
_p2p_broken = [False]


def _peer_exchange(group, world, nq, k, device):
    """One PeerExchange per (group, shape); None when symmetric memory cannot be set up here (then NCCL gathers)."""
    if _p2p_broken[0]:
        return None
    # one pair of buffers per STREAM: callers that pipeline batches over several streams (bench.py) must not share them
    # (the reuse argument above orders steps of one stream only)
    key = (id(group), world, nq, k, str(device), torch.cuda.current_stream(device).cuda_stream)
    if key not in _exchanges:
        try:
            _exchanges[key] = PeerExchange(group, world, nq, k, device)
        except Exception as e:                                          # no P2P mapping on this system / build
            import warnings
            warnings.warn(f"torchpq_b200.dist: symmetric memory unavailable ({e!r}); using the NCCL all-gather exchange")
            _p2p_broken[0] = True
            return None
    return _exchanges[key]


def make_grid(world: int, query_groups: int = 1):
    """(cell_shards, query_groups) with cell_shards * query_groups == world."""
    assert query_groups >= 1 and world % query_groups == 0, f"query_groups={query_groups} must divide world={world}"
    return world // query_groups, query_groups


def sharded_search(index, x: torch.Tensor, k: int, group=None, return_address: bool = False,
                   split_coarse: bool = True, grid=None, coarse_group=None, exchange: str = "auto"):
    """``index`` holds this rank's shard (``dist.distribute``; or the full reference state with
    ``index.set_shard(rank % cell_shards, cell_shards)``).  Returns the same (values, ids[, address]) for the whole
    batch on every rank.

    split_coarse (default): the coarse probe -- the one stage that does not shrink with the shard -- is itself split
    by QUERIES among the ranks that share a query group: each probes 1/cell_shards of the group's queries and a small
    all-gather (2 n_probe + 1 int64 per query) hands every rank of the group the full probe lists.  Same deterministic
    kernel on every rank, so the lists are bit-identical to the replicated computation.  split_coarse=False runs the
    group's whole coarse probe on every rank: exactly one collective per batch.  ``coarse_group`` = the process group
    of this rank's query group (needed for split_coarse when query_groups > 1; ``dist.new_group`` per group).

    exchange: "nccl" = scan to a local buffer, then ``all_gather_into_tensor``; "p2p" = the fused scan + exchange
    (``PeerExchange``): the scan kernel's CTAs store their keys into every rank's gather buffer over NVLink while the
    other CTAs are still scanning, a symmetric-memory barrier replaces the collective; "auto" = p2p on CUDA/NCCL when
    symmetric memory can be set up and the batch is large enough not to be sliced, else nccl."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    shards, groups = grid if grid is not None else (world, 1)
    assert shards * groups == world
    crank, qg = rank % shards, rank // shards
    nq_all = x.shape[1]
    per_group = (nq_all + groups - 1) // groups
    g_lo = min(nq_all, qg * per_group)
    g_hi = min(nq_all, g_lo + per_group)
    xg = x if groups == 1 else x[:, g_lo:g_hi].contiguous()
    nq, n_probe = xg.shape[1], int(index.n_probe)
    if groups > 1 and nq < per_group:                                  # ragged last group: pad so every rank gathers equal rows
        xg = torch.cat([xg, xg.new_zeros(xg.shape[0], per_group - nq)], 1)
    ex = None
    if world > 1 and exchange in ("auto", "p2p") and x.device.type == "cuda" and hasattr(index, "scan_push"):
        ex = _peer_exchange(group, world, xg.shape[1], k, x.device)
        assert ex is not None or exchange == "auto", "exchange='p2p' requested but symmetric memory is unavailable"
    cells = base = npl = None
    xq = xg
    if shards > 1 and split_coarse and (groups == 1 or coarse_group is not None):
        cg = group if groups == 1 else coarse_group
        xq = fn.normalize(xg.contiguous()) if index.distance == "cosine" else xg.contiguous()   # IVFPQIndex.py:474-475
        nqg = xq.shape[1]
        per = (nqg + shards - 1) // shards
        lo = min(nqg, crank * per)
        hi = min(nqg, lo + per)
        mine = torch.zeros(per, 2 * n_probe + 1, dtype=torch.long, device=x.device)
        if hi > lo:
            sims, c, n = fn.coarse_probe(xq[:, lo:hi].contiguous(), index.vq_codec.codebook, n_probe,
                                         index.use_smart_probing, index.smart_probing_temperature)
            mine[:hi - lo, :n_probe] = c
            mine[:hi - lo, n_probe] = n
            mine[:hi - lo, n_probe + 1:] = sims.view(torch.int32).to(torch.long)      # fp32 bits, exact round trip
        allp = _gather_rows(mine, shards, cg)[:nqg]
        base = allp[:, n_probe + 1:].to(torch.int32).view(torch.float32).contiguous()
        cells, npl = allp[:, :n_probe].contiguous(), allp[:, n_probe].contiguous()
    keys_all = None
    if ex is not None:
        buf, hdl, ptrs = ex.next()
        try:
            index.scan_push(xq, k, ptrs, world, rank, cells=cells, base_sims=base, n_probe_list=npl)
            hdl.barrier(channel=0)                                   # every rank's keys have landed in every buffer
            keys_all = buf
        except NotImplementedError:                                   # sliced small batch: gathered path below
            ex.step -= 1
    if keys_all is None:
        if cells is not None:
            keys = index.search_cells(xq, cells, base_sims=base, n_probe_list=npl, k=k, return_keys=True)[2]
        else:
            keys = index.search(xg, k=k, return_keys=True)[2]
        if world == 1:
            keys_all = keys[None]
        else:
            keys_all = torch.empty((world * keys.shape[0], keys.shape[1]), dtype=keys.dtype, device=keys.device)
            dist.all_gather_into_tensor(keys_all, keys, group=group)      # THE collective of the path: 8 B per candidate
            keys_all = keys_all.view(world, keys.shape[0], keys.shape[1])
    if groups == 1:
        values, ids, address = merge_gathered(keys_all, index._address2id)
    else:                                                              # rows [g*shards, (g+1)*shards) are query group g's parts
        outs = [merge_gathered(keys_all[g * shards:(g + 1) * shards], index._address2id) for g in range(groups)]
        values, ids, address = (torch.cat([o[j] for o in outs], 0)[:nq_all] for j in range(3))
    return (values, ids, address) if return_address else (values, ids)


def _bcast_tensor(t, shape, dtype, dev, src, group, rank):
    if rank != src:
        t = torch.empty(shape, dtype=dtype, device=dev)
    dist.broadcast(t, src=src, group=group)
    return t


def distribute(index, src: int = 0, group=None, grid=None):
    """Hand every rank ITS shard of rank ``src``'s index (trained + populated there, or loaded from a reference
    checkpoint) and nothing more: the scan layout of the rank's own cells (1/cell_shards of the codes), the small
    replicated state (codebooks, per-cell tables, address->id) -- no rank other than ``src`` ever sees the
    reference-layout code store, and ``src`` drops it too unless ``keep_full``.  After the call ``index`` on every
    rank is a shard-only index ready for ``sharded_search``."""
    if hasattr(index, "n_subvectors_rerank"):
        raise NotImplementedError("an IVFPQRIndex cannot be distributed: its re-rank pass reads the full _storage")
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    shards, groups = grid if grid is not None else (world, 1)
    assert shards * groups == world
    dev = torch.device(index.device)
    small = ["_cell_start", "_cell_size", "_cell_capacity", "_address2id"]
    meta = [None]
    if rank == src:
        meta[0] = {n: (tuple(getattr(index, n).shape), getattr(index, n).dtype) for n in small}
        meta[0]["vq"] = tuple(index.vq_codec.codebook.shape)
        meta[0]["pq"] = tuple(index.pq_codec.codebook.shape)
        meta[0]["max_id"] = index._max_id
        meta[0]["n_probe"] = index.n_probe
    dist.broadcast_object_list(meta, src=src, group=group)
    m = meta[0]
    for n in small:
        t = _bcast_tensor(getattr(index, n) if rank == src else None, *m[n], dev, src, group, rank)
        if rank != src:
            delattr(index, n)
            index.register_buffer(n, t)
    vq = _bcast_tensor(index.vq_codec.codebook if rank == src else None, m["vq"], torch.float32, dev, src, group, rank)
    pq = _bcast_tensor(index.pq_codec.codebook if rank == src else None, m["pq"], torch.float32, dev, src, group, rank)
    if rank != src:
        index.vq_codec.set_codebook(vq)
        index.pq_codec.set_codebook(pq)
        index._max_id, index.n_probe = m["max_id"], m["n_probe"]
    # one cell shard at a time: src lays it out, the ranks of that shard (one per query group) receive it
    from .index import ScanLayout
    mine = None
    for c in range(shards):
        owners = [c + shards * g for g in range(groups)]
        sizes = [None]
        lay = None
        if rank == src:
            lay = ScanLayout(index, c, shards)
            sizes[0] = (lay.n_blocks, lay.codes_scan.numel(), lay.block_valid.numel())
        dist.broadcast_object_list(sizes, src=src, group=group)
        n_blocks, n_codes, n_valid = sizes[0]
        if rank == src:
            parts = (lay.codes_scan, lay.block_valid, lay.cell_block_start)
            for o in owners:
                if o != src:
                    for t in parts:
                        dist.send(t, dst=o, group=group)
            if src in owners:
                mine = parts + (n_blocks,)
        elif rank in owners:
            parts = (torch.empty(n_codes, dtype=torch.uint8, device=dev), torch.empty(n_valid, dtype=torch.int32, device=dev),
                     torch.empty(index.n_cells + 1, dtype=torch.int32, device=dev))
            for t in parts:
                dist.recv(t, src=src, group=group)
            mine = parts + (n_blocks,)
        del lay
    index.adopt_shard(rank % shards, shards, *mine)
    if rank == src:
        torch.cuda.empty_cache()
    return index


def broadcast_state(index, src: int = 0, group=None):
    """Replicate rank ``src``'s FULL index state (reference layout included) to every rank -- for callers that want
    every rank able to add / remove; ``distribute`` is the search-only, memory-sharded alternative."""
    rank = dist.get_rank(group)
    dev = torch.device(index.device)
    names = ["_storage", "_is_empty", "_cell_start", "_cell_size", "_cell_capacity", "_address2id"]
    meta = [None]
    if rank == src:
        meta[0] = {n: (tuple(getattr(index, n).shape), getattr(index, n).dtype) for n in names}
        meta[0]["vq"] = tuple(index.vq_codec.codebook.shape)
        meta[0]["pq"] = tuple(index.pq_codec.codebook.shape)
        meta[0]["max_id"] = index._max_id
    dist.broadcast_object_list(meta, src=src, group=group)
    m = meta[0]
    for n in names:
        if rank != src:
            shape, dtype = m[n]
            delattr(index, n)
            index.register_buffer(n, torch.empty(shape, dtype=dtype, device=dev))
        dist.broadcast(getattr(index, n), src=src, group=group)
    vq = index.vq_codec.codebook if rank == src else torch.empty(m["vq"], dtype=torch.float32, device=dev)
    pq = index.pq_codec.codebook if rank == src else torch.empty(m["pq"], dtype=torch.float32, device=dev)
    dist.broadcast(vq, src=src, group=group)
    dist.broadcast(pq, src=src, group=group)
    if rank != src:
        index.vq_codec.set_codebook(vq)
        index.pq_codec.set_codebook(pq)
        index._max_id = m["max_id"]
    index._state_changed()
