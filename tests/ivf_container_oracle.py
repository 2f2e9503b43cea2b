"""numpy restatement of the IVF container's add / remove / lookups with holes (TEST INFRASTRUCTURE, in the spirit of
``oracle/``): the bookkeeping ``build.container_add`` / ``build.container_remove`` give IVFPQIndex, IVFPQRIndex,
IVFFlatIndex and IVFSQIndex.  The state is ``oracle.ivfpq_oracle.IndexState``; only its container fields are read or
written, and the code width is the store's, ``storage [code_size / 4, capacity, 4]`` u8, whatever ``n_subvectors``
says (IVFPQ: M bytes, IVFPQR: M + Mr, IVFFlat: the 4 d bytes of the fp32 column, IVFSQ: d or 2 d).

    add      free space of a cell = capacity - live items (is_empty == 0 in its range).  While some cell is short, every
             short cell grows in one round (ivfpq_oracle._expand: by its capacity in "double" mode, by expand_step_size
             in "step" mode or when its capacity is 0).  Item i goes to the ioa[i]-th empty slot of its cell, ascending
             address; its bytes, id and is_empty = 0 are written; cell_size[c] = max(cell_size[c], highest written
             position in c + 1); max_id = max(max_id, ids).  Default ids: max_id + 1, max_id + 2, ...
    remove   by ids (through get_address_by_id) or by address: entries outside [0, capacity), duplicates and holes are
             ignored; each removed slot gets is_empty = 1 and address2id = -1; cell_size is unchanged.
    lookups  get_address_by_id: the live slot holding the id, else -1; get_id_by_address: address2id inside
             [0, capacity), else -1.
    load     every buffer as given; max_id = max(address2id) (-1 for an empty store).

The statements are plain loops over cells and items: slow, and independent of the library's prefix sums and kernels.
"""
from __future__ import annotations

import numpy as np

from oracle import ivfpq_oracle as O


def empty(code_size, n_cells, initial_size, **fields) -> O.IndexState:
    """A fresh container of n_cells cells of initial_size slots, code_size bytes per item.  `fields` go to the
    IndexState (d_vector, n_subvectors, distance, codebooks, ...) for the searches that read the same state."""
    assert code_size % 4 == 0
    cap = n_cells * initial_size
    kw = dict(d_vector=code_size, n_subvectors=code_size, distance="euclidean",
              vq_codebook=np.zeros((0, n_cells), np.float32), pq_codebook=np.zeros((0, 0, 256), np.float32))
    kw.update(fields)
    return O.IndexState(n_cells=n_cells, storage=np.zeros((code_size // 4, cap, 4), np.uint8),
                        is_empty=np.ones(cap, np.uint8), cell_start=np.arange(n_cells, dtype=np.int64) * initial_size,
                        cell_size=np.zeros(n_cells, np.int64),
                        cell_capacity=np.zeros(n_cells, np.int64) + initial_size,
                        address2id=-np.ones(cap, np.int64), **kw)


def code_size(st) -> int:
    return st.storage.shape[0] * 4


def live_count(st, c) -> int:
    s, cap = int(st.cell_start[c]), int(st.cell_capacity[c])
    return int((st.is_empty[s:s + cap] == 0).sum())


def empty_slots(st, c) -> np.ndarray:
    """The empty slots of cell c, ascending."""
    s, cap = int(st.cell_start[c]), int(st.cell_capacity[c])
    return s + np.flatnonzero(st.is_empty[s:s + cap] != 0)


def add(st, codes, cells, ids=None, expand_mode="double", expand_step_size=128):
    """codes [code_size, n] u8, cells [n] -> (ids, write address [n])."""
    codes = np.ascontiguousarray(codes, np.uint8)
    cells = np.asarray(cells, np.int64)
    n = cells.shape[0]
    assert codes.shape == (code_size(st), n)
    assert ((cells >= 0) & (cells < st.n_cells)).all()
    ids = np.arange(n, dtype=np.int64) + st.max_id + 1 if ids is None else np.asarray(ids, np.int64)
    if n == 0:
        return ids, np.zeros(0, np.int64)
    counts = np.bincount(cells, minlength=st.n_cells)
    while True:
        short = [c for c in range(st.n_cells) if counts[c] > st.cell_capacity[c] - live_count(st, c)]
        if not short:
            break
        before = st.capacity
        O._expand(st, np.asarray(short, np.int64), expand_mode, expand_step_size)
        assert st.capacity > before, "an expansion round added no slot: the add would never end"
    ioa = O.get_ioa(cells)
    free = {c: empty_slots(st, c) for c in np.unique(cells)}
    write = np.array([free[c][r] for c, r in zip(cells, ioa)], np.int64)
    for i in range(n):
        a, c = write[i], cells[i]
        st.storage[:, a, :] = codes[:, i].reshape(-1, 4)
        st.address2id[a] = ids[i]
        st.is_empty[a] = 0
        st.cell_size[c] = max(st.cell_size[c], a - st.cell_start[c] + 1)
    st.max_id = max(st.max_id, int(ids.max()))
    return ids, write


def get_address_by_id(st, ids) -> np.ndarray:
    """The live slot holding each id, else -1 (the sequences keep live ids unique)."""
    out = -np.ones(len(ids), np.int64)
    for j, i in enumerate(np.asarray(ids, np.int64)):
        hit = np.flatnonzero((st.address2id == i) & (st.is_empty == 0))
        assert hit.size <= 1, f"id {i} is live in {hit.size} slots"
        if i >= 0 and hit.size:
            out[j] = hit[0]
    return out


def get_id_by_address(st, address) -> np.ndarray:
    return O.get_id_by_address(st.address2id, np.asarray(address, np.int64))


def remove(st, ids=None, address=None) -> np.ndarray:
    """-> the slots that became holes, ascending."""
    if ids is not None:
        address = get_address_by_id(st, ids)
    elif address is None:
        raise RuntimeError("Need either ids or address")
    gone = sorted({int(a) for a in np.asarray(address, np.int64) if 0 <= a < st.capacity and st.is_empty[a] == 0})
    for a in gone:
        st.is_empty[a] = 1
        st.address2id[a] = -1
    return np.asarray(gone, np.int64)


def load(st) -> O.IndexState:
    """A checkpoint load: the buffers as given, max_id re-derived."""
    st.max_id = int(st.address2id.max()) if st.capacity else -1
    return st


def codes_at(st, address) -> np.ndarray:
    """[code_size, n] bytes of the given slots."""
    s = st.storage[:, np.asarray(address, np.int64), :]
    return s.transpose(0, 2, 1).reshape(code_size(st), -1)
