"""CPU: the holes-aware container oracle (ivf_container_oracle.py) -- equal to ivfpq_oracle.container_add on hole-free
sequences, and pinned rule by rule on designed cases -- and the growth rule of build.container_add as a pure function,
so that the zero-capacity rule is checked without running an expansion loop."""
import numpy as np
import pytest
import torch

import ivf_container_oracle as CO
from oracle import ivfpq_oracle as O


def _codes(rng, width, n):
    return rng.integers(0, 256, (width, n)).astype(np.uint8)


def _same_state(a, b):
    for name in ("storage", "is_empty", "cell_start", "cell_size", "cell_capacity", "address2id"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    assert a.capacity == b.capacity and a.max_id == b.max_id


# ----------------------------------------------------------------------------------------- against ivfpq_oracle
@pytest.mark.parametrize("width", [8, 24, 64])
@pytest.mark.parametrize("mode", ["double", "step"])
@pytest.mark.parametrize("initial", [1, 3, 8])
def test_hole_free_sequences_equal_container_add(width, mode, initial):
    """Without holes the new oracle places as ivfpq_oracle.container_add: the same write addresses, buffers, capacity
    and cell_size, with default and explicit ids, for any code width (IVFPQ M, IVFPQR M + Mr, IVFFlat 4 d)."""
    rng = np.random.default_rng(width * 100 + initial)
    C = 7
    old = O.empty_state(width, width, C, initial)
    old.storage = np.zeros((width // 4, old.capacity, 4), np.uint8)
    new = CO.empty(width, C, initial)
    for step, n in enumerate((1, 40, 300, 2, 17)):
        cells = rng.choice([0, 2, 3, 6], n)                           # cells 1, 4, 5 are never chosen
        codes = _codes(rng, width, n)
        ids = None if step % 2 == 0 else rng.choice(10 ** 6, n, replace=False) + 10 ** 4
        oid, oadr = O.container_add(old, codes, cells, ids, expand_mode=mode, expand_step_size=5)
        nid, nadr = CO.add(new, codes, cells, ids, expand_mode=mode, expand_step_size=5)
        assert np.array_equal(oid, nid) and np.array_equal(oadr, nadr)
        _same_state(old, new)
        assert np.array_equal(CO.codes_at(new, nadr), codes)
    assert np.array_equal(new.cell_size, [CO.live_count(new, c) for c in range(C)])


# ----------------------------------------------------------------------------------------- designed cases
def _filled(C=3, initial=8, per_cell=(5, 3, 0), mode="double", step=4):
    st = CO.empty(8, C, initial)
    cells = np.repeat(np.arange(C), per_cell)
    CO.add(st, np.zeros((8, cells.size), np.uint8) + np.arange(cells.size, dtype=np.uint8), cells,
           expand_mode=mode, expand_step_size=step)
    return st


def test_holes_are_filled_lowest_address_first():
    st = _filled()                                                    # cell 0 holds ids 0..4 at 0..4
    CO.remove(st, ids=np.array([3, 1]))
    ids, adr = CO.add(st, np.zeros((8, 4), np.uint8), np.array([0, 1, 0, 0]))
    assert adr.tolist() == [1, 11, 3, 5]                              # holes 1, 3 in input order, then the tail
    assert ids.tolist() == [8, 9, 10, 11]
    assert st.cell_size.tolist() == [6, 4, 0]


def test_space_of_removed_items_is_reused_without_expanding():
    st = _filled(initial=5, per_cell=(5, 5, 5))                       # every cell full
    cap = st.capacity
    CO.remove(st, address=np.array([0, 2, 4, 7]))
    _, adr = CO.add(st, np.zeros((8, 4), np.uint8), np.array([0, 0, 0, 1]))
    assert st.capacity == cap and adr.tolist() == [0, 2, 4, 7]
    CO.add(st, np.zeros((8, 1), np.uint8), np.array([1]))             # one more than the cell's holes: it doubles
    assert st.cell_capacity.tolist() == [5, 10, 5] and st.capacity == cap + 5


def test_cell_size_is_a_high_water_mark():
    st = _filled()
    CO.remove(st, ids=np.array([4, 3]))                               # the tail of cell 0
    assert st.cell_size[0] == 5 and CO.live_count(st, 0) == 3
    _, adr = CO.add(st, np.zeros((8, 1), np.uint8), np.array([0]))
    assert adr.tolist() == [3] and st.cell_size[0] == 5               # below the mark: unchanged
    _, adr = CO.add(st, np.zeros((8, 2), np.uint8), np.array([0, 0]))
    assert adr.tolist() == [4, 5] and st.cell_size[0] == 6            # past it: highest written position + 1


def test_step_and_double_growth():
    """A short cell grows by its capacity ("double") or by expand_step_size ("step"), round after round, until the
    add fits; the cells after it shift, the others keep their size."""
    for mode, first, second in (("double", 8, 16), ("step", 7, 13)):
        st = CO.empty(8, 3, 4)
        CO.add(st, np.zeros((8, 13), np.uint8), np.array([0] * 6 + [1] * 7), expand_mode=mode, expand_step_size=3)
        assert st.cell_capacity.tolist() == [first, first, 4], mode   # 6 and 7 items: 4 -> 8, or 4 -> 7
        assert st.cell_start.tolist() == [0, first, 2 * first] and st.capacity == 2 * first + 4
        CO.add(st, np.zeros((8, 5), np.uint8), np.zeros(5, np.int64), expand_mode=mode, expand_step_size=3)
        assert st.cell_capacity[0] == second, mode                    # 11 items: 8 -> 16, or 7 -> 10 -> 13
        assert st.cell_start[1] == second and st.cell_size[0] == 11


@pytest.mark.parametrize("mode", ["double", "step"])
def test_zero_capacity_cell(mode):
    """A cell of capacity 0 (initial_size=0, or a loaded state) grows by expand_step_size in both modes, then by its
    capacity in "double" mode."""
    st = CO.empty(8, 3, 0)
    CO.add(st, np.zeros((8, 2), np.uint8), np.array([1, 1]), expand_mode=mode, expand_step_size=5)
    assert st.cell_capacity.tolist() == [0, 5, 0] and st.cell_start.tolist() == [0, 0, 5]
    _, adr = CO.add(st, np.zeros((8, 9), np.uint8), np.array([1] * 4 + [2] * 5), expand_mode=mode, expand_step_size=5)
    assert st.cell_capacity.tolist() == [0, 10, 5]                   # 6 in cell 1: 5 -> 10 either way
    assert adr.tolist() == [2, 3, 4, 5, 10, 11, 12, 13, 14] and st.cell_size.tolist() == [0, 6, 5]
    CO.add(st, np.zeros((8, 11), np.uint8), np.array([1] * 11), expand_mode=mode, expand_step_size=5)
    assert st.cell_capacity[1] == 20                                  # 17 items: 10 -> 20, or 10 -> 15 -> 20
    CO.add(st, np.zeros((8, 4), np.uint8), np.array([1] * 4), expand_mode=mode, expand_step_size=5)
    assert st.cell_capacity[1] == (40 if mode == "double" else 25)    # 21 items


def test_zero_capacity_expand_is_one_round():
    """ivfpq_oracle._expand on a zero-capacity cell adds expand_step_size slots in either mode (one call: no loop)."""
    for mode in ("double", "step"):
        st = O.empty_state(8, 8, 2, 0)
        O._expand(st, np.array([1]), mode, 6)
        assert st.cell_capacity.tolist() == [0, 6] and st.capacity == 6 and (st.is_empty == 1).all()


def test_remove_ignores_unknown_negative_duplicate_and_holes():
    st = _filled()                                                    # ids 0..7: cell 0 at 0..4, cell 1 at 8..10
    gone = CO.remove(st, ids=np.array([2, 2, -1, -5, 99, 9]))
    assert gone.tolist() == [2]                                       # 9 is not an id either
    gone = CO.remove(st, ids=np.array([6, 2, 6]))                     # 2 is gone already
    assert gone.tolist() == [9]
    before = st.is_empty.copy()
    gone = CO.remove(st, address=np.array([-1, 2, 5, 9, st.capacity, st.capacity + 7, 0, 0]))
    assert gone.tolist() == [0]                                       # 2, 9 holes; 5 never held an item
    assert np.array_equal(np.flatnonzero(before != st.is_empty), [0])
    assert st.address2id[[0, 2, 9]].tolist() == [-1, -1, -1] and st.cell_size.tolist() == [5, 3, 0]
    assert st.max_id == 7                                             # removing never lowers max_id


def test_lookups():
    st = _filled()
    CO.remove(st, ids=np.array([1]))
    CO.add(st, np.zeros((8, 1), np.uint8), np.array([1]), ids=np.array([1]))
    ids = np.array([0, 1, 2, 5, 7, 8, -1, 100])
    assert CO.get_address_by_id(st, ids).tolist() == [0, 11, 2, 8, 10, -1, -1, -1]
    adr = np.array([-3, 0, 1, 8, 11, 12, st.capacity, st.capacity + 1])
    assert CO.get_id_by_address(st, adr).tolist() == [-1, 0, -1, 5, 1, -1, -1, -1]


def test_load_rederives_max_id():
    st = _filled()
    CO.remove(st, ids=np.array([7, 6]))
    assert CO.load(st).max_id == 5
    assert CO.add(st, np.zeros((8, 1), np.uint8), np.array([2]))[0].tolist() == [6]
    assert CO.load(CO.empty(8, 4, 0)).max_id == -1


# ----------------------------------------------------------------------------------------- the library's growth rule
def test_growth_rule_zero_capacity():
    """build.growth, the rule container_add applies once per expansion round: a short cell of capacity 0 grows by
    expand_step_size in "double" mode (doubling it would add nothing, and the round would repeat forever); every
    other cell as the reference: by its capacity ("double") or by expand_step_size ("step"); cells with room by 0."""
    from torchpq_b200 import build
    cap = torch.tensor([0, 3, 5, 0, 1], dtype=torch.long)
    short = torch.tensor([True, True, False, False, True])
    assert build.growth(cap, short, "double", 7).tolist() == [7, 3, 0, 0, 1]
    assert build.growth(cap, short, "step", 7).tolist() == [7, 7, 0, 0, 7]
    big = torch.tensor([2 ** 40, 0], dtype=torch.long)
    assert build.growth(big, torch.tensor([True, True]), "double", 128).tolist() == [2 ** 40, 128]
    assert build.growth(big, torch.tensor([False, False]), "double", 128).tolist() == [0, 0]
