"""MutableBuffer semantics of the dynamic index's search, on the CPU.

* The one-by-one restatement (tests/mutable_model.py) reproduces the reference's known answers
  (/root/reference/tests/svs/index/vamana/search_buffer.cpp:618-910, "MutableBuffer": "All Valid", "Collapsing" and the
  three "Push-back initialization" sections, which pin the entry-point path push_back + sort).
* The lean kernel's MUT mode merges candidates in groups of up to 32 (csrc/search_fast.cuh).  Fuzzing with random
  validity, ties and repeated ids shows that each group leaves the same buffer, valid count and next() / done()
  behaviour as inserting its candidates one by one, and that a buffer with too little room is always detected.
"""
import numpy as np
import pytest

from mutable_model import GroupState, MutableBuffer, group_merge


def entries(b):
    return [(e[0], e[1], e[2]) for e in b.c]


def test_known_answers_all_valid():
    b = MutableBuffer(4)
    b.insert(0, 100, True)
    assert entries(b) == [(0, 100, True)] and not b.full()
    b.insert(1, 50, True)
    assert entries(b) == [(1, 50, True), (0, 100, True)] and not b.full()
    b.insert(2, 150, True)
    assert entries(b) == [(1, 50, True), (0, 100, True), (2, 150, True)] and not b.full()
    b.insert(3, 40, True)
    four = [(3, 40, True), (1, 50, True), (0, 100, True), (2, 150, True)]
    assert entries(b) == four and b.full()
    b.insert(4, 1000, True)                       # full: a larger element has no effect
    assert entries(b) == four and b.full()
    b.insert(5, 0, True)                          # a smaller one shifts everything back
    assert entries(b) == [(5, 0, True), (3, 40, True), (1, 50, True), (0, 100, True)] and b.full()
    b.insert(6, 1, False)                         # an invalid one in front grows the buffer
    grown = [(5, 0, True), (6, 1, False), (3, 40, True), (1, 50, True), (0, 100, True)]
    assert entries(b) == grown and b.full()
    b.insert(7, 2000, False)                      # an invalid one at the end is dropped
    assert entries(b) == grown and b.full()


def test_known_answers_collapsing():
    b = MutableBuffer(4)
    for i in range(100):
        b.insert(i, float(1000 - i), False)
    assert len(b.c) == 100 and not b.full() and b.valid == 0
    for n, (id, key) in enumerate(((100, 10), (101, 8), (102, 6)), start=1):
        b.insert(id, float(key), True)
        assert len(b.c) == 100 + n and not b.full() and b.valid == n
    b.insert(103, 4.0, True)
    assert len(b.c) == 4 and b.full()


def push_all(b, items):
    """push_back each (id, key, valid, expected size, expected valid count, expected full())."""
    for id, key, valid, size, nvalid, full in items:
        b.push_back(id, float(key), valid)
        assert (len(b.c), b.valid, b.full()) == (size, nvalid, full), id


def walk(b, want):
    """next() until done(): the ids in order, each entry marked visited."""
    for id in want:
        assert not b.done()
        pos = b.best
        assert b.next() == id and b.c[pos][3]
    assert b.done()


# search_buffer.cpp:727-910, "Push-back initialization" on MutableBuffer{{2, 4}}: the entry-point path
# (push_back + sort) of greedy search, including the sort-time trimming of trailing invalid entries.
def test_known_answers_push_back_full_buffer():
    b = MutableBuffer(2, 4)
    push_all(b, [(1, 10, True, 1, 1, False), (2, 9, False, 2, 1, False), (3, 8, True, 3, 2, False),
                 (4, 7, True, 4, 3, False), (5, 6, False, 5, 3, False), (6, 5, False, 6, 3, False),
                 (7, 4, True, 7, 4, True),
                 (8, 3, True, 7, 4, True),            # another valid one has no effect
                 (8, 2, False, 8, 4, True),           # an invalid one still grows the buffer
                 (9, 100, False, 9, 4, True), (10, 110, False, 10, 4, True)])
    b.sort()                                          # the invalid tail falls off
    assert len(b.c) == 8 and b.valid == 4 and b.c[-1][2]
    assert entries(b) == [(8, 2, False), (7, 4, True), (6, 5, False), (5, 6, False), (4, 7, True), (3, 8, True),
                          (2, 9, False), (1, 10, True)]
    walk(b, [8, 7, 6, 5, 4])


def test_known_answers_push_back_partially_full_buffer():
    b = MutableBuffer(2, 4)
    push_all(b, [(1, 10, True, 1, 1, False), (2, 9, False, 2, 1, False), (3, 8, True, 3, 2, False),
                 (4, 7, True, 4, 3, False), (5, 20, False, 5, 3, False)])
    b.sort()                                          # invariant 6 not active: the last entry may be invalid
    assert len(b.c) == 5 and b.valid == 3 and not b.c[-1][2]
    walk(b, [4, 3])


def test_known_answers_push_back_non_full_buffer():
    b = MutableBuffer(2, 4)
    push_all(b, [(1, 10, True, 1, 1, False), (2, 9, False, 2, 1, False), (3, 8, False, 3, 1, False)])
    b.sort()
    assert len(b.c) == 3 and b.valid == 1 and b.c[-1][2]
    walk(b, [3, 2, 1])


def run_pair(rng, window, capacity, steps, p_invalid, nkeys, room=None):
    """Random groups + next() on both models; returns how many groups overflowed `room`."""
    ref = MutableBuffer(window, capacity)
    st = GroupState(window, capacity)
    key_of, valid_of = {}, {}
    overflowed = 0
    for step in range(steps):
        if rng.random() < 0.3 and not ref.done():
            want = ref.next()
            assert st.next() == want, step
        else:
            g = int(rng.integers(1, 33))
            ids = rng.choice(200, size=g, replace=False)   # distinct inside a group, repeats across groups
            cands = []
            for id in ids.tolist():
                key = key_of.setdefault(id, float(rng.integers(0, nkeys)))   # same id => same key; many ties
                valid = valid_of.setdefault(id, bool(rng.random() >= p_invalid))
                cands.append((id, key, valid))
            for id, key, valid in cands:
                ref.insert(id, key, valid)
            snapshot = (list(map(list, st.buf)), st.nvalid, st.roi_end, st.cursor)
            ok = group_merge(st, cands, room)
            if not ok:
                # the kernel stops such a query and re-runs it with more room: restart the model from scratch
                overflowed += 1
                assert room is not None and len(snapshot[0]) + len(cands) > room
                return overflowed
        assert [(e[0], e[1], e[2], e[3]) for e in st.buf] == [tuple(e) for e in ref.c], step
        assert st.nvalid == ref.valid, step
        assert st.roi_end == (len(ref.c) if ref.valid < window else ref.roi_end), step
        # next()/done(): both point at the same first unvisited entry inside the region of interest
        first = next((i for i in range(st.roi_end) if not st.buf[i][3]), None)
        assert (first is None) == ref.done(), step
        if first is not None:
            assert first == ref.best, step
    return overflowed


@pytest.mark.parametrize("window,capacity", [(1, 10), (10, 20), (15, 15), (4, 4), (3, 7), (32, 64)])
@pytest.mark.parametrize("p_invalid", [0.0, 0.1, 0.5, 0.9])
def test_group_merge_equals_one_by_one(window, capacity, p_invalid):
    rng = np.random.default_rng(window * 1000 + capacity * 10 + int(p_invalid * 10))
    for trial in range(6):
        run_pair(rng, window, capacity, 400, p_invalid, nkeys=int(rng.choice([4, 16, 1000])))


@pytest.mark.parametrize("window,capacity", [(10, 20), (15, 15)])
def test_tiny_room_is_always_detected(window, capacity):
    """With a buffer of `capacity + 2` entries a query either matches the one-by-one model step for step or reports
    an overflow; it never silently differs."""
    rng = np.random.default_rng(capacity)
    overflowed = 0
    for trial in range(40):
        overflowed += run_pair(rng, window, capacity, 300, 0.5, nkeys=1000, room=capacity + 2)
    assert overflowed > 0
