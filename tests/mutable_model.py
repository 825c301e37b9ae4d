"""Plain-Python models of the dynamic index's search (shared by the CPU and GPU tests; test infrastructure only).

* :class:`MutableBuffer`  -- a line-by-line restatement of the reference's one-by-one ``MutableBuffer``
  (include/svs/index/vamana/dynamic_search_buffer.h:41-617).
* :func:`group_merge`     -- what the lean kernel's MUT mode does with one group of up to 32 candidates
  (csrc/search_fast.cuh): survivors against the state before the group, a stable merge, then the cut behind the
  capacity-th valid entry and roi_end behind the window-th.
* :func:`mutable_search`  -- ``MutableVamanaIndex::search`` of one query (dynamic_index.h:482-571 with greedy_search,
  greedy_search.h:124-203) over any distance function.
"""
from __future__ import annotations

import bisect


class MutableBuffer:
    """Entries are [id, key, valid, visited]; keys are ordered by ``<`` (negate them for std::greater)."""

    def __init__(self, window: int, capacity: int | None = None):
        capacity = window if capacity is None else capacity
        self.target, self.cap = window, capacity
        self.c = []
        self.best = 0
        self.roi_end = 0
        self.valid = 0

    def full(self):
        return self.valid == self.cap

    def done(self):
        return self.best == (len(self.c) if self.valid < self.target else self.roi_end)

    def next(self):
        node = self.c[self.best]
        node[3] = True
        self.best += 1
        while self.best != self.roi_end and self.c[self.best][3]:
            self.best += 1
        return node[0]

    def push_back(self, id, key, valid):
        if self.full() and valid:
            return
        self.c.append([id, key, valid, False])
        self.valid += int(valid)
        self.roi_end = len(self.c)

    def sort(self):
        self.c.sort(key=lambda e: e[1])
        if self.valid < self.target:
            self.roi_end = len(self.c)
            return
        count = 0
        for i, e in enumerate(self.c):
            if e[2]:
                count += 1
                if count == self.target:
                    self.roi_end = i + 1
                    break
        self.best = 0
        while self.best < self.roi_end and self.c[self.best][3]:
            self.best += 1
        if self.valid - self.cap == 0:
            while not self.c[-1][2]:
                self.c.pop()

    def _walk_back(self, i):
        while not self.c[i][2]:
            i -= 1
        return i

    def insert(self, id, key, valid):
        """Returns the reference's insert() value: size() when skipped, size()+1 for a repeat, else the position."""
        if self.full() and self.c[-1][1] < key:
            return len(self.c)
        pos = bisect.bisect_right(self.c, key, key=lambda e: e[1])   # lower_bound with !cmp(d, other)
        j = pos
        while j > 0:
            j -= 1
            if self.c[j][1] < key:
                break
            if self.c[j][0] == id:
                return len(self.c) + 1
        self.valid += int(valid)
        self._unsafe_insert([id, key, valid, False], pos)
        self.best = min(self.best, pos)
        return pos

    def _unsafe_insert(self, e, offset):
        self.c.insert(offset, e)
        at_threshold = self.valid == self.target
        below = offset < self.roi_end
        if self.valid < self.target:
            self.roi_end = len(self.c)
        elif at_threshold:
            if e[2]:
                assert self.roi_end == len(self.c) - 1
                while not self.c[self.roi_end][2]:
                    self.roi_end -= 1
                self.roi_end += 1
            elif below:
                self.roi_end += 1
        elif below:
            if not e[2]:
                self.roi_end += 1
            else:
                self.roi_end -= 1
                while not self.c[self.roi_end][2]:
                    self.roi_end -= 1
                self.roi_end += 1
        slack = self.valid - self.cap
        if self.target == self.cap:
            del self.c[self.roi_end:]
            if slack > 0:
                assert slack == 1
                self.valid -= 1
        elif slack == 0:
            del self.c[self._walk_back(len(self.c) - 1) + 1:]
        elif slack > 0:
            assert slack == 1 and self.c[-1][2]
            del self.c[self._walk_back(len(self.c) - 2) + 1:]
            self.valid -= 1

    def cleanup(self):
        self.c = [e for e in self.c if e[2]]


class GroupState:
    """The kernel's per-query state: entries [id, key, valid, visited], valid count, roi_end, cursor."""

    def __init__(self, window, capacity):
        self.W, self.C = window, capacity
        self.buf, self.nvalid, self.roi_end, self.cursor = [], 0, 0, 0

    def next(self):
        """First unvisited entry inside [cursor, roi_end) -- None when done()."""
        for pos in range(self.cursor, self.roi_end):
            if not self.buf[pos][3]:
                self.buf[pos][3] = True
                self.cursor = pos + 1
                return self.buf[pos][0]
        return None


def group_merge(st: GroupState, cands, room: int | None = None):
    """Merge one group of (id, key, valid) candidates (distinct ids, adjacency order) the way the MUT kernel does.
    ``room`` is the buffer's entry limit (buf_cap); returns False when the query would overflow it."""
    full = st.nvalid == st.C
    back = st.buf[-1][1] if full else None
    surv = []
    for id, key, valid in cands:
        if full and back < key:
            continue
        pos = bisect.bisect_right([e[1] for e in st.buf], key)
        j, dup = pos, False
        while j > 0:
            j -= 1
            if st.buf[j][1] < key:
                break
            if st.buf[j][0] == id:
                dup = True
                break
        if not dup:
            surv.append((pos, id, key, valid))
    if not surv:
        return True
    minpos = min(s[0] for s in surv)
    merged = list(st.buf)
    # stable: survivors after the old entries of equal key, among themselves in adjacency order
    for _, id, key, valid in sorted(surv, key=lambda s: s[2]):
        merged.insert(bisect.bisect_right([e[1] for e in merged], key), [id, key, valid, False])
    total = len(merged)
    if room is not None:
        merged = merged[:room]
    v, cut, roiw = 0, None, None
    for i, e in enumerate(merged):
        if e[2]:
            v += 1
            if v == st.W and roiw is None:
                roiw = i
            if v == st.C:
                cut = i
                break
    if cut is not None:
        merged = merged[:cut + 1]
        st.nvalid = st.C
    else:
        st.nvalid = v
        if total > len(merged):
            return False
    st.buf = merged
    st.roi_end = roiw + 1 if st.nvalid >= st.W else len(merged)
    st.cursor = min(st.cursor, minpos)
    return True


def mutable_search(entry_point, neighbours, key_of, valid_of, window, capacity, k):
    """One query of MutableVamanaIndex::search with the one-by-one buffer: ``neighbours(v)`` is v's adjacency row,
    ``key_of(ids)`` the keys (sign * distance) of a list of ids, ``valid_of(v)`` False for a Deleted slot.
    Returns the first k valid (slot, key) pairs after cleanup()."""
    if capacity < k:
        window = capacity = k
    b = MutableBuffer(window, capacity)
    b.push_back(entry_point, float(key_of([entry_point])[0]), valid_of(entry_point))
    b.sort()
    while not b.done():
        node = b.next()
        row = list(neighbours(node))
        if not row:
            continue
        for id, key in zip(row, key_of(row)):
            b.insert(id, float(key), valid_of(id))
    b.cleanup()
    return [(e[0], e[1]) for e in b.c[:k]]
