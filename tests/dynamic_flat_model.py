"""A pure-Python model of the dynamic flat index's slot rules (the reference's DynamicFlatIndex,
include/svs/index/flat/dynamic_flat.h:214-367), and the mutation script the dynamic flat tests run.

tests/test_dynamic_flat_slots.py checks the model against the reference's own index (oracle/_ref façade) without a GPU;
tests/test_gpu_dynamic_flat.py then checks the GPU index against the model and against a static Flat over the rows the
model says are live."""
import numpy as np

EMPTY, VALID = 0, 1
RESERVED = 2**64 - 1


class SlotModel:
    """Slots Valid / Empty, external ids, first_empty_, and one payload per slot (the pool row it holds)."""

    def __init__(self, ids, payload=None):
        ids = [int(i) for i in ids]
        self.status = [VALID] * len(ids)
        self.ext = list(ids)
        self.payload = list(payload) if payload is not None else [None] * len(ids)
        self.slot_of = {e: s for s, e in enumerate(ids)}
        self.first_empty = len(ids)

    def add(self, ids, reuse_empty=False, payload=None):
        """add_points: Empty slots from first_empty_ (from 0 with reuse_empty), then appended ones; refused before any
        change on a repeated, present or reserved id."""
        ids = [int(i) for i in ids]
        payload = list(payload) if payload is not None else [None] * len(ids)
        if len(set(ids)) != len(ids) or any(i == RESERVED or i in self.slot_of for i in ids):
            raise ValueError("repeated, present or reserved id")
        slots = []
        s = 0 if reuse_empty else self.first_empty
        while s < len(self.status) and len(slots) < len(ids):
            if self.status[s] == EMPTY:
                slots.append(s)
            s += 1
        while len(slots) < len(ids):
            slots.append(len(self.status))
            self.status.append(EMPTY)
            self.ext.append(RESERVED)
            self.payload.append(None)
        for s, e, p in zip(slots, ids, payload):
            self.status[s], self.ext[s], self.payload[s] = VALID, e, p
            self.slot_of[e] = s
        if slots:
            self.first_empty = max(self.first_empty, slots[-1] + 1)
        return slots

    def delete(self, ids):
        """delete_entries: every id present and listed once, else nothing changes; the slots are Empty at once."""
        ids = [int(i) for i in ids]
        if len(set(ids)) != len(ids) or any(i not in self.slot_of for i in ids):
            raise KeyError("unknown or repeated id")
        for e in ids:
            s = self.slot_of.pop(e)
            self.status[s], self.ext[s], self.payload[s] = EMPTY, RESERVED, None
            self.first_empty = min(self.first_empty, s)

    def compact(self):
        """compact: the Valid slots, in ascending order, move to [0, size); first_empty_ = size."""
        live = self.live_slots()
        self.ext = [self.ext[s] for s in live]
        self.payload = [self.payload[s] for s in live]
        self.status = [VALID] * len(live)
        self.slot_of = {e: s for s, e in enumerate(self.ext)}
        self.first_empty = len(live)

    def live_slots(self):
        return np.array([s for s, st in enumerate(self.status) if st == VALID], dtype=np.int64)

    def live_ids(self):
        return np.array([self.ext[s] for s in self.live_slots()], dtype=np.uint64)

    def live_payload(self):
        return np.array([self.payload[s] for s in self.live_slots()], dtype=np.int64)

    def export(self):
        return np.array(self.status, dtype=np.uint8), np.array(self.ext, dtype=np.uint64)


# ragged add sizes that cross several 256-row tiles
RAGGED = (1, 37, 255, 256, 257, 300)


def mutation_script(model, n0, seed):
    """The mutation steps, generated lazily from the model's state (apply each step to the model before asking for the
    next): delete 10 % at random; add with and without reuse_empty; grow across several 256-row tiles with ragged
    batch sizes; delete then re-add the same ids; compact.  Steps: ("delete", ids) | ("add", pool_rows, ids, reuse) |
    ("compact",).  Pool rows of adds are taken in order from row n0; new external ids are not contiguous."""
    rng = np.random.default_rng(seed)
    row = n0
    next_id = 5 * n0 + 11

    def fresh(count):
        nonlocal row, next_id
        rows = np.arange(row, row + count)
        ids = next_id + 3 * np.arange(count, dtype=np.uint64)
        row += count
        next_id += 3 * count + 1
        return rows, ids

    live = model.live_ids()
    yield ("delete", rng.choice(live, size=len(live) // 10, replace=False))
    yield ("add",) + fresh(max(1, n0 // 20)) + (False,)
    yield ("add",) + fresh(max(1, n0 // 20)) + (True,)
    for c in RAGGED:
        yield ("add",) + fresh(c) + (c % 2 == 1,)
    live = model.live_ids()
    gone = rng.choice(live, size=len(live) // 8, replace=False)
    yield ("delete", gone)
    rows, _ = fresh(len(gone))   # the same ids again, with new rows
    yield ("add", rows, gone, True)
    yield ("compact",)


def pool_size(n0):
    """Rows a mutation_script over n0 initial rows takes from its pool."""
    grown = n0 + 2 * max(1, n0 // 20) + sum(RAGGED)
    return grown + grown // 8 + 1


def run_script(index, model, pool, n0, seed, check):
    """Applies the mutation script to `index` (any object with add / delete / compact, add returning the slots) and to
    the model in step, calling check(step) after each step."""
    for step in mutation_script(model, n0, seed):
        if step[0] == "delete":
            index.delete(step[1])
            model.delete(step[1])
        elif step[0] == "add":
            _, rows, ids, reuse = step
            got = index.add(pool[rows], ids, reuse_empty=reuse)
            want = model.add(ids, reuse_empty=reuse, payload=rows)
            assert np.asarray(got).tolist() == want, step[:1]
        else:
            index.compact()
            model.compact()
        check(step)
