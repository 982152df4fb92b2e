"""GPU: every entry point that changes the device store voids what is keyed to the store's version — a prepared plan is refused as
stale, the closed token of kb_datalog_fixpoint / kb_datalog_maintain is gone unless the call records it again — and leaves the store
equal to a host model of its segments. A load that is rejected still empties the store, so it voids the token too."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import helpers as H
from tests.window_oracle import as_rows, rows_set

pytestmark = pytest.mark.gpu

_EMP = {}


def employees():
    if "d" not in _EMP:
        _EMP["d"] = datagen.employee_dataset(400)
    return _EMP["d"]


def rel_rows(r):
    return r.to_numpy([0, 1, 2]) if r.n_rows else np.empty((0, 3), np.uint32)


class Window:
    """tagged base segments on the device and the same on the host, plus the inferred facts; check() compares them"""

    def __init__(self, cx, d):
        self.cx = cx
        self.newp = d.n_ids + 10  # a predicate of its own for the inferred facts
        self.rules = [{"premise": [c.pattern(c.V(0), c.K(d.ids["foaf:name"]), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(self.newp), c.V(1))],
                       "filters": []}]
        self.segs = {}
        self.inferred = set()
        cx.store_clear()

    def append(self, tag, rows):
        rows = np.asarray(rows, np.uint32).reshape(-1, 3)
        self.cx.store_append(rows[:, 0], rows[:, 1], rows[:, 2], tag)
        self.segs[tag] = rows

    def fixpoint(self):
        rel, _ = self.cx.datalog_fixpoint(self.rules)
        self.inferred = rows_set(rel_rows(rel))
        assert self.inferred and all(r[1] == self.newp for r in self.inferred)

    def closed(self):
        """whether kb_datalog_maintain accepts the store as closed (nothing evicted, nothing added: the store does not change)"""
        try:
            self.cx.datalog_maintain(self.rules)
            return True
        except c.KolibrieError as e:
            assert e.status == c.KB_E_INVALID and "not closed" in e.message, e
            return False

    def rows(self):
        parts = list(self.segs.values()) + [as_rows(self.inferred)]
        return np.concatenate(parts, axis=0) if parts else np.empty((0, 3), np.uint32)

    def check(self, label):
        want = self.rows()
        s, p, o = self.cx.store_download()
        H.assert_same_bag(np.stack([s, p, o], axis=1), want, f"{label}: store")
        assert self.cx.store_size()[0] == len(want), label


def split(d, k):
    rows = np.stack([d.s, d.p, d.o], axis=1).astype(np.uint32)
    return [rows[i::k] for i in range(k)]


def setup(cx, closed):
    """three tagged segments, closed under the rules (or not), indexed, with a plan prepared over them"""
    d = employees()
    w = Window(cx, d)
    for tag, rows in enumerate(split(d, 3), start=1):
        w.append(tag, rows)
    if closed:
        w.fixpoint()
    cx.build_index()
    js, pats, filt = datagen.employee_queries(d)["cfg1"]
    plan = cx.prepare_star_join(js, pats, filt, ring=2)
    assert plan.collect(plan.submit()) > 0
    return d, w, plan


def op_clear(cx, d, w, tmp_path, keep):
    cx.store_clear()
    w.segs, w.inferred = {}, set()


def op_load(cx, d, w, tmp_path, keep):
    rows = split(d, 3)[0]
    cx.store_load(rows[:, 0], rows[:, 1], rows[:, 2])
    w.segs, w.inferred = {0: rows}, set()


def op_load_device(cx, d, w, tmp_path, keep):
    import torch

    rows = split(d, 3)[1]
    cols = [torch.from_numpy(np.ascontiguousarray(rows[:, j])).cuda() for j in range(3)]
    keep.append(cols)
    cx.store_load_device(cols[0].data_ptr(), cols[1].data_ptr(), cols[2].data_ptr(), len(rows))
    w.segs, w.inferred = {0: rows}, set()


def op_append(cx, d, w, tmp_path, keep):
    w.append(7, split(d, 5)[2])


def op_append_device(cx, d, w, tmp_path, keep):
    import torch

    rows = split(d, 5)[3]
    cols = [torch.from_numpy(np.ascontiguousarray(rows[:, j])).cuda() for j in range(3)]
    keep.append(cols)
    cx.store_append_device(cols[0].data_ptr(), cols[1].data_ptr(), cols[2].data_ptr(), len(rows), 7)
    w.segs[7] = rows


def op_append_file(cx, d, w, tmp_path, keep):
    rows = split(d, 5)[4]
    path = str(tmp_path / "slide.kbs")
    c.segment_write(path, rows[:, 0], rows[:, 1], rows[:, 2], tag=7)
    cx.store_append_file(path, 7)
    w.segs[7] = rows


def op_evict(cx, d, w, tmp_path, keep):
    cx.store_evict(2)
    del w.segs[2]


def op_delete(cx, d, w, tmp_path, keep):
    gone = np.concatenate([w.segs[1][::4], w.segs[3][1::5]], axis=0)
    cx.store_delete(gone[:, 0], gone[:, 1], gone[:, 2])
    drop = rows_set(gone)  # (every copy of a deleted triple goes)
    for t, rows in w.segs.items():
        w.segs[t] = rows[np.array([tuple(r) not in drop for r in rows.tolist()], dtype=bool).reshape(-1)]
    w.inferred -= drop


def op_star_join_host(cx, d, w, tmp_path, keep):
    rows = split(d, 1)[0]
    js, pats, filt = datagen.employee_queries(d)["cfg1"]
    out, _ = cx.star_join_host(rows[:, 0], rows[:, 1], rows[:, 2], js, pats, filt)
    assert len(out) > 0
    w.segs, w.inferred = {0: rows}, set()


def op_fixpoint(cx, d, w, tmp_path, keep):
    w.fixpoint()


def op_maintain(cx, d, w, tmp_path, keep):
    add = split(d, 5)[0]
    gone, new, _ = cx.datalog_maintain(w.rules, [2], add, 7)
    del w.segs[2]
    w.segs[7] = add
    w.inferred = (w.inferred - rows_set(rel_rows(gone))) | rows_set(rel_rows(new))


# op, whether the store is closed before it, whether it is closed after it
OPS = {
    "clear": (op_clear, True, False),
    "load": (op_load, True, False),
    "load_device": (op_load_device, True, False),
    "append": (op_append, True, False),
    "append_device": (op_append_device, True, False),
    "append_file": (op_append_file, True, False),
    "evict": (op_evict, True, False),
    "delete": (op_delete, True, False),
    "star_join_host": (op_star_join_host, True, False),
    "fixpoint": (op_fixpoint, False, True),
    "maintain": (op_maintain, True, True),
}


@pytest.mark.parametrize("name", sorted(OPS))
def test_mutation_voids_version_keyed_state(ctx, tmp_path, name):
    op, closed_before, closed_after = OPS[name]
    d, w, plan = setup(ctx, closed_before)
    assert w.closed() == closed_before
    keep = []
    op(ctx, d, w, tmp_path, keep)
    with pytest.raises(c.KolibrieError) as e:
        plan.submit()
    assert e.value.status == c.KB_E_INVALID and "stale" in e.value.message
    plan.free()
    assert w.closed() == closed_after, name
    w.check(name)


@pytest.mark.parametrize("entry", ["kb_store_load", "kb_store_load_device"])
def test_rejected_load_voids_the_closed_token(ctx, entry):
    """NULL columns with n > 0 are rejected; the load has emptied the store first, so the store is no longer the closed one"""
    d = employees()
    w = Window(ctx, d)
    for tag, rows in enumerate(split(d, 3), start=1):
        w.append(tag, rows)
    w.fixpoint()
    assert w.closed()
    rc = getattr(c.lib(), entry)(ctx.h, None, None, None, 4)
    assert rc == c.KB_E_INVALID
    assert not w.closed()
    w.segs, w.inferred = {}, set()
    w.check(entry)
