"""CPU: the store model of tests/store_sequences.py against tests/update_reference.py and hand-worked cases, the generator's determinism,
and the events the GPU sequences reach (computed from the model alone)."""
import numpy as np
import pytest

from tests import store_sequences as S
from tests.update_reference import batch_insert, batch_remove


def seg(*rows):
    return np.array(rows, np.uint32).reshape(-1, 3)


def bag(model):
    return sorted(map(tuple, model.rows().tolist()))


@pytest.mark.parametrize("seed", range(6))
def test_model_set_writes_equal_the_restatement(seed):
    rng = np.random.default_rng(seed)

    def batch(n):
        return [tuple(int(x) for x in t) for t in rng.integers(0, [6, 3, 6], (n, 3))]

    m = S.Model("rank16")
    m.append(1, seg(*batch(30)))
    m.append(2, seg(*batch(30)))
    ref = S.as_set(m.rows())
    for step in range(40):
        b = batch(int(rng.integers(1, 12)))
        k = step % 4
        if k == 0:
            assert m.insert(int(rng.integers(0, 3)), seg(*b)) == batch_insert(ref, b)
        elif k == 1:
            assert m.remove(seg(*b)) == batch_remove(ref, b)
        elif k == 2:  # set-difference by value
            m.delete(seg(*b))
            ref -= set(b)
        else:  # the template (x M y), (x F v) filled row by row, then one remove batch
            rel = rng.integers(0, 6, (3, 3)).astype(np.uint32)
            filled = [(int(x), S.M, int(y)) for x, y, _ in rel] + [(int(x), S.F, int(v)) for x, _, v in rel]
            n_ref = sum(batch_remove(ref, filled))
            assert m.remove_template(rel) == n_ref
        assert S.as_set(m.rows()) == ref, step


def test_hand_worked_bag_cases():
    t, u, w = (1, 2, 3), (4, 5, 6), (7, 8, 9)
    m = S.Model("rank16")
    m.append(1, seg(t, u))
    m.append(2, seg(t, w))                   # t held by two tags
    assert m.remove(seg(t, t)) == [True, False]  # every stored copy goes, once flagged
    assert bag(m) == [u, w]
    m = S.Model("rank16")
    m.append(1, seg(t, u))
    m.append(2, seg(t, w))
    m.delete(seg(t))
    assert bag(m) == [u, w] and m.tags() == [1, 2]
    m.delete(seg(w))
    assert m.tags() == [1, 2] and m.evict(2)   # delete keeps the emptied segment: its tag is still there
    m = S.Model("rank16")
    m.append(1, seg(t, u))
    m.append(2, seg(t, w))
    assert m.evict(1) and bag(m) == [t, w]   # the copy of the other tag stays
    assert not m.evict(1)                    # absent tag: KB_E_NOT_FOUND, store unchanged
    assert m.remove(seg(w)) == [True] and m.tags() == [2]
    assert m.remove(seg(t)) == [True] and m.tags() == []  # remove drops a segment it empties
    assert not m.evict(2)
    m.append(3, seg(u))
    assert m.insert(500, seg(u, w, w)) == [False, True, False] and bag(m) == [u, w]
    assert m.insert(500, seg(u)) == [False] and "noop_insert" in m.events
    m.append(3, seg(t))
    assert m.evict(3) and "multi_segment_evict" in m.events and bag(m) == [w]
    assert m.evict(500) and "evict_insert_tag" in m.events and bag(m) == []


def test_closure_and_maintain():
    m = S.Model("rank16")
    m.append(1, seg((10, S.F, S.VAL0), (10, S.C, 100), (10, S.C, 101), (11, S.C, 102)))
    m.append(2, seg((11, S.F, S.VAL0 + 1), (12, S.F, S.VAL0)))
    had, inf = m.fixpoint()
    assert not had and S.as_set(inf) == {(10, S.G, 100), (10, S.G, 101), (11, S.G, 102)}
    gone, new = m.maintain([2], 3, seg((12, S.C, 103)))
    assert gone == {(11, S.G, 102)} and new == set()  # 12 left with tag 2: its C fact finds no F
    assert S.as_set(m.rows()) == {(10, S.F, S.VAL0), (10, S.C, 100), (10, S.C, 101), (11, S.C, 102), (12, S.C, 103),
                                  (10, S.G, 100), (10, S.G, 101)}
    assert "maintain_slide" in m.events


def test_generator_is_deterministic():
    a, _ = S.generate(1, "maintained")
    b, _ = S.generate(1, "maintained")
    assert S.digest(a) == S.digest(b)
    assert S.digest(a) == DIGESTS[(1, "maintained")]
    assert S.digest(S.generate(2, "sharded")[0]) == DIGESTS[(2, "sharded")]


def test_sharded_subjects_are_shard_blocks():
    g = S.Gen(1, "sharded")
    ks = [0, 1, 1023, 1024, 5000]
    assert all(S.shard_of(g.subj(k)) == S.SHARD_RANK for k in ks)
    assert all(S.shard_of(g.subj(k, foreign=True)) != S.SHARD_RANK for k in ks)
    assert all(S.shard_of(g.subj(k) + S.IOFF) == S.SHARD_RANK for k in ks)


def test_sequences_reach_every_event():
    seen = set()
    for mode in S.MODES:
        for seed in S.SEEDS:
            seen |= S.events(seed, mode)
    assert set(S.EVENTS) <= seen, sorted(set(S.EVENTS) - seen)


DIGESTS = {
    (1, "maintained"): "7d6bfe68fa647c7609f1a5412e9219408cf4cf1a2f61848d8266afcb963d4759",
    (2, "sharded"): "10b9a7c654eeb834138d929f5c7bab5eb2601a5059f11a097008e8a8c8682c7b",
}
