"""CPU: the restatement of the RSP engine's multi-window emit path (tests/rsp_join_reference.py) — the join's algebra on rows with
missing variables, and the single-thread and coordinator emit rules on scripted sequences (Timeout with an injected clock)."""
import random
from collections import Counter

from tests import rsp_join_reference as J
from tests.r2s_reference import Relation2Stream


def bag(rows):
    return Counter(tuple(sorted(r.items())) for r in rows)


def random_rows(rng, n, vars_, p_missing=0.3, domain=3):
    return [{v: f"v{rng.randrange(domain)}" for v in vars_ if rng.random() > p_missing} for _ in range(n)]


def test_natural_join_semantics():
    left = [{"a": "1", "b": "2"}, {"a": "1"}, {"b": "3"}]
    right = [{"b": "2", "c": "x"}, {"c": "y"}]
    got = bag(J.natural_join(left, right))
    want = Counter({
        (("a", "1"), ("b", "2"), ("c", "x")): 2,  # rows 0 and 1 (an unbound b is compatible with any b)
        (("a", "1"), ("b", "2"), ("c", "y")): 1,  # row 0
        (("a", "1"), ("c", "y")): 1,              # row 1
        (("b", "3"), ("c", "y")): 1,              # row 2 (b=3 clashes with b=2)
    })
    assert got == want
    assert J.natural_join([], right) == [] and J.natural_join(left, []) == []  # rsp_engine.rs:688-690
    assert len(J.natural_join([{"a": "1"}] * 2, [{"z": "q"}] * 3)) == 6  # no shared variable: the cartesian product, bag


def test_join_is_commutative_and_associative_on_bags():
    rng = random.Random(7)
    for _ in range(60):
        a = random_rows(rng, rng.randrange(0, 7), ["x", "y", "z"])
        b = random_rows(rng, rng.randrange(0, 7), ["y", "z", "w"])
        d = random_rows(rng, rng.randrange(0, 7), ["x", "w", "u"])
        assert bag(J.natural_join(a, b)) == bag(J.natural_join(b, a))
        assert bag(J.natural_join(J.natural_join(a, b), d)) == bag(J.natural_join(a, J.natural_join(b, d)))
        assert bag(J.join_window_results({"A": a, "B": b, "D": d}, ["A", "B", "D"])) == bag(J.join_window_results({"A": a, "B": b, "D": d}, ["D", "A", "B"]))


def _emitter(log):
    def emit(last, ts):
        out = J.emit_results(last, None, Relation2Stream("RSTREAM"), ["A", "B"])
        log.append((ts, out))
        return out
    return emit


def test_single_thread_rules():
    A, B = [{"s1": "a0"}], [{"s2": "b0"}]
    for policy, want in (("wait", [5, 9]), ("timeout", [5, 9]), ("steal", [5, 7, 9])):
        log = []
        st = J.SingleThreadEmitter(["A", "B"], policy, _emitter(log))
        st.send("A", A, 3)
        assert st.process() is None  # only A: wait for B (rsp_engine.rs:586-592)
        assert st.process() is None  # nothing new (:567-569)
        st.send("B", B, 5)
        assert st.process() is not None  # both: emit at the largest timestamp drained
        st.send("A", A, 7)
        st.process()  # Steal reuses B's stale result, Wait / Timeout wait for B again
        st.send("B", B, 9)
        st.process()
        assert [ts for ts, _ in log] == want, policy
        assert all(rows == [(("s1", "a0"), ("s2", "b0"))] for _, rows in log)


def test_single_thread_only_one_window_never_emits():
    """rsp_engine_test.rs:355-371: with Wait, a window that never fires means no result"""
    log = []
    st = J.SingleThreadEmitter(["A", "B"], "wait", _emitter(log))
    for i in range(10):
        st.send("A", [{"s1": f"a{i}"}], i)
        st.process()
    assert log == []


def test_coordinator_rules():
    A, B = [{"s1": "a0"}], [{"s2": "b0"}]
    # Wait: an emit per completed cycle
    log = []
    co = J.Coordinator(["A", "B"], "wait", _emitter(log))
    co.receive([("A", A, 1)], 0.0)
    co.receive([("A", A, 2)], 0.1)
    assert log == []
    co.receive([("B", B, 3)], 0.2)
    assert [ts for ts, _ in log] == [3]
    co.receive([("A", A, 4), ("B", B, 6)], 0.3)  # a result and the one drained with it complete a cycle
    assert [ts for ts, _ in log] == [3, 6]
    # Steal: emits as soon as every window has some result, then restarts the cycle
    log = []
    co = J.Coordinator(["A", "B"], "steal", _emitter(log))
    co.receive([("A", A, 1)], 0.0)
    assert log == []  # B never fired: nothing to steal (rsp_engine_test.rs:309-323)
    co.receive([("B", B, 2)], 0.1)
    co.receive([("A", A, 3)], 0.2)
    co.receive([("A", A, 4)], 0.3)
    assert [ts for ts, _ in log] == [2, 3, 4]


def test_coordinator_timeout_with_injected_clock():
    A, B = [{"s1": "a0"}], [{"s2": "b0"}]
    for fallback, want in (("steal", [2, 5]), ("drop", [2])):
        log = []
        co = J.Coordinator(["A", "B"], ("timeout", 1.0, fallback), _emitter(log))
        co.receive([("A", A, 1)], 0.0)
        co.receive([("B", B, 2)], 0.5)  # inside the deadline: a complete cycle
        co.receive([("A", A, 5)], 1.0)  # a new cycle starts at 1.0
        co.tick(1.5)
        assert [ts for ts, _ in log] == [2]  # deadline not reached
        co.tick(2.0)  # reached: Steal emits with B's stale result, Drop discards the cycle
        assert [ts for ts, _ in log] == want, fallback
        assert co.cycle_start is None and not co.cycle_triggered and co.max_ts == 0
        co.tick(10.0)
        assert [ts for ts, _ in log] == want  # nothing pending: no second emit
    # rsp_engine_test.rs:374-420: only A ever fires -> no result under either fallback
    for fallback in ("steal", "drop"):
        log = []
        co = J.Coordinator(["A", "B"], ("timeout", 0.2, fallback), _emitter(log))
        for i in range(5):
            co.receive([("A", [{"s1": f"a{i}"}], i)], 0.3 * i)
        co.tick(5.0)
        assert log == []


def test_emit_with_static_data_and_r2s():
    """rsp_engine_test.rs:572-646 shape: a window joined with static data on a shared variable; ISTREAM emits only new rows"""
    r2s = Relation2Stream("ISTREAM")
    static = [{"sensor": "s0", "room": "r1"}]
    w1 = {"W": [{"sensor": "s0"}, {"sensor": "s1"}]}
    assert J.emit_results(w1, static, r2s) == [(("room", "r1"), ("sensor", "s0"))]
    assert J.emit_results(w1, static, r2s) == []  # same answer: nothing new
    assert J.emit_results({"W": [{"sensor": "s2"}]}, static, r2s) == []  # no compatible static row
    assert J.emit_results({"W": [{}]}, static, r2s) == [(("room", "r1"), ("sensor", "s0"))]  # an empty row is compatible with all


def fixture_cases():
    from tests.rsp_multi_window_cases import CASES

    return CASES


def check_expect(case, rows):
    """the assertions of the reference test over every row it emitted (RSTREAM)"""
    e = case["expect"]
    if e.get("nonempty"):
        assert rows, case["name"]
    if e.get("no_rows"):
        assert not rows, case["name"]
    names = [dict(r) for r in rows]
    if "rows_bind" in e:
        assert any(all(v in r for v in e["rows_bind"]) for r in names), case["name"]
    if "only" in e:
        assert all(r[k] == v for r in names if all(k in r for k in e["only"]) for k, v in e["only"].items()), case["name"]
    if "n_rows" in e:
        assert len(rows) == e["n_rows"], case["name"]
        for k, vals in e["values"].items():
            assert sorted(r[k] for r in names) == vals, case["name"]


def test_restatement_meets_the_reference_tests_assertions():
    for case in fixture_cases():
        emits = J.replay_case(case, "RSTREAM", Relation2Stream)
        check_expect(case, [r for em in emits for r in em])
