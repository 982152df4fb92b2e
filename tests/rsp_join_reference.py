"""A Python restatement of the RSP engine's multi-window emit path (kolibrie/src/rsp_engine.rs): natural_join, join_window_results,
emit_results and the two emit rules around them, transcribed line by line over rows that are dicts of strings (variable name -> value,
an unbound variable is simply absent). This is what kb_natural_join and engine.WindowJoin are compared with.

The reference's R2S operator takes each row as its `(name, value)` pairs sorted by name (rsp_engine.rs:668-675); `r2s` here is any
object with `eval(rows) -> rows` over such tuples (tests/r2s_reference.py's Relation2Stream)."""
from typing import Callable, Dict, List, Optional, Sequence

Row = Dict[str, str]


def natural_join(left: Sequence[Row], right: Sequence[Row]) -> List[Row]:
    """rsp_engine.rs:684-718"""
    if not left or not right:  # :688-690
        return []
    result = []
    for left_binding in left:  # :694
        for right_binding in right:  # :695
            compatible = True  # :697-705: every variable of the left row that the right row binds must agree
            for var, val in left_binding.items():
                if var in right_binding and right_binding[var] != val:
                    compatible = False
                    break
            if compatible:  # :707-713: the right values overwrite
                merged = dict(left_binding)
                merged.update(right_binding)
                result.append(merged)
    return result


def join_window_results(window_buffers: Dict[str, List[Row]], order: Optional[Sequence[str]] = None) -> List[Row]:
    """rsp_engine.rs:721-739. The reference folds in HashMap order; the join is commutative and associative on bags, so any fixed
    `order` gives the same bag."""
    if not window_buffers:  # :722-724
        return []
    all_windows = [window_buffers[k] for k in (order or list(window_buffers))]  # :726
    if len(all_windows) == 1:  # :728-730
        return list(all_windows[0])
    joined = all_windows.pop(0)  # :733
    for window_results in all_windows:  # :734-736
        joined = natural_join(joined, window_results)
    return joined


def emit_results(last_materialized: Dict[str, List[Row]], static_bindings: Optional[List[Row]], r2s, order: Optional[Sequence[str]] = None) -> list:
    """rsp_engine.rs:647-681: the emitted rows as sorted (name, value) tuples. static_bindings = the static plan's result, None when the
    query has no static plan (:659-665)"""
    joined = join_window_results(last_materialized, order)  # :657
    final_results = natural_join(joined, static_bindings) if static_bindings is not None else joined  # :659-665
    outputs = [tuple(sorted(b.items())) for b in final_results]  # :668-675
    return r2s.eval(outputs)  # :676


class SingleThreadEmitter:
    """process_single_thread_window_results (rsp_engine.rs:549-593): window results queue up (the channel) and are drained by the next
    call; an emit needs a result from every window; then Wait and Timeout clear the results, Steal keeps them (stale data is reused)."""

    def __init__(self, windows: Sequence[str], policy: str, emit: Callable[[Dict[str, List[Row]], int], object]):
        self.windows, self.policy, self.emit = list(windows), policy, emit
        self.pending: list = []  # the channel (:561)
        self.last_mat: Dict[str, List[Row]] = {}  # single_thread_last_materialized (:185)

    def send(self, window_iri: str, results: List[Row], ts: int):
        self.pending.append((window_iri, results, ts))

    def process(self):
        """returns what emit returned, or None when nothing was emitted"""
        had_new_results, max_ts = False, 0  # :559-560
        while self.pending:  # :561-565
            iri, results, ts = self.pending.pop(0)
            max_ts = max(max_ts, ts)
            self.last_mat[iri] = results
            had_new_results = True
        if not had_new_results:  # :567-569
            return None
        if len(self.last_mat) == len(self.windows):  # :572
            out = self.emit(self.last_mat, max_ts)  # :575
            if self.policy in ("wait", "timeout"):  # :580-582: no wall clock here, Timeout acts as Wait
                self.last_mat = {}
            return out  # :584 Steal keeps last_mat
        return None  # :586-592


class Coordinator:
    """start_cross_window_coordinator (rsp_engine.rs:387-508) without its thread: `receive` is one recv (:444-447, or :419-420 inside the
    deadline) followed by the try_recv drain (:469-473) of the results that arrived with it; `tick(now)` is the recv_timeout expiring
    (:421-440). The clock is the caller's: `now` in seconds. policy: "wait", "steal", ("timeout", duration, "steal" | "drop")."""

    def __init__(self, windows: Sequence[str], policy, emit: Callable[[Dict[str, List[Row]], int], object]):
        self.windows, self.policy, self.emit = list(windows), policy, emit
        self.last_materialized: Dict[str, List[Row]] = {}  # :401
        self.cycle_triggered: set = set()  # :403
        self.cycle_start: Optional[float] = None  # :405
        self.max_ts = 0  # :406
        self.emitted: list = []

    def _timeout(self):
        return self.policy if isinstance(self.policy, tuple) and self.policy[0] == "timeout" else None

    def _reset(self):
        self.cycle_triggered.clear()
        self.cycle_start = None
        self.max_ts = 0

    def tick(self, now: float):
        """the deadline elapsed without a result (:421-440)"""
        t = self._timeout()
        if t is None or self.cycle_start is None or now - self.cycle_start < t[1]:  # :410-415: no finite deadline, or not reached
            return
        if self.cycle_triggered:  # :423
            if t[2] == "steal" and len(self.last_materialized) == len(self.windows):  # :425-429
                self.emitted.append(self.emit(self.last_materialized, self.max_ts))
            self._reset()  # :435-437 (Drop discards the cycle, :430-432)

    def receive(self, batch: Sequence[tuple], now: float):
        """batch = [(window_iri, results, ts), ...]: the first is the recv, the rest the drain"""
        self.tick(now)  # a deadline that passed before this result arrived fires first
        iri, results, ts = batch[0]
        self.max_ts = max(self.max_ts, ts)  # :457
        self.last_materialized[iri] = results  # :459-462
        if not self.cycle_triggered:  # :463-465
            self.cycle_start = now
        self.cycle_triggered.add(iri)  # :466
        for iri, results, ts in batch[1:]:  # :469-473
            self.max_ts = max(self.max_ts, ts)
            self.last_materialized[iri] = results
            self.cycle_triggered.add(iri)
        if len(self.cycle_triggered) == len(self.windows):  # :475-480
            self.emitted.append(self.emit(self.last_materialized, self.max_ts))
            self._reset()
        elif self.policy == "steal":  # :483-491
            if len(self.last_materialized) == len(self.windows):
                self.emitted.append(self.emit(self.last_materialized, self.max_ts))
            self._reset()
        # :492-500 Wait / Timeout: keep waiting


def pattern_rows(store, pattern) -> List[Row]:
    """one triple pattern (strings, '?x' a variable) over a set of string triples: what a window plan of one TableScan returns"""
    rows = []
    for t in sorted(store):
        b: Row = {}
        if all((b.setdefault(q[1:], v) == v) if q.startswith("?") else q == v for q, v in zip(pattern, t)):
            rows.append(b)
    return rows


def replay_case(case, stream: str, r2s_factory) -> list:
    """a tests/rsp_multi_window_cases.py case through the restated emit path: every firing evicts its window's previous content from
    the ONE store the windows share, adds the new content and runs the window's pattern over the store (rsp_engine.rs:84-139); a drain
    (single thread) or each firing (coordinator) goes through the emit rule. Returns the emits, each a list of sorted (name, value)
    tuples."""
    r2s = r2s_factory(stream)
    static = pattern_rows({tuple(t) for t in case["static_triples"]}, case["static_pattern"]) if case["static_pattern"] else None
    order = [w["iri"] for w in case["windows"]]
    pattern = {w["iri"]: w["pattern"] for w in case["windows"]}
    emits: list = []
    emit = lambda last, ts: emits.append(emit_results(last, static, r2s, order))
    policy = case["policy"]
    rule = SingleThreadEmitter(order, policy, emit) if case["mode"] == "single_thread" else Coordinator(order, policy, emit)
    store, prev = set(), {w: [] for w in order}
    for step in case["steps"]:
        if step == "drain":
            rule.process()
            continue
        w = step["window"]
        store.difference_update(tuple(t) for t in prev[w])
        store.update(tuple(t) for t in step["content"])
        prev[w] = step["content"]
        results = pattern_rows(store, pattern[w])
        if case["mode"] == "single_thread":
            rule.send(w, results, step["ts"])
        else:
            rule.receive([(w, results, step["ts"])], 0.0)
    return emits
