"""Hand transcriptions of the INPUTS and ASSERTIONS of the reference's multi-window and static-data tests, in the manner of
tests/golden/make_fixtures.py, as the RSP engine's emit path sees them (rsp_engine.rs:387-508, 549-593, 647-741). The window
firings are computed by a transcription of CSPARQLWindow (below); the emitted rows themselves come from tests/rsp_join_reference.py.
tests/test_rsp_join_cpu.py holds the restatement to the `expect` assertions, tests/test_gpu_natural_join.py replays every case on
the device."""
import math

SOURCE = ("kolibrie/tests/rsp_engine_test.rs:198-232 (two-window engine), :340-570 (multi-window, joining, single-thread, static join), "
              ":572-646 (single window + static data), :648-760 (Steal / Wait / Timeout), :763-870 (two windows + static data), "
              ":872-933 (static data not visible to window queries)")

NOTE = ("Inputs of the reference's multi-window and static-data tests as the emit path sees them. `steps` is the engine's sequence: "
            "a firing (window, timestamp, the window's content, rsp_engine.rs:84-139) or \"drain\" (process_single_thread_window_results, "
            "called by every add_to_stream in single-thread mode and by stop, :512-517, :603-611). Firings are computed by the "
            "CSPARQLWindow transcription below (s2r.rs:173-286, OnWindowClose + TimeDriven); stop()'s flush reports every "
            "open window, here from the latest-opened to the earliest, where the reference iterates a HashMap; a drain keeps the last content a window sent, so this order keeps the earliest-opened window, the one holding the most events. Windows share one store: a firing "
            "evicts that window's previous content and adds the new one (:94-104), and the window's pattern runs over the whole store. "
            "In coordinator mode every firing is received on its own (no drain batches, no deadline). `expect` holds what the reference "
            "test asserts: nonempty = some emitted row (:400, :552, :633); no_rows = nothing emitted (:463, :658, :676, :704, :730, :754); "
            "rows_bind = an emitted row binds these variables (:628-636, :843-849); only = every row binding both has these values "
            "(:852-868); n_rows / values = exactly these rows (:917-923). Emitted rows themselves come from tests/rsp_join_reference.py.")

A_ = "http://www.w3.org/1999/02/22-rdf-syntax-ns#type"
W3T = "http://www.w3.org/test/"


def csparql_window(width, slide):
    """CSPARQLWindow::add_to_window with the default OnWindowClose report and TimeDriven tick (kolibrie/src/rsp/s2r.rs:173-265,
    query_builder.rs:33-34): add(item, ts) returns the content of the window that fires on this event (or None) and the content's
    last_timestamp_changed; flush() the content of every open window (s2r.rs:277-286)."""
    state = {"app_time": 0, "active": {}}  # (open, close) -> [items, last_ts]

    def add(item, ts):
        c_sup = math.ceil(abs(ts - 0) / slide) * slide  # s2r.rs:237-238 (t_0 = 0)
        o_i = c_sup - width  # :240
        while True:  # :247-264; `as usize` saturates a negative bound at 0
            w = (max(0, o_i), max(0, o_i + width))
            state["active"].setdefault(w, [[], 0])
            o_i += slide
            if o_i > ts:
                break
        fired = None
        due = [w for w in state["active"] if w[1] <= ts]  # :203-207 the report runs on the contents BEFORE this event is added
        if due:
            w = max(due, key=lambda w_: w_[1])
            if ts > state["app_time"]:  # :210-213
                state["app_time"] = ts
                fired = (list(state["active"][w][0]), state["active"][w][1])
        kept = {}
        for w, (items, last) in state["active"].items():  # :177-201: add to the windows that contain ts, drop the others
            if w[0] <= ts < w[1]:
                kept[w] = [items + ([item] if item not in items else []), ts]
        state["active"] = kept
        return fired

    def flush():
        return [(list(items), last) for w, (items, last) in sorted(state["active"].items(), reverse=True)]

    return add, flush


def rsp_steps(windows, events, single_thread):
    """what the engine does with `events` ([stream, triple, ts], rsp_engine.rs:511-547): in single-thread mode each add_to_stream first
    drains the results of earlier firings (:512-517); every window whose stream matches gets the event and may fire, a firing being
    (window, timestamp = the content's last change, content); stop() flushes every window (:603-611) and drains"""
    wins = {w["iri"]: csparql_window(w["range"], w["step"]) for w in windows}
    steps = []
    for stream, triple, ts in events:
        if single_thread:
            steps.append("drain")
        for w in windows:
            if w["stream"] in ("?", stream):
                fired = wins[w["iri"]][0](triple, ts)
                if fired is not None:
                    steps.append({"window": w["iri"], "ts": fired[1], "content": fired[0]})
    for w in windows:
        for content, last in wins[w["iri"]][1]():
            steps.append({"window": w["iri"], "ts": last, "content": content})
    if single_thread:
        steps.append("drain")
    return steps


def typed(stream, prefix, typ, ts_list, offset=0):
    return [[stream, [prefix.format(i), A_, typ], i + offset] for i in ts_list]


def two_window_case(name, line, policy, events):
    ws = [{"iri": "windA", "stream": "streamA", "range": 10, "step": 2, "pattern": ["?s1", A_, "http://test/TypeA"]},
          {"iri": "windB", "stream": "streamB", "range": 10, "step": 2, "pattern": ["?s2", A_, "http://test/TypeB"]}]
    return {"name": name, "line": line, "mode": "single_thread", "policy": policy, "windows": ws, "static_triples": [], "static_pattern": None,
            "steps": rsp_steps(ws, events, True), "expect": {"no_rows": True} if "no_emission" in name else {"nonempty": True}}


CASES = []
ws = [{"iri": "wind", "stream": "stream1", "range": 10, "step": 2, "pattern": ["?s", A_, W3T + "Temperature"]},
      {"iri": "wind2", "stream": "stream2", "range": 5, "step": 1, "pattern": ["?s2", A_, W3T + "CO2"]}]
ev = typed("stream1", "http://test.be/temp{}", W3T + "Temperature", range(10)) + typed("stream2", "http://test.be/co2{}", W3T + "CO2", range(10), 10)
CASES.append({"name": "multi_window", "line": 340, "mode": "coordinator", "policy": "wait", "windows": ws, "static_triples": [], "static_pattern": None,
           "steps": rsp_steps(ws, ev, False), "expect": {"nonempty": True}})
ws = [dict(ws[0]), dict(ws[1], pattern=["?s", A_, W3T + "CO2"])]
CASES.append({"name": "joining_multi_window", "line": 404, "mode": "coordinator", "policy": "wait", "windows": ws, "static_triples": [], "static_pattern": None,
           "steps": rsp_steps(ws, ev, False), "expect": {"no_rows": True}})
ws = [{"iri": "wind1", "stream": "stream1", "range": 10, "step": 2, "pattern": ["?s1", A_, W3T + "TypeOne"]},
      {"iri": "wind2", "stream": "stream2", "range": 5, "step": 1, "pattern": ["?s2", A_, W3T + "TypeTwo"]}]
ev = [e for i in range(5) for e in (typed("stream1", "http://test.be/one_{}", W3T + "TypeOne", [i]) + typed("stream2", "http://test.be/two_{}", W3T + "TypeTwo", [i], 10))]
CASES.append({"name": "single_thread_multi_window", "line": 468, "mode": "single_thread", "policy": "wait", "windows": ws, "static_triples": [],
           "static_pattern": None, "steps": rsp_steps(ws, ev, True), "expect": {"nonempty": True}})
ws = [{"iri": "wind", "stream": "stream1", "range": 10, "step": 2, "pattern": ["?sensor", A_, W3T + "Sensor"]}]
ev = typed("stream1", "http://test.be/sensor{}", W3T + "Sensor", range(5))
CASES.append({"name": "single_window_static_join", "line": 572, "mode": "single_thread", "policy": "wait", "windows": ws,
           "static_triples": [["http://test.be/sensor0", W3T + "locatedIn", "http://test.be/room1"]], "static_pattern": ["?sensor", W3T + "locatedIn", "?room"],
           "steps": rsp_steps(ws, ev, True), "expect": {"nonempty": True, "rows_bind": ["room", "sensor"]}})
evA = typed("streamA", "http://test/a{}", "http://test/TypeA", range(5))
evB = typed("streamB", "http://test/b{}", "http://test/TypeB", range(3))
CASES.append(two_window_case("steal_no_emission_before_b_fires", 648, "steal", evA))
CASES.append(two_window_case("steal_emits_with_stale", 666, "steal", evB + typed("streamA", "http://test/a{}", "http://test/TypeA", range(5), 20)))
CASES.append(two_window_case("wait_no_emission_when_only_a_fires", 693, "wait", evA))
CASES.append(two_window_case("timeout_steal_no_emission_when_only_a_fires", 712, "timeout", evA))
CASES.append(two_window_case("timeout_drop_no_emission_when_only_a_fires", 736, "timeout", evA))
ws = [{"iri": "wind1", "stream": "stream1", "range": 10, "step": 2, "pattern": ["?sensor", A_, W3T + "Sensor"]},
      {"iri": "wind2", "stream": "stream2", "range": 10, "step": 2, "pattern": ["?room", A_, W3T + "Room"]}]
ev = typed("stream1", "http://test.be/sensor{}", W3T + "Sensor", range(3)) + typed("stream2", "http://test.be/room{}", W3T + "Room", range(3), 10)
CASES.append({"name": "multi_window_static_join", "line": 763, "mode": "single_thread", "policy": "wait", "windows": ws,
           "static_triples": [["http://test.be/sensor0", W3T + "locatedIn", "http://test.be/room0"]], "static_pattern": ["?sensor", W3T + "locatedIn", "?room"],
           "steps": rsp_steps(ws, ev, True), "expect": {"nonempty": True, "rows_bind": ["room", "sensor"],
                                                        "only": {"sensor": "http://test.be/sensor0", "room": "http://test.be/room0"}}})
ws = [{"iri": "w", "stream": "?", "range": 10, "step": 10, "pattern": ["?s", A_, "http://example.org/Type"]}]
CASES.append({"name": "static_data_not_visible_in_window_query", "line": 872, "mode": "single_thread", "policy": "wait", "windows": ws,
           "static_triples": [["http://example.org/static1", A_, "http://example.org/Type"]], "static_pattern": None,
           "steps": rsp_steps(ws, [["any", ["http://example.org/stream1", A_, "http://example.org/Type"], 1]], True),
           "expect": {"n_rows": 1, "values": {"s": ["http://example.org/stream1"]}}})

