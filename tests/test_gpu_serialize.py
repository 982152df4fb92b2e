"""GPU: kb_serialize_begin / kb_serialize_next against the restatement of generate_ntriples / generate_turtle
(tests/serialize_reference.py), byte for byte: the hand-worked cases, seeded stores with repeated triples, the store after appends,
evictions and deletes (index built and not), ids at the edges of the u32 domain, every capacity from the largest unit up, the
refusals, and cfg2's 10 M-triple store by SHA-256."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import serialize_reference as R
from tests.serialize_cases import CASES, Q

pytestmark = pytest.mark.gpu

FORMATS = [(c.SER_NTRIPLES, "nt"), (c.SER_TURTLE, "ttl")]


@pytest.fixture(scope="module")
def ctx():
    """a context of this module's own: the tests here load dictionaries and quoted-triple tables (cycles included) that no other test
    should inherit"""
    x = c.Context(0)
    yield x
    x.close()


def load(ctx, strings, quoted, triples):
    t = np.array(list(triples), dtype=np.uint32).reshape(-1, 3)
    ctx.store_load(t[:, 0], t[:, 1], t[:, 2])
    ctx.dict_strings_load(strings)
    ids = np.array(list(quoted), dtype=np.uint32)
    comp = np.array(list(quoted.values()), dtype=np.uint32).reshape(-1, 3)
    ctx.quoted_load(ids, comp[:, 0], comp[:, 1], comp[:, 2])


def text(ctx, fmt, prefixes=(), capacity=1 << 40, info=None):
    return b"".join(ctx.serialize(fmt, prefixes, capacity, info)).decode("utf-8")


def restated(fmt, triples, strings, quoted, prefixes=()):
    if fmt == c.SER_NTRIPLES:
        return R.generate_ntriples(triples, strings, quoted)
    return R.generate_turtle(triples, strings, quoted, prefixes)


def store_triples(ctx):
    s, p, o = ctx.store_download()
    return list(zip(s.tolist(), p.tolist(), o.tolist()))


class Raw:
    """the three entry points without the generator, to see a refusal where it happens"""

    def __init__(self, ctx, fmt, prefixes=()):
        self.ctx, self.h, self.info = ctx, C.c_void_p(), c.KbSerializeInfo()
        enc = [x.encode() for pr in prefixes for x in pr]
        off = np.zeros(len(enc) + 1, np.uint64)
        off[1:] = np.cumsum([len(b) for b in enc])
        data = np.frombuffer(b"".join(enc) or b"\0", np.uint8)
        self.rc = c.lib().kb_serialize_begin(ctx.h, fmt, c._ptr(off), c._ptr(data), len(prefixes), C.byref(self.h), C.byref(self.info))

    def next(self, capacity):
        buf = np.empty(max(capacity, 1), np.uint8)
        got = C.c_uint64(0)
        rc = c.lib().kb_serialize_next(self.ctx.h, self.h, c._ptr(buf), capacity, C.byref(got))
        return rc, buf[: got.value].tobytes()

    def free(self):
        if self.rc == c.KB_OK:
            c.lib().kb_serialize_free(self.h)


@pytest.mark.parametrize("case", CASES, ids=lambda k: k["name"])
def test_hand_worked_cases(ctx, case):
    load(ctx, case["strings"], case["quoted"], case["triples"])
    for fmt, key in FORMATS:
        info = {}
        got = text(ctx, fmt, case["prefixes"], info=info)
        assert got == case[key]
        assert info["total_bytes"] == len(case[key].encode())
        assert info["n_triples"] == len(set(case["triples"]))


def seeded_store(seed, n):
    rng = random.Random(seed)
    words = ["http://x/" + w for w in ("a", "ab", "b", "é", "z", "zz")] + ["https://y/%d" % k for k in range(40)] + \
            ["lit%d" % k for k in range(60)] + ["", "<< a b c >>", "ü", "a b", "\"q\"", "x\ny"]
    quoted = {Q: (0, 1, 2), Q + 1: (Q, 3, 4), Q + 2: (0, 999, 2), Q + 3: (Q + 1, 0, Q), Q + 5: (7, 8, Q + 1)}
    pool = list(range(len(words))) + [5000, 5001] + list(quoted) + [Q + 4, Q + 77]
    trip = [tuple(rng.choice(pool) for _ in range(3)) for _ in range(n)]
    return words, quoted, trip + [trip[rng.randrange(n)] for _ in range(n // 5)]  # repeats inside the segment


@pytest.mark.parametrize("seed", range(3))
def test_seeded_stores_with_repeats_across_segments(ctx, seed):
    words, quoted, trip = seeded_store(seed, 3000)
    load(ctx, words, quoted, trip[:2000])
    more = np.array(trip[1500:] + trip[:300], dtype=np.uint32)  # repeats across segments
    ctx.store_append(more[:, 0], more[:, 1], more[:, 2], tag=7)
    held = store_triples(ctx)
    prefixes = [("x", "http://x/"), ("y", "https://y/")]
    for fmt, _ in FORMATS:
        assert text(ctx, fmt, prefixes) == restated(fmt, held, words, quoted, prefixes)


@pytest.mark.parametrize("indexed", [False, True], ids=["no_index", "index"])
def test_after_append_evict_delete(ctx, indexed):
    words, quoted, trip = seeded_store(11, 4000)
    load(ctx, words, quoted, trip[:1000])
    if indexed:
        ctx.build_index()
    for tag, part in ((1, trip[1000:2500]), (2, trip[2000:4000]), (3, trip[:500])):
        a = np.array(part, dtype=np.uint32)
        ctx.store_append(a[:, 0], a[:, 1], a[:, 2], tag)
    ctx.store_evict(2)
    d = np.array(trip[:200] + trip[1200:1300], dtype=np.uint32)
    ctx.store_delete(d[:, 0], d[:, 1], d[:, 2])
    held = store_triples(ctx)
    for fmt, _ in FORMATS:
        assert text(ctx, fmt) == restated(fmt, held, words, quoted)


def test_u32_edge_ids(ctx):
    """0, 0x7FFFFFFF (a plain id past the dictionary), 0x80000000 (quoted index 0), 0xFFFFFFFE (a quoted id no table can hold) and plain
    ids just past the dictionary"""
    words = ["http://x/zero", "http://x/p", "lit"]
    quoted = {Q: (0, 1, 0x7FFFFFFF), Q + 1: (0, 1, 2)}
    edge = [0, 1, 2, 3, 4, 0x7FFFFFFF, Q, Q + 1, 0xFFFFFFFE]
    trip = [(s, p, o) for s in edge for p in (1, 0x7FFFFFFF, Q + 1, 0xFFFFFFFE) for o in edge]
    load(ctx, words, quoted, trip)
    for fmt, _ in FORMATS:
        assert text(ctx, fmt) == restated(fmt, trip, words, quoted)


def test_every_capacity_from_the_largest_unit(ctx):
    words, quoted, trip = seeded_store(5, 2000)
    load(ctx, words, quoted, trip)
    held = store_triples(ctx)
    prefixes = [("x", "http://x/"), ("y", "https://y/")]
    for fmt, _ in FORMATS:
        info = {}
        want = restated(fmt, held, words, quoted, prefixes).encode()
        text(ctx, fmt, prefixes, info=info)
        m = info["max_unit_bytes"]
        for cap in (m, m + 1, 4096, 1 << 40):
            pieces = list(ctx.serialize(fmt, prefixes, cap))
            assert b"".join(pieces) == want, cap
            assert all(0 < len(x) <= cap for x in pieces)
            if fmt == c.SER_NTRIPLES:
                assert all(x.endswith(b"\n") for x in pieces)  # whole lines only
        if fmt == c.SER_NTRIPLES:
            assert len(list(ctx.serialize(fmt, prefixes, m))) > 1


def test_refusals_leave_the_store_as_it_was(ctx):
    words, quoted, trip = seeded_store(9, 500)
    load(ctx, words, quoted, trip)
    before = store_triples(ctx)
    want = restated(c.SER_NTRIPLES, before, words, quoted).encode()
    # a capacity below the largest unit: refused, nothing consumed
    r = Raw(ctx, c.SER_NTRIPLES)
    assert r.rc == c.KB_OK
    m = r.info.max_unit_bytes
    assert r.next(m - 1)[0] == c.KB_E_LIMIT
    out = []
    while True:
        rc, piece = r.next(m + 5)
        assert rc == c.KB_OK
        if not piece:
            break
        out.append(piece)
    assert b"".join(out) == want
    r.free()
    # the store changed between begin and next
    r = Raw(ctx, c.SER_TURTLE)
    a = np.array(trip[:3], dtype=np.uint32)
    ctx.store_append(a[:, 0], a[:, 1], a[:, 2], 99)
    assert r.next(1 << 20)[0] == c.KB_E_INVALID
    r.free()
    ctx.store_evict(99)
    # an unknown format
    r = Raw(ctx, 7)
    assert r.rc == c.KB_E_INVALID
    # quoted ids without a table
    ctx.quoted_load([], [], [], [])
    assert Raw(ctx, c.SER_NTRIPLES).rc == c.KB_E_UNSUPPORTED
    # a quoted-triple cycle: the walk passes KB_QUOTED_MAX_DEPTH
    ctx.quoted_load([Q, Q + 1, Q + 2, Q + 3, Q + 5], [Q, Q, 0, Q + 1, 7], [1, 3, 999, 0, 8], [2, 4, 2, Q, Q + 1])
    assert Raw(ctx, c.SER_TURTLE).rc == c.KB_E_LIMIT
    # no device dictionary strings
    ctx.dict_strings_load([])
    assert Raw(ctx, c.SER_NTRIPLES).rc == c.KB_E_UNSUPPORTED
    assert sorted(store_triples(ctx)) == sorted(before)


def employee_strings(d):
    """cfg2's dictionary as text: IRIs for the entities and predicates, plain literals for the salaries (every object class occurs)"""
    out = np.array(["http://example.org/t%d" % i for i in range(d.n_ids)], dtype=object)
    out[d.ids["F"]] = "F"
    k = np.nonzero(d.is_num)[0]
    out[k] = [str(int(v)) for v in d.num_or0[k]]
    return out.tolist()


def test_cfg2_10m_digest(ctx):
    d = datagen.employee_dataset(1_666_667)
    strings = employee_strings(d)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_strings_load(strings)
    ctx.quoted_load([], [], [], [])
    trip = list(zip(d.s.tolist(), d.p.tolist(), d.o.tolist()))
    for fmt, _ in FORMATS:
        h = hashlib.sha256()
        for piece in ctx.serialize(fmt, [("ex", "http://example.org/")], 64 << 20):
            h.update(piece)
        want = hashlib.sha256(restated(fmt, trip, strings, {}, [("ex", "http://example.org/")]).encode()).hexdigest()
        assert h.hexdigest() == want
