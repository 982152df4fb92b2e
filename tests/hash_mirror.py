"""Bit-exact Python mirrors of the device's hash functions, and constructors of keys that collide in a chosen way.

Every open-addressing table on the device probes linearly from `hash & mask`, and every hash below is a fixed composition of mix32
(the murmur3 finaliser, a bijection on u32), 64-bit multiply-xorshift finalisers and FNV-1a. So a test can pick keys that share a
home slot, a home slot at the end of the table (the probe chain wraps to slot 0), or a stored 32-bit tag, instead of hoping random
data reaches those branches. Each mirror names the source it restates; tests/test_hash_mirror_cpu.py proves that every constructed
set has the property it claims.

All functions take and return numpy arrays (u32 or u64) or Python ints; arithmetic wraps like the device's.
"""
from __future__ import annotations

import functools

import numpy as np

NONE = 0xFFFFFFFF  # KB_ID_NONE == EMPTY32
QBIT = 0x80000000  # quoted-triple ids carry bit 31

U32 = np.uint32
U64 = np.uint64


def _wraps(f):
    """numpy warns when a scalar (not an array) product wraps; on the device wrapping is the point"""
    @functools.wraps(f)
    def g(*a, **k):
        with np.errstate(over="ignore"):
            return f(*a, **k)
    return g


def _u32(x):
    return np.asarray(x, dtype=np.uint64).astype(np.uint32) if not isinstance(x, np.ndarray) else x.astype(np.uint32)


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


# ---- the hashes

@_wraps
def mix32(x):
    """kb_device.cuh:32-35 (murmur3 fmix32)"""
    x = _u32(x).copy()
    x ^= x >> U32(16)
    x *= U32(0x85EBCA6B)
    x ^= x >> U32(13)
    x *= U32(0xC2B2AE35)
    x ^= x >> U32(16)
    return x


@_wraps
def mix32_inv(x):
    """the inverse of mix32: undo each step in reverse order (0x7ed1b41d and 0xa5cb9243 are the inverses of its multipliers mod 2^32)"""
    x = _u32(x).copy()
    x ^= x >> U32(16)
    x *= U32(0x7ED1B41D)
    x ^= (x >> U32(13)) ^ (x >> U32(26))
    x *= U32(0xA5CB9243)
    x ^= x >> U32(16)
    return x


FNV_OFFSET = 0xCBF29CE484222325
FNV_PRIME = 0x100000001B3


def fnv1a64_core(data: bytes) -> int:
    """64-bit FNV-1a before the fold (kb_dict.cu:26-27)"""
    h = FNV_OFFSET
    for b in data:
        h = ((h ^ b) * FNV_PRIME) & 0xFFFFFFFFFFFFFFFF
    return h


@_wraps
def fnv_fold(h):
    """kb_dict.cu:28-30: the fold that mixes FNV's weak low bits"""
    h = _u64(h).copy()
    h ^= h >> U64(32)
    h *= U64(0xD6E8FEB86659FD93)
    h ^= h >> U64(32)
    return h


def fnv1a64_folded(data) -> int:
    """fnv1a64 of kb_dict.cu:25-32, the hash of the dictionary's batch table and persistent index"""
    if isinstance(data, str):
        data = data.encode("utf-8")
    return int(fnv_fold(fnv1a64_core(data)))


@_wraps
def fnv1a64_folded_rows(prefix: bytes, rows: np.ndarray) -> np.ndarray:
    """fnv1a64_folded(prefix + bytes(row)) for every row of a u8 matrix, vectorised"""
    h = np.full(len(rows), fnv1a64_core(prefix), dtype=np.uint64)
    for j in range(rows.shape[1]):
        h ^= rows[:, j].astype(np.uint64)
        h *= U64(FNV_PRIME)
    return fnv_fold(h)


@_wraps
def triple_hash(s, p, o):
    """kb_quoted.cu:124-133, the hash of the quoted-triple batch table and reverse index (u64)"""
    s, p, o = _u64(s), _u64(p), _u64(o)
    h = ((s << U64(32)) | p) * U64(0x9E3779B97F4A7C15)
    h ^= o * U64(0xC2B2AE3D27D4EB4F)
    h ^= h >> U64(31)
    h *= U64(0xFF51AFD7ED558CCD)
    h ^= h >> U64(33)
    h *= U64(0xC4CEB9FE1A85EC53)
    h ^= h >> U64(33)
    return h


def tag(h):
    """the 32 bits a tag table keeps of a 64-bit hash (kb_tagtab.cuh:11)"""
    return _u64(h) >> U64(32)


def tag_home(h, slots: int):
    """the slot a tag table's probe starts at (kb_tagtab.cuh:16, 30)"""
    return _u64(h) & U64(slots - 1)


GROUP_SMEM = 64  # kb_group.cu:28, and PI_GROUP_SMEM (kb_join.cu:455)


def group1_cta_home(key):
    """group1_kernel's CTA-table home (kb_group.cu:268); the index probe's fused GROUP BY uses the same (kb_join.cu:682)"""
    return mix32(key) & U32(GROUP_SMEM - 1)


@_wraps
def group_kernel_hash(cols):
    """group_kernel's in-warp match value of a 1-4 column key (kb_group.cu:145): h = 0; h = mix32(h ^ k[c]) + c"""
    h = np.zeros(len(np.atleast_1d(cols[0])), dtype=np.uint32)
    for c, k in enumerate(cols):
        h = mix32(h ^ _u32(k)) + U32(c)
    return h


def group_kernel_cta_home(cols):
    """kb_group.cu:178"""
    return mix32(group_kernel_hash(cols)) & U32(GROUP_SMEM - 1)


GROUP_SEED, GROUP_MUL = 0x9E3779B9, 0x85EBCA77


@_wraps
def group_slot_hash(cols):
    """the global group table's hash before the mask (kb_group.cuh:29-32)"""
    h = np.full(len(np.atleast_1d(cols[0])), GROUP_SEED, dtype=np.uint32)
    for c, k in enumerate(cols):
        h = mix32(h ^ _u32(k)) * U32(GROUP_MUL) + U32(c)
    return mix32(h)


def group_slot_home(cols, n_slots: int):
    """kb_group.cuh:28-32"""
    return group_slot_hash(cols) & U32(n_slots - 1)


def distinct_home(v, n_slots: int):
    """distinct_kernel's home slot (kb_store.cu:36)"""
    return mix32(v) & U32(n_slots - 1)


SET_S, SET_O, SET_P = 0x9E3779B1, 0x632BE5AB, 0x85EBCA77


@_wraps
def set_hash(s, p, o):
    """the 96-bit key set's hash (kb_kernels.cuh:149): the store's INSERT / DELETE batch sets"""
    return mix32(mix32(s) * U32(SET_S) ^ mix32(_u32(o) + U32(SET_O)) ^ (_u32(p) * U32(SET_P)))


@_wraps
def set64_hash(s, o):
    """the 64-bit (s, o) set's hash before the mask (kb_kernels.cuh:195, 213)"""
    return mix32(mix32(s) * U32(SET_S) ^ mix32(_u32(o) + U32(SET_O)))


def set64_home(n_slots: int, s, o):
    """kb_datalog.cu:197"""
    return set64_hash(s, o) & U32(n_slots - 1)


# ---- table sizes, as the host sizes them

def tag_batch_slots(n: int) -> int:
    """tag_batch_table (kb_api.cu:67-74): a power of two >= 2n, 1024 at least"""
    s = 1024
    while s < 2 * n:
        s <<= 1
    return s


def tag_index_slots(n_keys: int, extra: int, current: int = 0) -> int:
    """tag_index_ensure (kb_internal.hpp:532-542): the index is kept while it has need = (n + extra) * 2 + 64 slots, else rebuilt with
    1.5x headroom, 1024 slots at least"""
    need = (n_keys + extra) * 2 + 64
    if current >= need:
        return current
    s = 1024
    while s < need + need // 2:
        s <<= 1
    return s


GROUP_FIRST_SLOTS = 1 << 12  # kb_group_aggregate's first global table (kb_group.cu:448), then 16x per overflow (:460)


def group_table_slots(attempt: int) -> int:
    return min(GROUP_FIRST_SLOTS * 16 ** attempt, 1 << 30)


CODE_SET_SLOTS = 512  # build_subject_codes' distinct set (kb_store.cu)
CODE_MAX = 255        # objects a coded subject table may hold


# ---- constructors

def _pick(cands: np.ndarray, n: int, ok: np.ndarray, what: str) -> np.ndarray:
    cands = cands[ok]
    _, first = np.unique(cands, return_index=True)
    cands = cands[np.sort(first)]
    assert len(cands) >= n, f"{what}: {len(cands)} candidates for {n}"
    return cands[:n].astype(np.uint32)


def _targets(rng, n: int, low_bits: int, low: int) -> np.ndarray:
    """4n distinct u32 whose low `low_bits` bits are `low`"""
    hi = rng.choice(1 << (32 - low_bits), size=min(4 * n, 1 << (32 - low_bits)), replace=False).astype(np.uint64)
    return ((hi << U64(low_bits)) | U64(low)).astype(np.uint32)


def _ids_ok(x: np.ndarray) -> np.ndarray:
    """plain dictionary ids: below bit 31 (quoted-triple ids) and so never KB_ID_NONE"""
    return x < U32(QBIT)


@_wraps
def keys_with_mix32_low(n: int, low_bits: int, low: int, seed: int = 1) -> np.ndarray:
    """n distinct ids k (below bit 31) with mix32(k) & (2^low_bits - 1) == low: the home `low` in every table of up to 2^low_bits
    slots that is indexed by mix32 (group1_kernel and the probe's CTA tables, distinct_kernel's set)"""
    rng = np.random.default_rng(seed)
    k = mix32_inv(_targets(rng, n, low_bits, low))
    return _pick(k, n, _ids_ok(k), "keys_with_mix32_low")


@_wraps
def group_slot_keys(n: int, low_bits: int = 16, low: int = 0xFFFF, seed: int = 2) -> np.ndarray:
    """n distinct one-column keys with group_slot_hash & (2^low_bits - 1) == low. The default puts every key at the last slot of
    every global group table up to 65536 slots: 4095 of the first, 65535 of the 16x retry."""
    rng = np.random.default_rng(seed)
    h = mix32_inv(_targets(rng, n, low_bits, low)) * U32(pow(GROUP_MUL, -1, 1 << 32))  # = mix32(GROUP_SEED ^ k)
    k = mix32_inv(h) ^ U32(GROUP_SEED)
    return _pick(k, n, _ids_ok(k), "group_slot_keys")


@_wraps
def group_slot_second_cols(k0: int, n: int, low_bits: int = 16, low: int = 0xFFFF, seed: int = 3) -> np.ndarray:
    """n distinct k1 such that every two-column key (k0, k1) has group_slot_hash & (2^low_bits - 1) == low: different groups that
    share their first column and their home slot"""
    rng = np.random.default_rng(seed)
    h1 = mix32(np.array([GROUP_SEED ^ k0], dtype=np.uint32)) * U32(GROUP_MUL)
    inner = (mix32_inv(_targets(rng, n, low_bits, low)) - U32(1)) * U32(pow(GROUP_MUL, -1, 1 << 32))  # = mix32(h1 ^ k1)
    k1 = mix32_inv(inner) ^ h1
    return _pick(k1, n, _ids_ok(k1), "group_slot_second_cols")


@_wraps
def group_kernel_twin(k0: int, k1: int, k0b: int) -> int:
    """the k1' with group_kernel_hash((k0, k1)) == group_kernel_hash((k0', k1')): mix32(k0) ^ k1 == mix32(k0') ^ k1'"""
    return int(mix32(np.array([k0], np.uint32))[0] ^ U32(k1) ^ mix32(np.array([k0b], np.uint32))[0])


@_wraps
def objects_for_set_hash(s: int, p: int, n: int, low_bits: int = 16, low: int = 0xFFFF, seed: int = 4) -> np.ndarray:
    """n distinct objects o (below bit 31) with set_hash(s, p, o) & (2^low_bits - 1) == low"""
    rng = np.random.default_rng(seed)
    y = mix32_inv(_targets(rng, n, low_bits, low)) ^ (mix32(np.array([s], np.uint32)) * U32(SET_S)) ^ (U32(p) * U32(SET_P))
    o = mix32_inv(y) - U32(SET_O)
    return _pick(o, n, _ids_ok(o), "objects_for_set_hash")


@_wraps
def objects_for_set64(s: int, n: int, low_bits: int = 16, low: int = 0xFFFF, seed: int = 5) -> np.ndarray:
    """n distinct objects o (below bit 31) with set64_hash(s, o) & (2^low_bits - 1) == low"""
    rng = np.random.default_rng(seed)
    y = mix32_inv(_targets(rng, n, low_bits, low)) ^ (mix32(np.array([s], np.uint32)) * U32(SET_S))
    o = mix32_inv(y) - U32(SET_O)
    return _pick(o, n, _ids_ok(o), "objects_for_set64")


# ---- tag collisions: seeded birthday searches

ALPHABET = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz012345", dtype=np.uint8)
STRING_PREFIX = b"http://example.org/h/"


def _twins(key: np.ndarray):
    """index pairs (i, j), i < j, of equal keys"""
    order = np.argsort(key, kind="stable")
    ks = key[order]
    d = np.flatnonzero(ks[1:] == ks[:-1])
    return [(int(min(order[x], order[x + 1])), int(max(order[x], order[x + 1]))) for x in d]


@functools.lru_cache(maxsize=None)
def tag_twin_strings(home_bits: int = 10, log2_n: int = 23, length: int = 10, seed: int = 11):
    """pairs of distinct strings whose folded FNV-1a hashes share the 32-bit tag and the low `home_bits` bits: the same tag and home
    slot in every tag table of up to 2^home_bits slots. A birthday search over 2^log2_n random strings of STRING_PREFIX + `length`
    characters; returns a tuple of (str, str) in the order found."""
    rng = np.random.default_rng(seed)
    rows = ALPHABET[rng.integers(0, len(ALPHABET), size=(1 << log2_n, length), dtype=np.uint8)]
    h = fnv1a64_folded_rows(STRING_PREFIX, rows)
    key = (tag(h) << U64(home_bits)) | tag_home(h, 1 << home_bits)
    out = []
    for i, j in _twins(key):
        a, b = (STRING_PREFIX + rows[x].tobytes() for x in (i, j))
        if a != b:
            out.append((a.decode(), b.decode()))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def home_strings(n: int, slots: int, home: int, length: int = 10, seed: int = 12):
    """n distinct strings whose folded FNV-1a hashes have home `home` in a tag table of `slots` slots"""
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    while len(out) < n:
        rows = ALPHABET[rng.integers(0, len(ALPHABET), size=(1 << 20, length), dtype=np.uint8)]
        h = fnv1a64_folded_rows(STRING_PREFIX, rows)
        for x in np.flatnonzero(tag_home(h, slots) == U64(home)).tolist():
            t = (STRING_PREFIX + rows[x].tobytes()).decode()
            if t not in seen:
                seen.add(t)
                out.append(t)
    return tuple(out[:n])


@functools.lru_cache(maxsize=None)
def tag_twin_triples(home_bits: int = 10, log2_n: int = 23, comp_bits: int = 12, seed: int = 13):
    """pairs of distinct (s, p, o) triples, components below 2^comp_bits (p below 2^4), whose triple_hash shares the tag and the low
    `home_bits` bits; a birthday search over 2^log2_n random triples"""
    rng = np.random.default_rng(seed)
    n = 1 << log2_n
    s = rng.integers(0, 1 << comp_bits, n, dtype=np.uint64)
    p = rng.integers(0, 16, n, dtype=np.uint64)
    o = rng.integers(0, 1 << comp_bits, n, dtype=np.uint64)
    h = triple_hash(s, p, o)
    key = (tag(h) << U64(home_bits)) | tag_home(h, 1 << home_bits)
    out = []
    for i, j in _twins(key):
        a, b = (int(s[i]), int(p[i]), int(o[i])), (int(s[j]), int(p[j]), int(o[j]))
        if a != b:
            out.append((a, b))
    return tuple(out)
