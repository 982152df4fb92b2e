"""CPU: tests/hash_mirror.py — the Python mirrors of the device's hashes and the colliding key sets built from them. mix32 is checked
against the device header itself (kb_device.cuh's mix32 is __host__ __device__: tests/cpp/mix32_driver.cu runs it on the host), FNV-1a
against its published test vectors, mix32_inv against mix32, and every constructed set against the property it claims under the
mirrors, at the table sizes the host picks for the GPU tests of tests/test_gpu_hash_collisions.py."""
import os
import subprocess

import numpy as np
import pytest

from tests import hash_mirror as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def u32(x):
    return np.asarray(x, dtype=np.uint64).astype(np.uint32)


def test_mix32_inv_inverts_mix32():
    x = np.concatenate([u32([0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]),
                        np.random.default_rng(1).integers(0, 1 << 32, 200_000, dtype=np.uint64).astype(np.uint32)])
    assert np.array_equal(M.mix32_inv(M.mix32(x)), x)
    assert np.array_equal(M.mix32(M.mix32_inv(x)), x)
    assert int(M.mix32(u32([0]))[0]) == 0  # fmix32 fixes 0


def test_mix32_matches_the_device_header(tmp_path):
    """kb_device.cuh's mix32, compiled by nvcc and run on the host, equals the mirror"""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    exe = os.path.join(str(tmp_path), "mix32_driver")
    src = os.path.join(ROOT, "tests", "cpp", "mix32_driver.cu")
    r = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    x = np.concatenate([u32([0, 1, 63, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF]),
                        np.random.default_rng(2).integers(0, 1 << 32, 5000, dtype=np.uint64).astype(np.uint32)])
    r = subprocess.run([exe], input="".join(f"{v}\n" for v in x.tolist()), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=120)
    assert r.returncode == 0, r.stdout
    got = u32([int(t) for t in r.stdout.split()])
    assert np.array_equal(got, M.mix32(x))


def test_fnv1a64_published_vectors():
    """the core before the fold: the 64-bit FNV-1a test vectors of the reference implementation"""
    assert M.fnv1a64_core(b"") == 0xCBF29CE484222325
    assert M.fnv1a64_core(b"a") == 0xAF63DC4C8601EC8C
    assert M.fnv1a64_core(b"foobar") == 0x85944171F73967E8
    rows = np.frombuffer(b"foobar", dtype=np.uint8)[None, :]
    assert int(M.fnv1a64_folded_rows(b"", rows)[0]) == M.fnv1a64_folded("foobar") == int(M.fnv_fold(0x85944171F73967E8))
    assert int(M.fnv1a64_folded_rows(b"foo", rows[:, 3:])[0]) == M.fnv1a64_folded("foobar")


def test_triple_hash_finaliser_is_murmur3_fmix64():
    """triple_hash = fmix64(((s << 32 | p) * c1) ^ (o * c2)): fmix64(0) == 0, so (0, 0, 0) hashes to 0"""
    assert int(M.triple_hash(0, 0, 0)) == 0
    assert int(M.triple_hash(1, 2, 3)) != int(M.triple_hash(3, 2, 1))


def test_tag_table_sizes():
    assert [M.tag_batch_slots(n) for n in (0, 1, 512, 513, 1024, 1025)] == [1024, 1024, 1024, 2048, 2048, 4096]
    # a new index has 1.5x headroom: 1024 slots up to 309 keys, 2048 from 310; an index is kept until its keys need more than its slots
    assert M.tag_index_slots(300, 9) == 1024 and M.tag_index_slots(300, 10) == 2048
    assert M.tag_index_slots(300, 180, current=1024) == 1024 and M.tag_index_slots(300, 181, current=1024) == 2048
    assert [M.group_table_slots(a) for a in range(4)] == [4096, 65536, 1 << 20, 1 << 24]


def test_tag_twin_strings():
    """distinct strings, same 32-bit tag, same home in a 1024-slot table; some of them also in a 2048-slot table"""
    tw = M.tag_twin_strings()
    assert len(tw) >= 6
    wide = 0
    for a, b in tw:
        ha, hb = M.fnv1a64_folded(a), M.fnv1a64_folded(b)
        assert a != b and ha != hb
        assert ha >> 32 == hb >> 32 and ha & 1023 == hb & 1023
        wide += ha & 2047 == hb & 2047
    assert wide >= 3
    assert len({s for pair in tw for s in pair}) == 2 * len(tw)


def test_home_strings():
    hs = M.home_strings(12, 1024, 1023)
    assert len(set(hs)) == 12 and all(M.fnv1a64_folded(s) & 1023 == 1023 for s in hs)


def test_tag_twin_triples():
    tt = M.tag_twin_triples()
    assert len(tt) >= 4
    for a, b in tt:
        ha, hb = int(M.triple_hash(*a)), int(M.triple_hash(*b))
        assert a != b and ha != hb and ha >> 32 == hb >> 32 and ha & 1023 == hb & 1023
        assert all(x < 1 << 12 for x in a + b)
    assert len({t for pair in tt for t in pair}) == 2 * len(tt)


def test_mix32_keys_home_at_the_last_slot():
    k = M.keys_with_mix32_low(300, 9, 511)
    assert len(np.unique(k)) == 300 and (k < M.QBIT).all()
    assert (M.distinct_home(k, M.CODE_SET_SLOTS) == 511).all()
    assert (M.group1_cta_home(k) == 63).all()  # 511 & 63


def test_group_slot_keys():
    k = M.group_slot_keys(5000)
    assert len(np.unique(k)) == 5000 and (k < M.QBIT).all()
    for slots in (M.group_table_slots(0), M.group_table_slots(1)):
        assert (M.group_slot_home([k], slots) == slots - 1).all()
    k1 = M.group_slot_second_cols(77, 40)
    assert len(np.unique(k1)) == 40
    assert (M.group_slot_home([np.full(40, 77, np.uint32), k1], 4096) == 4095).all()


def test_group_kernel_twins():
    rng = np.random.default_rng(3)
    for _ in range(100):
        k0, k1, k0b = (int(x) for x in rng.integers(0, 1 << 31, 3))
        k1b = M.group_kernel_twin(k0, k1, k0b)
        a, b = [u32([k0]), u32([k1])], [u32([k0b]), u32([k1b])]
        assert (k0, k1) != (k0b, k1b)
        assert M.group_kernel_hash(a)[0] == M.group_kernel_hash(b)[0]
        assert M.group_kernel_cta_home(a)[0] == M.group_kernel_cta_home(b)[0]


def test_set_hash_objects():
    s, p = 123456, 77
    o = M.objects_for_set_hash(s, p, 200)
    assert len(np.unique(o)) == 200 and (o < M.QBIT).all()
    for slots in (1024, 4096, 65536):
        assert ((M.set_hash(np.full(200, s, np.uint32), np.full(200, p, np.uint32), o) & (slots - 1)) == slots - 1).all()


def test_set64_objects():
    s = 4242
    o = M.objects_for_set64(s, 200)
    assert len(np.unique(o)) == 200 and (o < M.QBIT).all()
    for slots in (1024, 2048, 65536):
        assert (M.set64_home(slots, np.full(200, s, np.uint32), o) == slots - 1).all()
