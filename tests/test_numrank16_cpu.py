"""CPU: the 16-bit rank columns of the store index (kolibrie_b200/csrc/kb_numrank.cuh: rank_shift, rank16, range16), built on the host
with g++. tests/cpp/numrank16_driver.cpp checks, for value orders of 1 to 2^31 - 1 values and random rank ranges, that a stored rank
strictly inside the stored range is always in the rank range, one outside it never is, and that the stored range is exact while the
value order has at most 65535 values."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kolibrie_b200", "csrc")


def test_stored_rank_range(tmp_path):
    exe = os.path.join(str(tmp_path), "numrank16_driver")
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", CSRC, "-o", exe, os.path.join(ROOT, "tests", "cpp", "numrank16_driver.cpp")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    for seed in (1, 2):
        r = subprocess.run([exe, str(seed)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-4000:]
        assert int(r.stdout.split()[1]) > 1_000_000, r.stdout
