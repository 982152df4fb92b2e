"""CPU: the value order behind the table-mode index probe's FILTER (kolibrie_b200/csrc/kb_numrank.cuh), built on the host with g++.
A FILTER(?o <cmp> c) over num_of(o) becomes a range of ranks in V (the sorted distinct non-NaN values of the numeric side table, -0.0
folded, 0.0 included); tests/cpp/numrank_driver.cpp fuzzes that range against the direct double comparison on tables and constants
drawn from signed zeros, infinities, NaNs, subnormals, nextafter neighbours, values beyond both ends and random bit patterns, and checks
that V built through order keys (the device's route) equals V built by a plain sort."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kolibrie_b200", "csrc")


def build_driver(out_dir):
    """builds tests/cpp/numrank_driver.cpp into out_dir (the repository tree may be read-only)"""
    exe = os.path.join(str(out_dir), "numrank_driver")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", CSRC, "-o", exe, os.path.join(ROOT, "tests", "cpp", "numrank_driver.cpp")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_rank_range_matches_direct_comparison(tmp_path):
    exe = build_driver(tmp_path)
    for seed in (1, 2, 3):
        r = subprocess.run([exe, str(seed), "100"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-4000:]
        checks = int(r.stdout.split()[1])
        assert checks > 1_000_000, r.stdout
