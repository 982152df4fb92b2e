"""GPU (-m gpu): builds tests/cpp/fc_tests.cpp against the C++ host mirror + libkolibrie_b200.so and runs it.
The CPU half (-m "not gpu") only checks that the host mirror compiles and links against the C ABI. The executable goes to a
temporary directory: the repository tree may be read-only where the suite runs."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "fc_tests.cpp")
LIBDIR = os.path.join(ROOT, "kolibrie_b200")


def build(out_dir):
    exe = os.path.join(str(out_dir), "fc_tests")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", exe, SRC, f"-L{LIBDIR}", "-lkolibrie_b200", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_cpp_host_mirror_compiles_and_links(tmp_path):
    build(tmp_path)


@pytest.mark.gpu
def test_cpp_fc_tests_pass_on_device(tmp_path):
    exe = build(tmp_path)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    assert "0 failed" in r.stdout
