"""C++ host mirror (include/vmb200.hpp): compiles and links against libvmb200.so on CPU; runs its reference-KAT program on
the GPU box (-m gpu).  The program is linked into the test's temporary directory: the source tree may be read-only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    exe = os.path.join(str(out_dir), "host_mirror_test")
    libdir = os.path.join(ROOT, "victoriametrics_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "host_mirror_test.cpp"), "-L" + libdir, "-l:libvmb200.so",
           "-Wl,-rpath," + libdir, "-o", exe]
    subprocess.check_call(cmd)
    return exe


def test_cpp_host_mirror_compiles_and_links(tmp_path):
    exe = _build(tmp_path)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_cpp_host_mirror_reference_kats_on_gpu(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host_mirror_test: OK" in r.stdout
