"""The C++ host mirror's impulsive targeting (nyxb::Targeter in include/nyxb.hpp) compiles against the
C ABI; on a GPU box its test program runs."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "cpp" / "test_target_mirror.cpp"
LIBDIR = ROOT / "nyx_b200" / "csrc"


def _build(tmp_path):
    exe = tmp_path / "test_target_mirror"
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-I", str(ROOT / "include"), str(SRC), "-o", str(exe), "-L", str(LIBDIR), "-lnyxb",
           f"-Wl,-rpath,{LIBDIR}"]
    subprocess.run(cmd, check=True, capture_output=True)
    return exe


def test_cpp_target_mirror_compiles_and_links(tmp_path):
    assert _build(tmp_path).exists()


@pytest.mark.gpu
def test_cpp_target_mirror_runs(tmp_path):
    out = subprocess.run([str(_build(tmp_path))], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "OK" in out.stdout, out.stdout + out.stderr
