"""Builds and runs the C++ test of variational integrators (tests/cpp/test_variational.cpp) against the in-tree
library."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_variational")


def _build():
    src = os.path.join(ROOT, "tests", "cpp", "test_variational.cpp")
    lib = os.path.join(ROOT, "heyoka_b200", "lib")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(
            os.path.join(lib, "libheyoka_b200.so"))):
        subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), src, "-o", EXE, "-L" + lib,
                        "-lheyoka_b200", "-Wl,-rpath," + lib], check=True)
    return EXE


def test_cpp_variational_symbolic():
    res = subprocess.run([_build(), "cpu"], capture_output=True, text=True)
    assert res.returncode == 0 and "ALL PASSED (cpu)" in res.stdout, res.stdout + res.stderr


@pytest.mark.gpu
def test_cpp_variational_integrator():
    res = subprocess.run([_build(), "gpu"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ALL PASSED (gpu)" in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
