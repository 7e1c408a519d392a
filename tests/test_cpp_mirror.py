"""The C++ host mirror (include/jvector_b200.hpp) compiles against the C ABI and behaves like the reference's provider:
on a box without an sm_90 device it fails loudly (no CPU fallback); on the GPU box it matches the oracle."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp):
    from jvector_b200 import _native as nat
    import oracle_lib
    oracle_lib.load()
    exe = os.path.join(str(tmp), "host_mirror_test")
    cmd = ["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle"),
           os.path.join(ROOT, "tests", "cpp", "host_mirror_test.cpp"), "-o", exe, nat.SO, os.path.join(ROOT, "oracle", "libjv_oracle.so"),
           "-Wl,-rpath," + os.path.dirname(nat.SO), "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-lpthread", "-ldl"]
    subprocess.check_call(cmd)
    return exe


def test_cpp_mirror_compiles_and_fails_loudly_without_gpu(tmp_path):
    from jvector_b200 import _native as nat
    exe = _build(tmp_path)
    if nat.load().jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present: covered by the gpu test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "NO_DEVICE_OK" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_mirror_parity_on_gpu(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "PARITY_OK" in out.stdout, out.stdout + out.stderr
