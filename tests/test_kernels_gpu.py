"""-m gpu: every hand-written kernel against an fp32 torch reference of the same op (through the C ABI)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


def pytest_generate_tests(metafunc):
    if "check" in metafunc.fixturenames:
        import kernel_checks as kc

        metafunc.parametrize("check", kc.ALL_CHECKS, ids=[c.__name__ for c in kc.ALL_CHECKS])


def test_kernel(cuda, check):
    res = check()
    assert isinstance(res, dict)


def test_c_abi_gemm_program(cuda, tmp_path):
    """a C99 program with no Python and no torch drives one dk_gemm (bias + GELU epilogue) through include/dkb200.h on
    the GPU and checks it against its own CPU evaluation — the boundary as a non-Python host sees it"""
    import shutil

    from diffusionkit_b200 import _lib

    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = tmp_path / "abi_gemm"
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-O1", os.path.join(HERE, "c", "abi_gemm.c"), "-o", str(exe),
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda_home, "include"),
                           "-L", libdir, "-ldkb200", f"-Wl,-rpath,{libdir}",
                           "-L", os.path.join(cuda_home, "lib64"), "-lcudart", f"-Wl,-rpath,{cuda_home}/lib64", "-lm"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
