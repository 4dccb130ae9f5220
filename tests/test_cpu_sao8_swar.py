"""The byte-parallel primitives of k_sao8 (libde265_b200/csrc/sao8_swar.cuh: unsigned byte compare, zero-byte test, saturating
offset add / subtract, bit -> byte-mask expansion) checked EXHAUSTIVELY on the CPU: tests/sao8_emul.cu compiles the very same
__host__ __device__ functions for the host (PRMT replaced by its definition).  The GPU parity tests run k_sao8 against the oracle on
whole pictures; this one pins the arithmetic of the building blocks without a GPU."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libsao8_emul.so")
SRC = os.path.join(HERE, "sao8_emul.cu")
HDR = os.path.join(ROOT, "libde265_b200", "csrc", "sao8_swar.cuh")


@pytest.fixture(scope="module")
def lib():
    if not (os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in (SRC, HDR))):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-I" + os.path.dirname(HDR), "-o", SO, SRC])
    l = C.CDLL(SO)
    for f in ("sao8_check_lt", "sao8_check_apply", "sao8_check_eq_mask"):
        getattr(l, f).restype = C.c_long
    return l


def test_unsigned_byte_compare_all_pairs(lib):
    assert lib.sao8_check_lt() == 0


def test_saturating_offset_all_samples_and_offsets(lib):
    assert lib.sao8_check_apply() == 0


def test_zero_byte_test_and_mask_expansion(lib):
    assert lib.sao8_check_eq_mask() == 0
