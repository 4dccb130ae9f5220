"""The RGB export's arithmetic (libde265_b200/csrc/export.cuh) on the CPU: tests/export_emul.cu builds the very
__host__ __device__ coefficient derivation and per-pixel function k_export_rgb runs, and export_ref.py restates them.  The host
build is checked against the float64 definition (within +-1 everywhere) and against the numpy integer restatement (exactly);
test_gpu_export.py then checks the GPU's output against the same restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import export_ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libexport_emul.so")
SRC = os.path.join(HERE, "export_emul.cu")
HDR = os.path.join(ROOT, "libde265_b200", "csrc", "export.cuh")

I32P = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


@pytest.fixture(scope="module")
def lib():
    if not (os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in (SRC, HDR))):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-I" + os.path.dirname(HDR), "-o", SO, SRC])
    l = C.CDLL(SO)
    l.export_emul_coefs.argtypes = [C.c_int] * 4 + [I32P]
    l.export_emul_coefs.restype = None
    l.export_emul_rgb.argtypes = [C.c_int] * 4 + [I32P] * 3 + [C.c_long, np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")]
    l.export_emul_rgb.restype = None
    return l


def host_rgb(lib, matrix, full, bd_y, bd_c, y, cb, cr):
    y, cb, cr = (np.ascontiguousarray(a, np.int32) for a in (y, cb, cr))
    out = np.empty((len(y), 3), np.uint8)
    lib.export_emul_rgb(matrix, int(full), bd_y, bd_c, y, cb, cr, len(y), out)
    return out


DEPTHS = [(8, 8), (10, 10), (12, 12), (10, 12), (12, 9)]
CASES = [(m, full, bd_y, bd_c) for m in (1, 2, 3) for full in (False, True) for bd_y, bd_c in DEPTHS]


def test_coefficients_equal_the_restatement(lib):
    for m, full, bd_y, bd_c in CASES:
        got = np.empty(7, np.int32)
        lib.export_emul_coefs(m, int(full), bd_y, bd_c, got)
        assert got.tolist() == export_ref.coefs(m, full, bd_y, bd_c), (m, full, bd_y, bd_c)


@pytest.mark.parametrize("matrix", [1, 2, 3])
@pytest.mark.parametrize("full", [False, True])
def test_every_8bit_triple_within_one_of_the_definition(lib, matrix, full):
    y, cb, cr = (a.ravel() for a in np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij"))
    got = host_rgb(lib, matrix, full, 8, 8, y, cb, cr).astype(np.int64)
    want = export_ref.rgb_float(matrix, full, 8, 8, y, cb, cr)
    err = np.abs(got - want)
    assert err.max() <= 1.0, f"worst at {np.unravel_index(err.argmax(), err.shape)}: {err.max()}"


@pytest.mark.parametrize("bd_y,bd_c", [(10, 10), (12, 12), (10, 12), (12, 9)])
def test_every_luma_with_seeded_chroma_within_one_of_the_definition(lib, bd_y, bd_c):
    rng = np.random.default_rng(bd_y * 100 + bd_c)
    y = np.repeat(np.arange(1 << bd_y), 64)  # every Y, each with 64 chroma pairs
    cb, cr = (rng.integers(0, 1 << bd_c, len(y)) for _ in range(2))
    for matrix in (1, 2, 3):
        for full in (False, True):
            got = host_rgb(lib, matrix, full, bd_y, bd_c, y, cb, cr).astype(np.int64)
            err = np.abs(got - export_ref.rgb_float(matrix, full, bd_y, bd_c, y, cb, cr))
            assert err.max() <= 1.0, (matrix, full, err.max())


def test_host_build_equals_the_integer_restatement(lib):
    rng = np.random.default_rng(7)
    for m, full, bd_y, bd_c in CASES:
        n = 200000
        y, cb, cr = rng.integers(0, 1 << bd_y, n), rng.integers(0, 1 << bd_c, n), rng.integers(0, 1 << bd_c, n)
        got = host_rgb(lib, m, full, bd_y, bd_c, y, cb, cr)
        assert (got == export_ref.rgb_int(m, full, bd_y, bd_c, y, cb, cr)).all(), (m, full, bd_y, bd_c)


def test_grey_and_extremes(lib):
    """Mid-grey chroma gives R = G = B (the 4:0:0 export), and the nominal black and white map to 0 and 255 at every depth."""
    for m, full, bd_y, bd_c in CASES:
        oy, ry, oc, _ = export_ref.ranges(full, bd_y, bd_c)
        y = np.arange(1 << bd_y)
        g = host_rgb(lib, m, full, bd_y, bd_c, y, np.full_like(y, oc), np.full_like(y, oc))
        assert (g[:, 0] == g[:, 1]).all() and (g[:, 1] == g[:, 2]).all()
        ends = host_rgb(lib, m, full, bd_y, bd_c, [oy, oy + ry], [oc, oc], [oc, oc])
        assert ends[0].tolist() == [0, 0, 0] and ends[1].tolist() == [255, 255, 255], (m, full, bd_y, bd_c)
