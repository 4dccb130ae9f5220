"""The TMA-staged MC kernel's task bodies (libde265_b200/csrc/kernels_mct.cuh) executed ON THE CPU (tests/mct_emul.cu compiles the
very same __host__ __device__ functions for the host; the TMA box fetch becomes a copy out of a padded surface) against the
oracle's inter-prediction stage: every phase combination, PUs hanging off all picture edges, far motion vectors (windows
moved to the border's rim), all weighting modes, missing references, every tile class of the host planner.  The GPU parity
tests run the same code on the device; this one catches arithmetic / indexing mistakes without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib
from libde265_b200 import capi, synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libmct_emul.so")
SRC = os.path.join(HERE, "mct_emul.cu")
CSRC = os.path.join(ROOT, "libde265_b200", "csrc")


def build_emulator():
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("kernels_mct.cuh", "kernels_mc8.cuh", "dev_common.cuh")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", SO, SRC])


@pytest.fixture(scope="module")
def emul():
    build_emulator()
    lib = C.CDLL(SO)
    lib.mct_emulate.argtypes = [C.POINTER(capi.Picture), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint32), C.c_int]
    return lib


def plan_tiles(lib, pic):
    counts = (C.c_uint32 * 8)()
    capi.check(lib.b200_plan_picture_host(C.byref(pic.c), counts, None, 0, None, 0, None, 0, None, 0), "plan")
    n = counts[0]
    units = (C.c_uint32 * max(1, n))()
    capi.check(lib.b200_plan_picture_host(C.byref(pic.c), counts, units, n, None, 0, None, 0, None, 0), "plan")
    return units, n


def run_case(b200lib, emul, W, H, ptype, seed, refs_present=(0, 1), **kw):
    orc = oracle_lib.Oracle()
    pic = synth.make_picture(W, H, ptype, seed=seed, dst_slot=2, ref_slots=(0, 1), **kw)
    planes = {s: synth.random_planes(W, H, 8, 10 + s) for s in refs_present}
    for s, p in planes.items():
        orc.upload_slot(s, pic.params, p)
    pic.c.params.stop_after_stage = capi.STAGE_INTER_PRED
    orc.reconstruct(pic)
    want = orc.read_slot(2, pic.params)
    orc.close()
    units, n = plan_tiles(b200lib, pic)
    refp = (C.c_void_p * 96)()
    for s, p in planes.items():
        for c in range(3):
            refp[3 * s + c] = p[c].ctypes.data
    got = [np.zeros((H, W), np.uint8), np.zeros((H // 2, W // 2), np.uint8), np.zeros((H // 2, W // 2), np.uint8)]
    dst = (C.c_void_p * 3)(*[g.ctypes.data for g in got])
    assert emul.mct_emulate(C.byref(pic.c), refp, dst, units, n) == 0
    for c in range(3):
        d = np.argwhere(got[c] != want[c])
        assert len(d) == 0, f"plane {c}: {len(d)} samples differ, first at (x={d[0][1]}, y={d[0][0]}): kernel {got[c][tuple(d[0])]} != oracle {want[c][tuple(d[0])]}"
    classes = {(int(u) >> 24) & 7 for u in units[:n] if u != 0xFFFFFFFF}
    return classes


def test_planner_emits_class_pure_batches(b200lib):
    pic = synth.make_picture(416, 240, "B", seed=3, dst_slot=2, ref_slots=(0, 1))
    units, n = plan_tiles(b200lib, pic)
    u = np.frombuffer(units, np.uint32)[:n]
    covered = np.zeros((240, 416), np.int32)
    batches, first = [], 0
    while first < n:  # batches are self-describing: the first tile's class gives the batch size (32 tile-list items with small boxes, else 16)
        cls = (int(u[first]) >> 24) & 7
        size = (16 if cls & 5 else 32) >> (1 if cls & 2 else 0)
        batches.append(u[first:first + size])
        first += size
    assert first == n
    for batch in batches:
        assert batch[0] != 0xFFFFFFFF
        cls = (batch[0] >> 24) & 7
        for w in batch:
            if w == 0xFFFFFFFF:
                continue
            assert (w >> 24) & 7 == cls
            pu = pic.pus[w & 0xFFFFF]
            tx, ty = int((w >> 20) & 3), int((w >> 22) & 3)
            tw, th = min(16, int(pu["w"]) - 16 * tx), min(16, int(pu["h"]) - 16 * ty)
            assert tw > 0 and th > 0 and (tw > 8) == bool(cls & 1) and (th > 8) == bool(cls & 4)
            assert bool(cls & 2) == ((pu["flags"] & 3) == 3)
            covered[int(pu["y"]) + 16 * ty:int(pu["y"]) + 16 * ty + th, int(pu["x"]) + 16 * tx:int(pu["x"]) + 16 * tx + tw] += 1
    inter = np.zeros((240, 416), np.int32)
    for pu in pic.pus:
        if pu["flags"] & 3:
            x, y, w, h = int(pu["x"]), int(pu["y"]), int(pu["w"]), int(pu["h"])
            inter[y:y + h, x:x + w] += 1
    assert (covered == inter).all()  # every predicted sample belongs to exactly one tile


@pytest.mark.parametrize("ptype,seed,kw", [("P", 5, {}), ("B", 6, {}), ("B", 7, {"weighted": True}), ("B", 8, {"far_mv_frac": 0.3}),
                                           ("B", 9, {"size_area": (0.0, 0.0, 0.2, 0.8)}), ("B", 10, {"size_area": (0.6, 0.4, 0.0, 0.0), "weighted": True})])
def test_emulated_kernel_matches_oracle(b200lib, emul, ptype, seed, kw):
    run_case(b200lib, emul, 416, 240, ptype, seed, **kw)


def test_emulated_kernel_all_classes_ragged_sizes_and_missing_reference(b200lib, emul):
    seen = set()
    for size in ((72, 40), (200, 136), (1288, 8), (64, 64)):
        seen |= run_case(b200lib, emul, size[0], size[1], "B", 21, far_mv_frac=0.1)
    seen |= run_case(b200lib, emul, 320, 192, "B", 22, refs_present=(0,))  # slot 1 never written: mid-grey
    seen |= run_case(b200lib, emul, 320, 192, "B", 23, log2_ctb=4, size_area=(0.0, 0.0, 0.5, 0.5))
    assert seen == set(range(8)), f"tile classes exercised: {sorted(seen)}"
