"""GPU tests (-m gpu): the two paths of k_intra's large (16x16 / 32x32) intra TUs against the CPU oracle.  A TU whose own left
column, corner and top row are available, and whose bottom-left / top-right reach is available up to a point, takes the fused
path (substitution by clamping, prediction + residual straight to the picture).  Any other (picture, slice and tile edges)
takes the general path with the substitution process.  The pictures are coded mostly in 64x64 / 32x32 CUs and cut into tiles
and slices, so both paths run many times, angular modes included."""
import numpy as np
import pytest

from libde265_b200 import capi, synth
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def large_tu_counts(tus):
    """Intra TUs of 16x16 / 32x32 by path: (fused 32x32 angular luma, fused with all 4nT + 1 border samples available,
    fused with part of the bottom-left / top-right reach missing, general)"""
    t = tus[(tus["flags"] & capi.TU_INTRA) != 0]
    t = t[t["log2_size"] >= 4]
    av = t["avail"].astype(np.uint64)
    q = (1 << (t["log2_size"].astype(np.int64) - 2)).astype(np.uint64)
    g = (np.uint64(1) << q) - np.uint64(1)
    own = ((av & g) == g) & (((av >> np.uint64(16)) & np.uint64(1)) == 1) & (((av >> np.uint64(17)) & g) == g)
    bl, tr = (av >> q) & g, (av >> (np.uint64(17) + q)) & g
    fused = own & ((bl & (bl + np.uint64(1))) == 0) & ((tr & (tr + np.uint64(1))) == 0)
    full = fused & (bl == g) & (tr == g)
    n32 = int((fused & (t["log2_size"] == 5) & (t["cidx"] == 0) & (t["intra_mode"] >= 2)).sum())
    return n32, int(full.sum()), int((fused & ~full).sum()), int((~fused).sum())


@pytest.mark.parametrize("bd", [8, 10])
@pytest.mark.parametrize("strong", [True, False])
def test_large_intra_tus_both_paths(eng, oracle_mod, bd, strong):
    W, H = 640, 384
    p = synth.make_picture(W, H, "I", seed=41 + bd, bit_depth=bd, size_area=(0.5, 0.4, 0.1, 0.0), tiles=(2, 2), n_slices=3,
                           strong_smoothing=strong)
    counts = large_tu_counts(p.tus)
    assert min(counts) >= 20, counts
    orc = oracle_mod.Oracle()
    for st in (capi.STAGE_RECON, capi.STAGE_ALL):
        p.c.params.stop_after_stage = st
        eng.submit(p)
        orc.reconstruct(p)
        assert_same(eng.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"stage {st}")
    p.c.params.stop_after_stage = 0
    orc.close()
