"""GPU tests (-m gpu): k_intra on availability masks with gaps, from constrained intra prediction in P / B pictures, against the
CPU oracle (which test_cpu_range_edges.py pins to the reference on the same kind of pictures, masks included).

A TU whose own left column, corner and top row are available and whose bottom-left / top-right reach is available up to a
point takes the fast (4x4 / 8x8) or fused (16x16 / 32x32) path, where substitution is a clamp.  Any other takes the general
path: the ballot / shuffle substitution chain of tu_intra_small (with the 33rd sample of an 8x8 TU in its own register) or the
chunked scan of tu_intra_large (with a value carried across 32-sample chunks).  The range-edge loop runs the constrained-intra
cases of range_cases.py stage by stage; this file adds the path counts, the intra task shapes and full-size pictures."""
import pytest

import range_cases
from intra_plan_cases import fast_clamps
from libde265_b200 import capi, synth
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same

pytestmark = pytest.mark.gpu

KINDS = range_cases.SIZE_KINDS


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def path_counts(tus):
    """Per size kind: (general path because of a gap, fast / fused path with only a prefix of a reach available)."""
    gap_classes = {"own_partial", "corner_missing", "reach_gap", "outer_only", "corner_only"}
    out = {k: [0, 0] for k in KINDS}
    for tu in tus[(tus["flags"] & capi.TU_INTRA) != 0]:
        log2 = int(tu["log2_size"])
        kind = {2: "4", 3: "8c" if tu["cidx"] else "8y", 4: "16", 5: "32"}[log2]
        if fast_clamps(tu) is not None:
            q = 1 << (log2 - 2)
            full = (1 << q) - 1
            av = int(tu["avail"])
            if (av >> q) & full != full or (av >> (capi.AVAIL_TOP_BIT0 + q)) & full != full:
                out[kind][1] += 1
        elif gap_classes & set(range_cases.tu_gap_classes(tu)):
            out[kind][0] += 1
    return out


def upload_refs(engines, params, slots, seed=5):
    for s in slots:
        r = synth.random_planes(params.width, params.height, params.bit_depth_luma, seed + s)
        for e in engines:
            e.upload_slot(s, params, r)


@pytest.mark.parametrize("bd", [8, 10])
def test_gap_paths_on_a_cip_b_picture(eng, oracle_mod, bd):
    """A constrained-intra B picture, 70 % intra CUs, cut by tiles and slices: at every TU size, at least 10 TUs take the general
    path because of a gap and at least 5 take the fast / fused path with part of a reach missing."""
    W, H = 640, 384
    p = synth.make_picture(W, H, "B", seed=51 + bd, dst_slot=2, ref_slots=(0, 1), bit_depth=bd, intra_frac=0.7,
                           size_area=(0.2, 0.5, 0.15, 0.15), tiles=(2, 2), n_slices=3, constrained_intra=True)
    counts = path_counts(p.tus)
    for k in KINDS:
        assert counts[k][0] >= 10, (k, counts)
        assert counts[k][1] >= 5, (k, counts)
    orc = oracle_mod.Oracle()
    upload_refs((eng, orc), p.params, (0, 1))
    for st in (capi.STAGE_RECON, capi.STAGE_ALL):
        p.c.params.stop_after_stage = st
        eng.submit(p)
        orc.reconstruct(p)
        assert_same(eng.read_slot(2, p.params), orc.read_slot(2, p.params), f"stage {st}")
    p.c.params.stop_after_stage = 0
    orc.close()


@pytest.mark.parametrize("env", [{"B200_INTRA_SPLIT": "0"}, {"B200_REGION": "8"}, {"B200_INTRA_ORDER": "level_i"}, {"B200_INTRA_ORDER": "diag"}],
                         ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_intra_task_shapes_on_cip(oracle_mod, monkeypatch, env):
    """The non-default shapes of the intra work list on a constrained-intra sequence, a fresh engine each: planes of a region
    merged into one task (pictures with inter prediction), 8x8 regions (an 8x8 luma or 4x4 chroma TU is then a task of its own
    and takes the large-TU code), the level order in intra pictures only, and the CTB anti-diagonal order."""
    c = range_cases.BY_ID["cip10_tiles_slices"]
    planes, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    orc = oracle_mod.Oracle()
    orc.upload_slot(5, pics[0].params, planes)
    expect = []
    for p in pics:
        orc.reconstruct(p)
        expect.append(orc.read_slot(p.params.dst_slot, p.params))
    orc.close()
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    e = Engine(0)
    e.upload_slot(5, pics[0].params, planes)
    for p, x in zip(pics, expect):
        e.submit(p)
        assert_same(e.read_slot(p.params.dst_slot, p.params), x, f"{env} slot {p.params.dst_slot}")
    e.close()


def test_4k_cip_b_and_10bit_cip_p(eng, oracle_mod):
    """Full size: a 3840x2160 8-bit constrained-intra B picture (30 % intra CUs) and a 10-bit constrained-intra P picture."""
    W, H = 3840, 2160
    orc = oracle_mod.Oracle()
    for bd, kind, seed, refs in ((8, "B", 61, (0, 1)), (10, "P", 62, (0,))):
        p = synth.make_picture(W, H, kind, seed=seed, dst_slot=3, ref_slots=refs, bit_depth=bd, intra_frac=0.3, constrained_intra=True)
        assert sum(n for n, _ in path_counts(p.tus).values()) >= 1000
        upload_refs((eng, orc), p.params, refs)
        eng.submit(p)
        orc.reconstruct(p)
        assert_same(eng.read_slot(3, p.params), orc.read_slot(3, p.params), f"4K {bd}-bit CIP {kind}")
    orc.close()
