"""GPU tests (-m gpu) at the edges of what a record may carry (range_cases.py): 4:0:0, 9..12 bit and unequal luma / chroma
depths, extreme QP, deblocking / chroma QP offsets, weights, offsets, MVs and SAO offsets, the smoothing / boundary-filter /
PCM / per-slice filter switches.  The engine against the CPU oracle, stage by stage, sample for sample; the oracle is pinned to
the reference on the same cases by test_cpu_range_edges.py."""
import numpy as np
import pytest

import range_cases
from libde265_b200 import capi, synth
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same, md5_planes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def upload(engines, planes, params):
    for e in engines:
        e.upload_slot(5, params, planes)


@pytest.mark.parametrize("case", range_cases.CASE_IDS)
def test_engine_matches_oracle_at_the_edges(eng, oracle_mod, case):
    c = range_cases.BY_ID[case]
    planes, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    orc = oracle_mod.Oracle()
    upload((eng, orc), planes, pics[0].params)
    for p in pics:  # samples no record covers keep the slot's content: the engine's slots still hold the previous case's pictures
        eng.fill_slot(p.params.dst_slot, p.params, 77, 99)
        orc.fill_slot(p.params.dst_slot, p.params, 77, 99)
    for i, p in enumerate(pics):
        for st in (capi.STAGE_INTER_PRED, capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL):
            p.c.params.stop_after_stage = st
            eng.submit(p)
            orc.reconstruct(p)
            assert_same(eng.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
        p.c.params.stop_after_stage = 0
    orc.close()


def test_4k_main12_b_and_4k_mono_i(eng, oracle_mod):
    """Full size: a 3840x2160 12-bit B picture (both lists, weights and offsets across their whole range, MVs up to the int16
    ends on the border PUs, SAO offsets at the maximum) and a 4:0:0 I picture, against the oracle."""
    W, H = 3840, 2160
    orc = oracle_mod.Oracle()
    b = synth.make_picture(W, H, "B", seed=25, dst_slot=2, ref_slots=(0, 1), bit_depth=12, weighted=True, weight_range="spec",
                           extreme_mv_frac=0.3, sao_offset="max")
    assert (b.pus["mv"] == -32768).any() and (b.pus["mv"] == 32767).any()
    for s in (0, 1):
        r = synth.random_planes(W, H, 12, 5 + s)
        eng.upload_slot(s, b.params, r)
        orc.upload_slot(s, b.params, r)
    eng.submit(b)
    orc.reconstruct(b)
    assert_same(eng.read_slot(2, b.params), orc.read_slot(2, b.params), "4K Main12 B")
    i = synth.make_picture(W, H, "I", seed=26, dst_slot=3, chroma_format_idc=0, special_frac=0.03)
    eng.submit(i)
    orc.reconstruct(i)
    assert_same(eng.read_slot(3, i.params), orc.read_slot(3, i.params), "4K 4:0:0 I")
    orc.close()


def _read_async(e, p):
    """Queues a read of the picture's slot into fresh arrays (luma only in 4:0:0); valid after e.sync()."""
    dt = np.uint16 if p.params.bit_depth_luma > 8 else np.uint8
    W, H = p.params.width, p.params.height
    bufs = [np.empty((H, W), dt)] + ([np.empty((H // 2, W // 2), dt) for _ in range(2)] if p.params.chroma_format_idc else [])
    capi.check(e.lib.b200_engine_read_slot_async(e.handle, p.params.dst_slot, capi.PlaneArray(*[x.ctypes.data for x in bufs] + [None] * (3 - len(bufs))),
                                                 capi.StrideArray(*[x.strides[0] for x in bufs] + [0] * (3 - len(bufs)))), "read_slot_async")
    return bufs


@pytest.mark.parametrize("case", ["mono8_ctb64", "bd12", "bd12_chroma9"])
def test_prepared_async_and_streams_match_submit(case):
    """The prepared (HBM-resident) path, the asynchronous call and four CUDA streams give the same pictures as submit()."""
    c = range_cases.BY_ID[case]
    planes, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    e = Engine(0)
    upload((e,), planes, pics[0].params)
    expect = []
    for p in pics:
        e.submit(p)
        expect.append(md5_planes(e.read_slot(p.params.dst_slot, p.params)))
    for p, want in zip(pics, expect):  # the prepared path, in decode order (later pictures read the earlier ones)
        h = e.prepare(p)
        e.fill_slot(p.params.dst_slot, p.params, 0, 0)
        e.run_prepared(h)
        assert md5_planes(e.read_slot(p.params.dst_slot, p.params)) == want, f"{case}: prepared picture {p.params.dst_slot}"
        e.free_prepared(h)
    e.close()
    for n, submit_async in ((1, True), (4, False), (4, True)):
        e = Engine(0)
        e.set_streams(n)
        upload((e,), planes, pics[0].params)
        bufs = []
        for p in pics:
            (e.submit_async if submit_async else e.submit)(p)
            bufs.append(_read_async(e, p))
        e.sync()
        got = [md5_planes(b) for b in bufs]
        assert got == expect, f"{case}, {n} stream(s), async={submit_async}: pictures {[i for i, (g, x) in enumerate(zip(got, expect)) if g != x]} differ"
        e.close()


def test_mono_intra_task_variants(oracle_mod, monkeypatch):
    """The non-default shapes of the intra work list on 4:0:0 pictures, where every region has luma tasks only: planes of a region
    merged into one task (B200_INTRA_SPLIT=0) and CTB anti-diagonal ticket order (B200_INTRA_ORDER=diag)."""
    c = range_cases.BY_ID["mono8_ctb64"]
    planes, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    i16 = synth.make_picture(208, 120, "I", seed=15, dst_slot=4, chroma_format_idc=0, log2_ctb=4, size_area=(0.0, 0.0, 0.5, 0.5))
    orc = oracle_mod.Oracle()
    orc.upload_slot(5, pics[0].params, planes)
    expect = []
    for p in pics + [i16]:
        orc.reconstruct(p)
        expect.append(orc.read_slot(p.params.dst_slot, p.params))
    orc.close()
    for env in ({"B200_INTRA_SPLIT": "0"}, {"B200_INTRA_ORDER": "diag"}, {"B200_INTRA_SPLIT": "0", "B200_INTRA_ORDER": "diag"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = Engine(0)
        e.upload_slot(5, pics[0].params, planes)
        for p, x in zip(pics + [i16], expect):
            e.submit(p)
            assert_same(e.read_slot(p.params.dst_slot, p.params), x, f"{env} slot {p.params.dst_slot}")
        e.close()
        for k in env:
            monkeypatch.delenv(k)


def test_out_of_range_records_are_rejected(eng, oracle_mod):
    """A chroma TU in a 4:0:0 picture, bit depth 13 and mixed 8 / 10-bit planes raise B200Error, and the engine keeps working."""
    mono = synth.make_picture(64, 64, "I", seed=45, dst_slot=1, chroma_format_idc=0)
    with_chroma = synth.make_picture(64, 64, "I", seed=45, dst_slot=1)
    bad = synth.SynthPicture(mono.params, mono.pus, mono.weights, with_chroma.tus, with_chroma.coeffs, mono.slices, mono.ctbs, mono.bs_map,
                             mono.qp_map, mono.nofilt_map)
    assert (bad.tus["cidx"] != 0).any()
    with pytest.raises(capi.B200Error, match="TU"):
        eng.submit(bad)
    deep = synth.make_picture(64, 64, "I", seed=46, dst_slot=1, bit_depth=12)
    deep.c.params.bit_depth_luma = deep.c.params.bit_depth_chroma = 13
    with pytest.raises(capi.B200Error, match="bit depth"):
        eng.submit(deep)
    for bd_y, bd_c in ((8, 10), (10, 8)):
        mixed = synth.make_picture(64, 64, "I", seed=47, dst_slot=1, bit_depth=10)
        mixed.c.params.bit_depth_luma, mixed.c.params.bit_depth_chroma = bd_y, bd_c
        with pytest.raises(capi.B200Error, match="mixed"):
            eng.submit(mixed)
    orc = oracle_mod.Oracle()
    for p in (mono, synth.make_picture(64, 64, "I", seed=48, dst_slot=2, bit_depth=12, bit_depth_chroma=9)):
        eng.submit(p)
        orc.reconstruct(p)
        assert_same(eng.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), "after the rejections")
    orc.close()
