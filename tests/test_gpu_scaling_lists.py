"""GPU tests (-m gpu) of scaling lists on every residual path (scaling_cases.py): res4_lane, res8_quarter and tu_residual in
k_residual (added onto the picture) and in k_intra (into the int16 scratch), 8-bit and 16-bit samples, factors over 1..255, qP'
up to 51 + QpBdOffset, transform skip of every size with RDPCM and rotation, unequal depths, 4:0:0, CTB 16 / 32.  The engine
against the CPU oracle sample for sample, a fresh engine per test, on each way a picture can reach it; the oracle is pinned to
the reference on the same cases by test_cpu_scaling_lists.py."""
import pytest

import scaling_cases
from libde265_b200 import capi, synth
from libde265_b200.engine import Engine
from test_cpu_scaling_lists import flag_cleared
from test_gpu_parity import assert_same
from test_gpu_range_edges import _read_async

pytestmark = pytest.mark.gpu
STAGES = (capi.STAGE_INTER_PRED, capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL)


def _oracle_pictures(oracle_mod, planes, pics):
    """The oracle's full pictures of the sequence, in decode order (slots filled with 77 / 99 first, as the engine's)."""
    orc = oracle_mod.Oracle()
    orc.upload_slot(5, pics[0].params, planes)
    out = []
    for p in pics:
        orc.fill_slot(p.params.dst_slot, p.params, 77, 99)
        orc.reconstruct(p)
        out.append(orc.read_slot(p.params.dst_slot, p.params))
    orc.close()
    return out


def _engine(planes, pics):
    e = Engine(0)
    e.upload_slot(5, pics[0].params, planes)
    for p in pics:
        e.fill_slot(p.params.dst_slot, p.params, 77, 99)
    return e


@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_submit_every_stage(oracle_mod, case):
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    e = _engine(planes, pics)
    orc = oracle_mod.Oracle()
    orc.upload_slot(5, pics[0].params, planes)
    for p in pics:
        orc.fill_slot(p.params.dst_slot, p.params, 77, 99)
    for i, p in enumerate(pics):
        for st in STAGES:
            p.c.params.stop_after_stage = st
            e.submit(p)
            orc.reconstruct(p)
            assert_same(e.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
        p.c.params.stop_after_stage = 0
    orc.close()
    e.close()


@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_submit_async_with_queued_reads(oracle_mod, case):
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    want = _oracle_pictures(oracle_mod, planes, pics)
    e = _engine(planes, pics)
    bufs = []
    for p in pics:
        e.submit_async(p)
        bufs.append(_read_async(e, p))
    e.sync()
    for i, (b, w) in enumerate(zip(bufs, want)):
        assert_same(b, w, f"{case} async pic {i}")
    e.close()


@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_prepared_path(oracle_mod, case):
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    want = _oracle_pictures(oracle_mod, planes, pics)
    e = _engine(planes, pics)
    for i, (p, w) in enumerate(zip(pics, want)):  # in decode order: later pictures read the earlier ones
        h = e.prepare(p)
        e.run_prepared(h)
        assert_same(e.read_slot(p.params.dst_slot, p.params), w, f"{case} prepared pic {i}")
        e.free_prepared(h)
    e.close()


@pytest.mark.parametrize("env", [{"B200_INTRA_SPLIT": "0"}, {"B200_REGION": "8"}], ids=["intra_split0", "region8"])
@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_other_intra_task_shapes(oracle_mod, monkeypatch, case, env):
    """k_intra with the planes of a region merged into one task, and with 8x8-luma regions: other groupings of the intra TUs that
    reach res4_lane / res8_quarter / tu_residual."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    want = _oracle_pictures(oracle_mod, planes, pics)
    e = _engine(planes, pics)
    for i, (p, w) in enumerate(zip(pics, want)):
        e.submit(p)
        assert_same(e.read_slot(p.params.dst_slot, p.params), w, f"{case} {env} pic {i}")
    e.close()


def test_4k_main10_b_and_i_with_default_lists(oracle_mod):
    """The headline size: a 3840x2160 10-bit B picture and I picture with the spec's default lists and transform skip up to 32x32,
    against the oracle."""
    W, H = 3840, 2160
    kw = dict(bit_depth=10, scaling_list="default", tskip_max_log2=5, special_frac=0.03)
    b = synth.make_picture(W, H, "B", seed=35, dst_slot=2, ref_slots=(0, 1), weighted=True, **kw)
    i = synth.make_picture(W, H, "I", seed=36, dst_slot=3, **kw)
    e, orc = Engine(0), oracle_mod.Oracle()
    for s in (0, 1):
        r = synth.random_planes(W, H, 10, 5 + s)
        e.upload_slot(s, b.params, r)
        orc.upload_slot(s, b.params, r)
    for p, tag in ((b, "4K Main10 B"), (i, "4K Main10 I")):
        assert (p.tus["flags"] & capi.TU_SCALING_LIST).any()
        e.submit(p)
        orc.reconstruct(p)
        assert_same(e.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), tag)
    orc.close()
    e.close()


@pytest.mark.parametrize("case", ["max10", "max8_ctb16"])
def test_factors_without_the_picture_flag_are_ignored(oracle_mod, case):
    """A picture whose TUs carry TU_SCALING_LIST, with factors present but PIC_SCALING_LIST clear, equals the same picture with
    scaling_factors NULL, and the oracle's picture."""
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    e = _engine(planes, pics)
    orc = oracle_mod.Oracle()
    orc.upload_slot(5, pics[0].params, planes)
    for p in pics:
        out = []
        for q in (flag_cleared(p, True), flag_cleared(p, False)):
            e.submit(q)
            out.append(e.read_slot(p.params.dst_slot, p.params))
        orc.reconstruct(flag_cleared(p, False))
        assert_same(out[0], out[1], f"{case} slot {p.params.dst_slot}: factors without the flag vs NULL")
        assert_same(out[0], orc.read_slot(p.params.dst_slot, p.params), f"{case} slot {p.params.dst_slot}: vs the oracle")
        e.submit(p)  # the later pictures reference the pictures with their matrices
        orc.reconstruct(p)
    orc.close()
    e.close()
