"""The oracle against the reference's own reconstruction functions (oracle/_ref/libref_replay.so, scalar and SIMD tables) on
sequences that change format mid-stream (format_cases.py), stage by stage, with every name read back at the end.  Without
oracle/_ref the oracle's pictures are checked against the stored digests of what the replay returned
(tests/golden/ref_pins.json).  A reference slot of another size, chroma format or bit depth predicts mid-grey, as in the
reference (motion.cc:385-405): test_mismatched_references_predict_as_missing holds the oracle to that rule directly."""
import numpy as np
import pytest

import format_cases
import oracle_lib
import ref_pins
from libde265_b200 import capi, synth
from test_cpu_ref_replay import same

HAVE_REF = oracle_lib.ref_replay_lib() is not None
pins = ref_pins.make_fixture(HAVE_REF)
STAGES = (capi.STAGE_INTER_PRED, capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL)


def params_of(case):
    """{slot: params of the picture it holds at the end}."""
    out = {}
    for (_, _, dst, _), p in zip(case.steps, format_cases.make_sequence(case.id)):
        out[dst] = p.params
    return out


@pytest.mark.parametrize("case", format_cases.CASE_IDS)
def test_every_case_reaches_its_switches(case):
    c = format_cases.BY_ID[case]
    pics = format_cases.make_sequence(case)
    missing = [desc for desc, ok in c.checks if not ok(c, pics)]
    assert not missing, f"{case}: the generated records lack {missing}"
    uncovered = [i for i, p in enumerate(pics) if not (format_cases.luma_coverage(p) > 0).all()]
    assert not uncovered, f"{case}: pictures {uncovered} leave luma samples that no PU or intra TU writes"
    for i, (f, _, _, refs) in enumerate(c.steps):
        p = pics[i]
        assert (p.params.width, p.params.height, p.params.bit_depth_luma, p.params.bit_depth_chroma, p.params.chroma_format_idc,
                p.params.log2_ctb_size) == (f.W, f.H, f.bd, f.bdc, f.cf, f.ctb)
    assert any(format_cases.mismatched_ref_slots(c, i) for i in range(len(pics))) or case == "ctb_64_16_32", \
        f"{case}: no picture references a slot of another format"


@pytest.mark.parametrize("simd", [False, True])
@pytest.mark.parametrize("case", format_cases.CASE_IDS)
def test_replay_matches_oracle_across_format_switches(pins, case, simd):
    c = format_cases.BY_ID[case]
    pics = format_cases.make_sequence(case)
    orc = oracle_lib.Oracle()
    # A replay library built from an older oracle/ref_replay.cc cannot rewrite a name with another CTB size: the stored digests
    # pin those cases.
    pins.have_ref = HAVE_REF and (oracle_lib.ref_replay_handles_ctb_change() or not format_cases.rewrites_ctb(c))
    ref = oracle_lib.RefReplay(simd=simd) if pins.have_ref else None
    for i, p in enumerate(pics):
        for st in STAGES:
            p.c.params.stop_after_stage = st
            orc.reconstruct(p)
            if ref is not None:
                ref.reconstruct(p)
            same(pins, ref and ref.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
        p.c.params.stop_after_stage = 0
    for s, prm in sorted(params_of(c).items()):  # every name at the end, the ones that still hold an earlier format's picture included
        same(pins, ref and ref.read_slot(s, prm), orc.read_slot(s, prm), f"{case} slot {s} at the end")
    orc.close()
    if ref is not None:
        ref.close()


def without_refs(p, slots):
    """The picture with every PU list that names one of `slots` pointed at no slot (-1)."""
    pus = p.pus.copy()
    for l in range(2):
        pus["ref_slot"][np.isin(pus["ref_slot"][:, l], slots), l] = -1
    return synth.SynthPicture(p.params, pus, p.weights, p.tus, p.coeffs, p.slices, p.ctbs, p.bs_map, p.qp_map, p.nofilt_map)


@pytest.mark.parametrize("case", [c for c in format_cases.CASE_IDS if c != "ctb_64_16_32"])
def test_mismatched_references_predict_as_missing(oracle_mod, case):
    """Every picture that references a slot of another format gives, stage by stage, the same samples as the picture with
    those references removed: the oracle treats them as missing references (mid-grey), as the reference does."""
    c = format_cases.BY_ID[case]
    pics = format_cases.make_sequence(case)
    orc = oracle_mod.Oracle()
    checked = 0
    for i, p in enumerate(pics):
        bad = format_cases.mismatched_ref_slots(c, i)
        if bad:
            q = without_refs(p, bad)
            used = (p.pus["flags"][:, None] & np.array([capi.PU_PRED_L0, capi.PU_PRED_L1], np.uint8)) != 0
            assert (used & (q.pus["ref_slot"] != p.pus["ref_slot"])).any(), f"{case} pic {i}: no PU predicts from slots {bad}"
            for st in STAGES:
                p.c.params.stop_after_stage = q.c.params.stop_after_stage = st
                orc.reconstruct(q)
                want = orc.read_slot(p.params.dst_slot, p.params)
                orc.reconstruct(p)
                got = orc.read_slot(p.params.dst_slot, p.params)
                for k, (a, b) in enumerate(zip(got, want)):
                    assert (a == b).all(), f"{case} pic {i} stage {st} plane {k}: a reference in slots {bad} of another format was used"
            p.c.params.stop_after_stage = 0
            checked += 1
        orc.reconstruct(p)
    orc.close()
    assert checked


def test_ctb_switch_keeps_references():
    """A slot that differs from the picture only in its CTB size is an ordinary reference: removing it changes the picture."""
    c = format_cases.BY_ID["ctb_64_16_32"]
    pics = format_cases.make_sequence(c.id)
    orc = oracle_lib.Oracle()
    changed = 0
    for i, p in enumerate(pics):
        held = format_cases.slot_formats(c)[0][i]
        other_ctb = [s for s in c.steps[i][3] if s in held and format_cases.ref_kind(c.steps[i][0], held[s]) == "ctb"]
        if other_ctb:
            orc.reconstruct(without_refs(p, other_ctb))
            grey = orc.read_slot(p.params.dst_slot, p.params)
            orc.reconstruct(p)
            changed += any((a != b).any() for a, b in zip(orc.read_slot(p.params.dst_slot, p.params), grey))
        orc.reconstruct(p)
    orc.close()
    assert changed >= 2
