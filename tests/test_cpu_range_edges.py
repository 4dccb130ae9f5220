"""The oracle against the reference's own reconstruction functions (oracle/_ref/libref_replay.so, scalar and SIMD tables) on the
edges of what a record may carry (range_cases.py): every case as an I -> P -> B -> weighted B sequence, stage by stage.
Without oracle/_ref the oracle's pictures are checked against the stored digests of what the replay returned
(tests/golden/ref_pins.json), as in test_cpu_ref_replay.py.  The cases with constrained intra prediction are replayed with
the reference's constrained_intra_pred_flag set, and every synthetic availability mask is checked against the one the
reference derives."""
import pytest

import oracle_lib
import ref_pins
import range_cases
from libde265_b200 import capi
import test_cpu_ref_replay
from test_cpu_ref_replay import same

HAVE_REF = oracle_lib.ref_replay_lib() is not None
pins = ref_pins.make_fixture(HAVE_REF)


@pytest.mark.parametrize("case", range_cases.CASE_IDS)
def test_every_case_reaches_its_edges(case):
    c = range_cases.BY_ID[case]
    _, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    missing = [desc for desc, ok in c.checks if not ok(pics)]
    assert not missing, f"{case}: the generated records lack {missing}"


@pytest.mark.parametrize("simd", [False, True])
@pytest.mark.parametrize("case", range_cases.CASE_IDS)
def test_replay_matches_oracle_at_the_edges(pins, case, simd):
    c = range_cases.BY_ID[case]
    planes, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    orc = oracle_lib.Oracle()
    cip = c.kw.get("constrained_intra", False)
    # A replay library built from an older oracle/ref_replay.cc cannot replay constrained intra: the stored digests pin those cases.
    pins.have_ref = HAVE_REF and (not cip or oracle_lib.ref_replay_has_options())
    ref = oracle_lib.RefReplay(simd=simd, constrained_intra=cip) if pins.have_ref else None
    for e in (orc, ref):
        if e is not None:
            e.upload_slot(5, pics[0].params, planes)
    for i, p in enumerate(pics):
        for st in (capi.STAGE_INTER_PRED, capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL):
            p.c.params.stop_after_stage = st
            orc.reconstruct(p)
            if ref is not None:
                ref.reconstruct(p)
            same(pins, ref and ref.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
        p.c.params.stop_after_stage = 0
    orc.close()
    if ref is not None:
        ref.close()


def test_cip_cases_cover_every_gap_class():
    """Over the constrained-intra cases together: every gap class at every TU size the geometry allows, an 8x8 TU whose only
    available group is top group 3, and a 32x32 TU whose substitution carries a value across a 32-sample chunk."""
    total = {}
    for case in range_cases.CIP_CASE_IDS:
        c = range_cases.BY_ID[case]
        _, pics = range_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
        for k, v in range_cases.gap_counts(pics).items():
            total[k] = total.get(k, 0) + v
    want = [(c, k) for c in range_cases.GAP_CLASSES for k in range_cases.SIZE_KINDS if (c, k) not in range_cases.GEOMETRY_FORBIDS]
    missing = [w for w in want + [("32_carry", "32")] if not total.get(w)]
    if not any(k[0] == "8_top3_only" for k in total):
        missing.append("8x8 with top group 3 only")
    assert not missing, f"no constrained-intra case reaches {missing}"


def _mask_sequences():
    for c in range_cases.CASES:
        yield c.id, c.W, c.H, c.bd, c.kw
    for name in ("EVERY_STAGE", "RAGGED", "SPECIAL"):
        for i, (W, H, bd, kw) in enumerate(getattr(test_cpu_ref_replay, name)):
            yield f"test_cpu_ref_replay.{name}[{i}]", W, H, bd, {k: v for k, v in kw.items() if k != "stages"}


@pytest.mark.skipif(not oracle_lib.ref_replay_has_options(),
                    reason="needs the replay executor built from the reference with rr_set_options (oracle/_ref/libref_replay.so)")
def test_synthetic_masks_match_the_reference():
    """The availability mask of every intra TU that synth records, in every range case and every sequence of
    test_cpu_ref_replay.py, equals the mask the reference derives for the same picture (intra_border_computer, with
    constrained_intra_pred_flag where the case sets it).  Pixel equality alone can hide a wrong mask where the substituted
    values happen to agree."""
    for name, W, H, bd, kw in _mask_sequences():
        planes, pics = range_cases.make_sequence(W, H, bd, **kw)
        ref = oracle_lib.RefReplay(simd=True, constrained_intra=kw.get("constrained_intra", False), check_avail=True)
        ref.upload_slot(5, pics[0].params, planes)
        for i, p in enumerate(pics):
            p.c.params.stop_after_stage = capi.STAGE_RECON
            try:
                ref.reconstruct(p)
            except oracle_lib.AvailMismatch as e:
                raise AssertionError(f"{name} pic {i}: {e}") from None
            finally:
                p.c.params.stop_after_stage = 0
        ref.close()
