"""The oracle against the reference's own reconstruction functions (oracle/_ref/libref_replay.so, scalar and SIMD tables) on the
edges of what a record may carry (range_cases.py): every case as an I -> P -> B -> weighted B sequence, stage by stage.
Without oracle/_ref the oracle's pictures are checked against the stored digests of what the replay returned
(tests/golden/ref_pins.json), as in test_cpu_ref_replay.py."""
import pytest

import oracle_lib
import ref_pins
import range_cases
from libde265_b200 import capi
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
    orc, ref = oracle_lib.Oracle(), oracle_lib.RefReplay(simd=simd) if HAVE_REF else None
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
