"""The in-loop filters branch by branch on the CPU (filter_cases.py): every case reaches its branches, the classifier of the
filter decisions agrees with the oracle sample for sample, its counts over all cases reach every deblocking and SAO branch,
the geometry cases reach every store width of the SAO kernels, and the oracle matches the reference's own filters
(oracle/_ref/libref_replay.so, scalar and SIMD tables) stage by stage on every case.  Without oracle/_ref the oracle's
pictures are checked against the stored digests of what the replay returned (tests/golden/ref_pins.json)."""
import pytest

import filter_cases
import oracle_lib
import ref_pins
from libde265_b200 import capi
from test_cpu_ref_replay import same

HAVE_REF = oracle_lib.ref_replay_lib() is not None
pins = ref_pins.make_fixture(HAVE_REF)

# Every branch must be taken at least N times over all cases; the rarest (the strong filter's clamp deciding p0 / q0) is
# taken about 100 times, so the count does not rest on a lucky seed.
N = 25
BRANCHES = (filter_cases.LUMA_DEBLOCK + filter_cases.STRONG_CLAMP + filter_cases.CHROMA_DEBLOCK + filter_cases.ONE_SIDED + filter_cases.SAO_EDGE +
            filter_cases.SAO_BAND +
            ["luma_weak_p1_clamped", "luma_weak_q1_clamped", "tc_0", "chroma_tc_0", "beta_idx_below_0", "beta_idx_above_51", "tc_idx_below_0",
             "tc_idx_above_53", "chroma_qpi_below_30", "chroma_qpi_table", "chroma_qpi_from_43", "sao_nofilt_Y", "sao_nofilt_C",
             "sao_nofilt_second_block", "sao_unavail_pic_border", "sao_unavail_earlier_slice", "sao_unavail_later_slice", "sao_unavail_tile",
             "sao_quirk"])


def run(case):
    return filter_cases.run_case(filter_cases.BY_ID[case], oracle_lib.Oracle)


@pytest.mark.parametrize("case", filter_cases.CASE_IDS)
def test_every_case_reaches_its_checks(case):
    r = run(case)
    missing = [desc for desc, ok in r.case.checks if not ok(r)]
    assert not missing, f"{case}: the sequence lacks {missing}"


@pytest.mark.parametrize("case", filter_cases.CASE_IDS)
def test_classifier_matches_oracle(case):
    """On pictures deblocked along one direction only (input: the reconstruction), the samples the classifier changes are the
    samples the oracle's deblocking changes, with the same values; the same between the deblocked and the final picture for
    SAO."""
    r = run(case)
    for i, st in enumerate(r.stages):
        for pred, got, base, what in (("pred_v", "deblock_v", "recon", "vertical edges"), ("pred_h", "deblock_h", "recon", "horizontal edges"),
                                      ("pred_sao", "all", "deblock", "SAO")):
            for c, (a, b, x) in enumerate(zip(st[pred], st[got], st[base])):
                moved_a, moved_b = a != x, b != x
                assert (moved_a == moved_b).all(), (f"{case} pic {i} {what} plane {c}: the classifier changes {int(moved_a.sum())} samples, "
                                                    f"the oracle {int(moved_b.sum())}, {int((moved_a != moved_b).sum())} differ")
                assert (a == b).all(), f"{case} pic {i} {what} plane {c}: {int((a != b).sum())} changed samples take other values"


def test_classifier_counts_reach_every_branch():
    total = {}
    for case in filter_cases.CASE_IDS:
        for k, v in run(case).counts.items():
            total[k] = total.get(k, 0) + v
    print("\nfilter branches over all cases:")
    for k in sorted(total):
        print(f"  {k:34s} {total[k]:8d}")
    low = {k: total.get(k, 0) for k in BRANCHES if total.get(k, 0) < N}
    assert not low, f"branches taken fewer than {N} times: {low}"


def test_geometry_cases_reach_every_remainder_and_store_width():
    """At CTB 16, 32 and 64, in 4:2:0 and 4:0:0: every width and height remainder modulo the CTB size.  The store widths of the
    SAO kernels' last groups: k_sao8 (8 bit, CTB 32 / 64) luma 8 and 16, chroma 4, 8, 12 and 16 samples; k_sao 4 and 8."""
    geo = [c for c in filter_cases.CASES if c.id.startswith("geom_")]
    for log2 in (4, 5, 6):
        S = 1 << log2
        for cf in (0, 1):
            cs = [c for c in geo if c.kw["log2_ctb"] == log2 and c.kw["chroma_format_idc"] == cf]
            for dim in ("W", "H"):
                rem = {getattr(c, dim) % S for c in cs}
                assert rem == set(range(0, S, 8)), f"CTB {S}, chroma_format_idc {cf}: {dim} remainders {sorted(rem)}"
    tails = set()
    for c in geo:
        tails |= {t for t in run(c.id).tails if t[0] == "sao" or (c.bd == 8 and c.kw["log2_ctb"] >= 5)}
    want = {("sao8", "Y", 8), ("sao8", "Y", 16)} | {("sao8", "C", n) for n in (4, 8, 12, 16)} | {("sao", "C", 4), ("sao", "C", 8), ("sao", "Y", 8)}
    assert want <= tails, f"store widths not reached: {sorted(want - tails)}"


@pytest.mark.parametrize("case", ["steer8", "steer8_ctb32"])
def test_checks_fail_on_random_planes(case):
    """The steering is what reaches the branches: on the noise of synth.random_planes the same records miss a named check."""
    c = filter_cases.BY_ID[case]
    r = filter_cases.run_case(c._replace(id=f"{case}_random", kw=dict(c.kw, steps="random")), oracle_lib.Oracle)
    assert [desc for desc, ok in c.checks if not ok(r)], f"{case}: every check still holds on random planes"


@pytest.mark.parametrize("simd", [False, True])
@pytest.mark.parametrize("case", filter_cases.CASE_IDS)
def test_replay_matches_oracle_on_the_filter_cases(pins, case, simd):
    c = filter_cases.BY_ID[case]
    planes, pics = filter_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    orc = oracle_lib.Oracle()
    ref = oracle_lib.RefReplay(simd=simd) if HAVE_REF else None
    for e in (orc, ref):
        if e is not None:
            e.upload_slot(5, pics[0].params, planes)
    for i, p in enumerate(pics):
        for st in (capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL):
            p.c.params.stop_after_stage = st
            orc.reconstruct(p)
            if ref is not None:
                ref.reconstruct(p)
            same(pins, ref and ref.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
        p.c.params.stop_after_stage = 0
    orc.close()
    if ref is not None:
        ref.close()
