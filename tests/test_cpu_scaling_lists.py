"""Scaling lists on the CPU: the oracle against the reference's own reconstruction functions (oracle/_ref/libref_replay.so,
scalar and SIMD tables) on every case of scaling_cases.py, stage by stage, and without oracle/_ref against the stored digests
of what the replay returned (tests/golden/ref_pins.json, see ref_pins.py); the cases against their edges; and the oracle's
dequantisation and transform skip against a plain big-integer restatement that needs no reference build."""
import numpy as np
import pytest

import oracle_lib
import ref_pins
import scaling_cases
from libde265_b200 import capi, synth
from test_cpu_ref_replay import same

HAVE_REF = oracle_lib.ref_replay_lib() is not None
pins = ref_pins.make_fixture(HAVE_REF)


@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_every_case_reaches_its_edges(b200lib, case):
    """The case's records carry every edge its checks name, and the planner (b200_plan_picture_host) sends TUs with a matrix
    down every residual path: the warp / 8x8 / 4x4 classes of k_residual and the intra TUs of k_intra at every size."""
    c = scaling_cases.BY_ID[case]
    _, pics = scaling_cases.make_sequence(c)
    missing = [desc for desc, ok in c.checks if not ok(pics)]
    paths = scaling_cases.planner_paths(b200lib, pics)
    missing += [f"TUs with a matrix on residual path {w}" for w in scaling_cases.planner_wants(c) if not paths.get(w)]
    assert not missing, f"{case}: the generated records lack {missing}"


@pytest.mark.parametrize("simd", [False, True])
@pytest.mark.parametrize("case", scaling_cases.CASE_IDS)
def test_replay_matches_oracle_with_scaling_lists(pins, case, simd):
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
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


def test_default_lists_follow_the_spec():
    """Spot values of Tables 7-5 / 7-6 after the 7.4.5 expansion: flat 4x4, the 8x8 intra / inter corners 115 / 91, symmetric
    matrices, the 16x16 / 32x32 ones replicated from the 8x8 list with DC 16."""
    f = synth.default_scaling_factors()
    mats = {(n, m): f[b + m * n * n:b + (m + 1) * n * n].reshape(n, n) for n, b in synth.SCALING_SIZES for m in range(6 if n < 32 else 2)}
    assert all((mats[(4, m)] == 16).all() for m in range(6))
    for n in (8, 16, 32):
        for m in range(6 if n < 32 else 2):
            a, inter = mats[(n, m)], (m >= 3 if n < 32 else m == 1)
            assert (a == a.T).all() and a[0, 0] == 16 and a[-1, -1] == (91 if inter else 115)
            if n > 8:
                assert (a[::n // 8, ::n // 8][1:, 1:] == mats[(8, 3 if inter else 0)][1:, 1:]).all()
    assert mats[(8, 0)][0].tolist() == [16, 16, 16, 16, 17, 18, 21, 24] and mats[(8, 0)][7].tolist() == [24, 25, 29, 36, 47, 65, 88, 115]
    assert [mats[(8, 3)][7 - k, k] for k in range(8)] == [24] * 8 and mats[(8, 3)][7].tolist() == [24, 25, 28, 33, 41, 54, 71, 91]


# ---- the oracle against a plain restatement: one transform-skip TU on a mid-grey inter prediction ----
def _one_tu_picture(bd_y, bd_c, cidx, log2, qp, rdpcm, scaling, levels):
    """A 64x64 P picture whose one PU copies slot 7 (mid-grey) and whose one TU (inter, transform skip, its matrix) carries
    `levels` ({position: level})."""
    base = synth.make_picture(64, 64, "P", seed=3, dst_slot=1, ref_slots=(7,), bit_depth=bd_y, bit_depth_chroma=bd_c, deblock=False, sao=False,
                              scaling_list=True)
    pu = np.zeros(1, synth.PU_DT)
    pu["w"], pu["h"], pu["flags"], pu["ref_slot"] = 64, 64, capi.PU_PRED_L0, (7, -1)
    flags = capi.TU_CBF | capi.TU_TSKIP | capi.TU_SCALING_LIST | capi.TU_INTER_MATRIX | rdpcm
    tu = np.array([(0, 0, log2, cidx, flags, 0, qp, len(levels), 0, 0)], synth.TU_DT)
    co = np.zeros(len(levels), synth.CO_DT)
    co["pos"], co["level"] = list(levels), list(levels.values())
    p = synth.SynthPicture(base.params, pu, np.zeros(0, synth.WT_DT), tu, co, base.slices, base.ctbs, base.bs_map, base.qp_map, base.nofilt_map, scaling)
    p.c.params.stop_after_stage = capi.STAGE_RECON
    return p


def _restated(bd, log2, qp, rdpcm, fac, levels, seen):
    """transform.cc:489-525 (dequantisation with a matrix, the low 32 bits clipped to int16) and fallback-dct.cc
    transform_skip_residual / rdpcm (tsShift = 5 + log2(nT), bdShift = 20 - BitDepth) on Python integers, added to mid-grey and
    clipped to [0, 2^bd).  `seen` collects "beyond int32" when a dequantised value needs the truncation."""
    nT = 1 << log2
    d = [0] * (nT * nT)
    for pos, lv in levels.items():
        d[pos] = scaling_cases.dequant_reference(lv, int(fac[pos]), qp, bd, log2)
        if not -(1 << 31) <= scaling_cases.dequant_exact(lv, int(fac[pos]), qp, bd, log2) < (1 << 31):
            seen.add("beyond int32")
    sh = 20 - bd
    r = [[((d[x + y * nT] << (5 + log2)) + (1 << (sh - 1))) >> sh for x in range(nT)] for y in range(nT)]
    for y in range(nT):
        for x in range(nT):
            if rdpcm == capi.TU_RDPCM_H and x:
                r[y][x] += r[y][x - 1]
            elif rdpcm == capi.TU_RDPCM_V and y:
                r[y][x] += r[y - 1][x]
    mid = 1 << (bd - 1)
    return np.array([[min((1 << bd) - 1, max(0, mid + v)) for v in row] for row in r], np.int64)


def _levels(rng, nT, fac, qp, bd, log2):
    """Levels at about a third of the positions, each aimed at a residual inside the sample range, past its top or past its
    bottom, or at the int16 ends; the level that lands nearest the aim (a level of 0 becomes +-1)."""
    out = {}
    for pos in rng.choice(nT * nT, max(3, nT * nT // 3), replace=False).tolist():
        step = (int(fac[pos]) * scaling_cases.LEVEL_SCALE[qp % 6] << (qp // 6)) / (1 << (bd + log2 - 5))  # dequantised value per level
        step *= 2.0 ** (5 + log2 - (20 - bd))  # residual per level
        aim = [rng.integers(-(1 << bd) // 3, (1 << bd) // 3 + 1), (1 << bd) + 40, -(1 << bd) - 40, None][int(rng.integers(0, 4))]
        lv = int(rng.choice([-32768, 32767])) if aim is None else int(np.clip(round(int(aim) / step), -32768, 32767))
        out[pos] = lv or int(rng.choice([-1, 1]))
    return out


@pytest.mark.parametrize("bd_y,bd_c", [(8, 8), (9, 9), (10, 10), (12, 12), (10, 12), (12, 9)])
def test_oracle_dequant_and_transform_skip_restated(bd_y, bd_c):
    """One-TU inter pictures at STAGE_RECON over a mid-grey prediction: transform skip with a matrix of factors over 1..255 at
    every size and plane, qP' from 0 to 51 + QpBdOffset, plain and both RDPCM directions.  The oracle's samples equal the
    restatement's exactly, and the restated samples cover the inside of the sample range and both of its ends, from levels that
    include dequantised values beyond the int32 range."""
    rng = np.random.default_rng(bd_y * 16 + bd_c)
    scaling = synth.max_scaling_factors(rng)
    orc = oracle_lib.Oracle()
    seen = set()
    for cidx in (0, 1, 2):
        bd = bd_c if cidx else bd_y
        for log2 in (2, 3, 4, 5) if cidx == 0 else (2, 3, 4):
            nT, (_, b) = 1 << log2, synth.SCALING_SIZES[log2 - 2]
            fac = scaling[b + scaling_cases.matrix_id(log2, cidx, True) * nT * nT:][:nT * nT]
            for qp in (0, 5, 22, 39, 51 + 6 * (bd - 8)):
                for rdpcm in (0, capi.TU_RDPCM_H, capi.TU_RDPCM_V):
                    levels = _levels(rng, nT, fac, qp, bd, log2)
                    p = _one_tu_picture(bd_y, bd_c, cidx, log2, qp, rdpcm, scaling, levels)
                    orc.fill_slot(7, p.params, 1 << (bd_y - 1), 1 << (bd_c - 1))
                    orc.reconstruct(p)
                    got = orc.read_slot(1, p.params)[cidx][:nT, :nT].astype(np.int64)
                    want = _restated(bd, log2, qp, rdpcm, fac, levels, seen)
                    d = np.argwhere(got != want)
                    assert not len(d), (f"plane {cidx} {nT}x{nT} qP' {qp} rdpcm {rdpcm}: {len(d)} samples differ, first at (x={d[0][1]}, y={d[0][0]}): "
                                        f"oracle {got[tuple(d[0])]} != restated {want[tuple(d[0])]}")
                    seen |= {"zero" if v == 0 else "max" if v == (1 << bd) - 1 else "inside" for v in want.reshape(-1).tolist()}
    orc.close()
    assert seen == {"zero", "max", "inside", "beyond int32"}, seen


# ---- one rule for the flag: the factors are used only under PIC_SCALING_LIST ----
def flag_cleared(p, keep_factors):
    """The picture with PIC_SCALING_LIST clear, its TUs still marked with their matrices; the factors kept or NULL."""
    q = synth.SynthPicture(p.params, p.pus, p.weights, p.tus, p.coeffs, p.slices, p.ctbs, p.bs_map, p.qp_map, p.nofilt_map,
                           p.scaling if keep_factors else None)
    q.c.params.flags &= ~capi.PIC_SCALING_LIST
    return q


@pytest.mark.parametrize("case", ["max10", "max8_ctb16"])
def test_factors_without_the_picture_flag_are_ignored(case):
    """A picture whose TUs carry TU_SCALING_LIST, with factors present but PIC_SCALING_LIST clear, reconstructs exactly like the
    same picture with scaling_factors NULL (flat dequantisation), in the oracle and in the reference replay."""
    c = scaling_cases.BY_ID[case]
    planes, pics = scaling_cases.make_sequence(c)
    engines = [oracle_lib.Oracle()] + ([oracle_lib.RefReplay(simd=True)] if HAVE_REF else [])
    for e in engines:
        e.upload_slot(5, pics[0].params, planes)
        for p in pics:
            out = []
            for q in (flag_cleared(p, True), flag_cleared(p, False), p):
                e.reconstruct(q)
                out.append(e.read_slot(p.params.dst_slot, p.params))
            tag = f"{type(e).__name__} {case} slot {p.params.dst_slot}"
            assert all((a == b).all() for a, b in zip(out[0], out[1])), f"{tag}: factors without the picture flag were used"
            assert any((a != b).any() for a, b in zip(out[1], out[2])), f"{tag}: the matrices change nothing"
        e.close()
