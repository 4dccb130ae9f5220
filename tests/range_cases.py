"""The edges of what a picture record may carry, as one shared case list: 4:0:0, 9 / 11 / 12 bit and unequal luma / chroma
depths, QP' from 0 to 51 + QpBdOffset, deblocking and chroma QP offsets at +-12, explicit weights and offsets at the ends of
their range, MVs anywhere in int16, SAO offsets at the legal maximum, the intra-smoothing / boundary-filter / PCM / per-slice
filter switches, intra availability masks with gaps (constrained intra prediction in P / B pictures, many slices).
test_cpu_range_edges.py pins the oracle to the reference on every case and test_gpu_range_edges.py the
engine to the oracle.

Every case carries the checks that prove its edge is present in the generated records, so that the list cannot quietly turn
into the easy cases (test_cpu_range_edges.py::test_every_case_reaches_its_edges)."""
from collections import namedtuple

import numpy as np

from libde265_b200 import capi, synth

Case = namedtuple("Case", "id W H bd kw checks")


def make_sequence(W, H, bd, pb_intra_frac=None, **kw):
    """Reference planes (uploaded to slot 5) and the I -> P -> B -> weighted B pictures of the parity tests' sequence.
    ``pb_intra_frac``: intra_frac of the P / B pictures (the I picture stays all intra)."""
    planes = synth.random_planes(W, H, bd, 99, bit_depth_chroma=kw.get("bit_depth_chroma"), chroma_format_idc=kw.get("chroma_format_idc", 1))
    pb = {} if pb_intra_frac is None else dict(intra_frac=pb_intra_frac)
    pics = [synth.make_picture(W, H, "I", seed=11, dst_slot=0, bit_depth=bd, **kw),
            synth.make_picture(W, H, "P", seed=12, dst_slot=1, ref_slots=(0, 5), bit_depth=bd, **pb, **kw),
            synth.make_picture(W, H, "B", seed=13, dst_slot=2, ref_slots=(0, 1, 5), bit_depth=bd, **pb, **kw),
            synth.make_picture(W, H, "B", seed=14, dst_slot=3, ref_slots=(0, 1, 2), weighted=True, bit_depth=bd, **pb, **kw)]
    return planes, pics


# ---- gaps in intra availability masks (b200_tu.avail: left groups from bit 0 down the column, corner bit 16, top groups from
# bit 17 along the row; q = nT / 4 groups per side belong to the TU's own column / row, the next q to its bottom-left /
# top-right reach) ----
GAP_CLASSES = ("own_partial", "corner_missing", "reach_gap", "outer_only", "corner_only", "none_off_origin")
SIZE_KINDS = ("4", "8y", "8c", "16", "32")


def gap_class_counts(tus):
    """{(class, size kind): number of intra TUs} over the TU records.  Classes: a partly available own column or row; own
    column and row available but the corner missing; a reach that is not available up to a point from the inner end (so the
    substitution is no clamp); own row missing with the top-right reach present, or own column missing with the bottom-left
    present; only the corner; nothing available away from the picture origin.  Extra keys: ("8_top3_only", kind), an 8x8 TU
    whose only available group is top group 3 (the 33rd border sample rides in its own register on the GPU), and
    ("32_carry", "32"), a 32x32 TU that is no clamp and misses a sample at the start of a 32-sample scan chunk (s = 32, 64,
    96, 128) while an earlier sample is available, so the chunk starts from the carried value."""
    out = {}
    for tu in tus[(tus["flags"] & capi.TU_INTRA) != 0]:
        kind = {2: "4", 3: "8c" if tu["cidx"] else "8y", 4: "16", 5: "32"}[int(tu["log2_size"])]
        for c in tu_gap_classes(tu):
            out[(c, kind)] = out.get((c, kind), 0) + 1
    return out


def tu_gap_classes(tu):
    """The gap classes of one intra TU record (see gap_class_counts)."""
    log2, av = int(tu["log2_size"]), int(tu["avail"])
    nT, q = 1 << log2, 1 << (log2 - 2)
    g = (1 << q) - 1
    lo, bl, co = av & g, (av >> q) & g, (av >> capi.AVAIL_CORNER_BIT) & 1
    to, tr = (av >> capi.AVAIL_TOP_BIT0) & g, (av >> (capi.AVAIL_TOP_BIT0 + q)) & g
    cls = []
    if 0 < lo < g or 0 < to < g:
        cls.append("own_partial")
    if lo == g and to == g and not co:
        cls.append("corner_missing")
    if (bl & (bl + 1)) or (tr & (tr + 1)):
        cls.append("reach_gap")
    if (to == 0 and tr) or (lo == 0 and bl):
        cls.append("outer_only")
    if av == 1 << capi.AVAIL_CORNER_BIT:
        cls.append("corner_only")
    if av == 0 and (tu["x"], tu["y"]) != (0, 0):
        cls.append("none_off_origin")
    if nT == 8 and av == 1 << (capi.AVAIL_TOP_BIT0 + 3):
        cls.append("8_top3_only")
    if nT == 32 and not (lo == g and to == g and co and "reach_gap" not in cls):
        # scan sample s -> availability; chunk starts s = 32 (left row 31), 64 (corner), 96 (top column 31), 128 (top column 63)
        def avail_at(s):
            i = s - 64
            return (av >> ((-i - 1) >> 2)) & 1 if i < 0 else co if i == 0 else (av >> (capi.AVAIL_TOP_BIT0 + ((i - 1) >> 2))) & 1
        if any(not avail_at(s) and any(avail_at(e) for e in range(s)) for s in (32, 64, 96, 128)):
            cls.append("32_carry")
    return cls


# ---- checks: (description, predicate over the sequence's pictures) ----
def _tus(pics):
    return np.concatenate([p.tus for p in pics])


def no_chroma_tus():
    return "no chroma TU and no chroma PCM", lambda pics: len(_tus(pics)) > 0 and (_tus(pics)["cidx"] == 0).all()


def tu_qp(cidx, qp):
    def f(pics):
        t = _tus(pics)
        return ((t["cidx"] == cidx) & ((t["flags"] & capi.TU_CBF) != 0) & ((t["flags"] & capi.TU_BYPASS) == 0) & (t["qp"] == qp)).any()
    return f"a coded plane-{cidx} TU with qp' = {qp}", f


def qpy_min(v):
    return f"QpY {v} in the qp map", lambda pics: any((p.qp_map == v).any() for p in pics)


def weights_hit(*vals):
    return f"weights {vals} occur on luma and chroma", lambda pics: all(
        (p.weights["w"][:, :, 0] == v).any() and (p.weights["w"][:, :, 1:] == v).any() for p in pics[3:] for v in vals)


def offsets_hit(bd_y, bd_c):
    def f(pics):
        o = pics[3].weights["o"]
        return all((o[:, :, 0] == v * (1 << (bd_y - 8))).any() and (o[:, :, 1:] == v * (1 << (bd_c - 8))).any() for v in (-128, 127))
    return f"offsets -128 / 127 << (bd - 8) per plane ({bd_y}/{bd_c} bit)", f


def log2wd(bd_y, bd_c):
    def f(pics):
        w = pics[3].weights
        return (w["log2wd_luma"] >= max(2, 14 - bd_y)).all() and (w["log2wd_chroma"] >= max(2, 14 - bd_c)).all() and \
            (w["log2wd_chroma"] - max(2, 14 - bd_c) < 8).all() and (w["log2wd_luma"] - max(2, 14 - bd_y) < 8).all()
    return "log2wd per plane with the plane's shift1", f


def mv_hit(*vals):
    return f"MV components {vals} occur", lambda pics: all(any((p.pus["mv"] == v).any() for p in pics if len(p.pus)) for v in vals)


def mv_past_rim(W, H):
    def f(pics):
        pu = np.concatenate([p.pus for p in pics[1:]])
        x0 = pu["x"].astype(np.int64)[:, None] + (pu["mv"][:, :, 0].astype(np.int64) >> 2) - 3
        y0 = pu["y"].astype(np.int64)[:, None] + (pu["mv"][:, :, 1].astype(np.int64) >> 2) - 3
        return (x0 == -synth._PAD_X - 1).any() or (x0 == W + synth._PAD_X - 22).any() or (y0 == -synth._PAD_Y - 1).any() or \
            (y0 == H + synth._PAD_Y - 22).any()
    return "an MC window one sample past the reference border's rim", f


def sao_max(bd_y, bd_c, chroma=True):
    def f(pics):
        ok = True
        for c, bd in enumerate((bd_y, bd_c, bd_c)[:3 if chroma else 1]):
            m = ((1 << (min(bd, 10) - 5)) - 1) << max(0, bd - 10)
            a = [np.abs(p.ctbs["sao_offset"][:, c].astype(np.int64)) for p in pics]
            ok &= any((x == m).any() for x in a) and all((x <= m).all() for x in a)
        return ok
    return f"SAO offsets up to and at +-((1 << (min(bd, 10) - 5)) - 1) << (bd - 10) on every plane ({bd_y}/{bd_c} bit)", f


def sao_band():
    return "band-offset CTBs", lambda pics: any(((p.ctbs["sao_type"] & 3) == 1).any() for p in pics)


def pic_flag(flag, on=True, name=""):
    return f"picture flag {name} {'set' if on else 'clear'}", lambda pics: all(bool(p.params.flags & flag) == on for p in pics)


def slice_flag_mix(flag, name):
    def f(pics):
        fl = np.concatenate([p.slices["flags"] for p in pics]) & flag
        return (fl != 0).any() and (fl == 0).any()
    return f"slices with and without {name}", f


def slices_all(flag, name):
    return f"every slice has {name}", lambda pics: all((p.slices["flags"] & flag != 0).all() for p in pics)


def lf_offsets(beta, tc):
    return f"slice beta / tc offsets {beta} / {tc}", lambda pics: all(((p.slices["beta_offset"] == beta) & (p.slices["tc_offset"] == tc)).all()
                                                                      for p in pics)


def chroma_qp_offsets(cb, cr):
    return f"pps cb / cr qp offsets {cb} / {cr}", lambda pics: all((p.params.pps_cb_qp_offset, p.params.pps_cr_qp_offset) == (cb, cr) for p in pics)


def pcm_in_nofilt():
    def f(pics):
        for p in pics:
            for t in p.tus[(p.tus["flags"] & capi.TU_PCM) != 0]:
                if t["cidx"] == 0 and p.nofilt_map[(t["y"] >> 3) * ((p.params.width + 7) // 8) + (t["x"] >> 3)]:
                    return True
        return False
    return "a PCM CU in the no-filter map", f


def tu_flag(flag, name, intra=None):
    def f(pics):
        t = _tus(pics)
        m = (t["flags"] & flag) != 0
        if intra is not None:
            m &= ((t["flags"] & capi.TU_INTRA) != 0) == intra
        return m.any()
    return f"TUs with {name}", f


def nbf_rdpcm():
    def f(pics):
        t = _tus(pics)
        intra_bypass = ((t["flags"] & capi.TU_INTRA) != 0) & ((t["flags"] & capi.TU_BYPASS) != 0)
        return (intra_bypass & ((t["flags"] & (capi.TU_RDPCM_H | capi.TU_RDPCM_V)) != 0)).any() and \
            (intra_bypass == (intra_bypass & ((t["flags"] & capi.TU_NO_BOUNDARY_FILTER) != 0))).all()
    return "implicit RDPCM and no boundary filter on every intra bypass TU", f


def bs_zero_in_disabled_slices():
    def f(pics):
        seen = False
        for p in pics:
            S = 1 << p.params.log2_ctb_size
            w4, wctb = (p.params.width + 3) // 4, (p.params.width + S - 1) // S
            bs = p.bs_map.reshape(-1, w4)
            ys, xs = np.mgrid[0:bs.shape[0], 0:w4]
            sl = p.ctbs["slice_idx"][(xs * 4 // S) + (ys * 4 // S) * wctb]
            off = (p.slices["flags"][sl] & capi.SLICE_DEBLOCK_DISABLED) != 0
            if off.any() and (bs[off] != 0).any():
                return False
            seen |= bool(off.any()) and bool((bs[~off] != 0).any() or (~off).sum() == 0)
        return seen
    return "slices with deblocking off have bS 0 on their edges", f


GEOMETRY_FORBIDS = {("own_partial", "4"), ("own_partial", "8y"), ("reach_gap", "4"), ("reach_gap", "8y")}  # one 8x8 CU per 8 luma samples


def gap_counts(pics):
    cnt = {}
    for p in pics:
        for k, v in gap_class_counts(p.tus).items():
            cnt[k] = cnt.get(k, 0) + v
    return cnt


def gaps(kinds=SIZE_KINDS, classes=GAP_CLASSES, skip=()):
    """Every gap class at every TU size kind, except where the geometry rules it out (a 4x4 / 8x8 luma TU's own column, own
    row and reach each lie in one 8x8 CU) and the listed (class, kind) pairs that the case's sizes make rare."""
    want = [(c, k) for c in classes for k in kinds if (c, k) not in GEOMETRY_FORBIDS and (c, k) not in skip]

    def f(pics):
        cnt = gap_counts(pics)
        return all(cnt.get(w, 0) > 0 for w in want)
    return f"intra TUs with availability gaps of each class {want}", f


def top3_only():
    return "an 8x8 TU whose only available group is top group 3", lambda pics: any(k[0] == "8_top3_only" for k in gap_counts(pics))


def carry32():
    return "a 32x32 TU whose substitution carries a value into a 32-sample chunk", lambda pics: gap_counts(pics).get(("32_carry", "32"), 0) > 0


def smoothed_32_on_substituted_border(n):
    def f(pics):
        t = _tus(pics)
        t = t[((t["flags"] & capi.TU_INTRA) != 0) & (t["log2_size"] == 5) & (t["cidx"] == 0)]
        g = np.uint64(0xFF)
        av = t["avail"].astype(np.uint64)
        own = ((av & g) == g) & (((av >> np.uint64(capi.AVAIL_CORNER_BIT)) & np.uint64(1)) == 1) & (((av >> np.uint64(capi.AVAIL_TOP_BIT0)) & g) == g)
        m = t["intra_mode"].astype(np.int64)
        smoothed = (m != 1) & (np.minimum(np.abs(m - 26), np.abs(m - 10)) > 0)
        return int((~own & smoothed).sum()) >= n
    return f"{n} 32x32 luma TUs with a smoothed mode and a gap in their own column, corner or row", f


def ctb_grid(log2, W, H):
    return f"CTB {1 << log2} on a {W}x{H} picture", lambda pics: all(p.params.log2_ctb_size == log2 and (p.params.width, p.params.height) == (W, H)
                                                                     for p in pics)


# ---- the case list: (id, W, H, bd, make_picture kwargs, checks) ----
_PCM = dict(special_frac=0.12, cbf_prob=0.9)
_CIP = dict(constrained_intra=True, pb_intra_frac=0.5)

CASES = [
    Case("mono8_ctb64", 192, 128, 8, dict(chroma_format_idc=0, **_PCM), [no_chroma_tus(), ctb_grid(6, 192, 128), tu_flag(capi.TU_PCM, "PCM")]),
    Case("mono8_ctb16", 208, 120, 8, dict(chroma_format_idc=0, log2_ctb=4, size_area=(0.0, 0.0, 0.5, 0.5)), [no_chroma_tus(), ctb_grid(4, 208, 120)]),
    Case("mono10_sao_max", 192, 128, 10, dict(chroma_format_idc=0, sao_offset="max", weight_range="spec", **_PCM),
         [no_chroma_tus(), sao_max(10, 10, chroma=False), sao_band(), tu_flag(capi.TU_PCM, "PCM")]),
    Case("mono8_200x136", 200, 136, 8, dict(chroma_format_idc=0, extreme_mv_frac=0.5), [no_chroma_tus(), mv_hit(-32768, 32767)]),
    Case("mono10_1288x8", 1288, 8, 10, dict(chroma_format_idc=0), [no_chroma_tus(), ctb_grid(6, 1288, 8)]),
    Case("bd9", 192, 128, 9, dict(sao_offset="max", weight_range="spec"), [sao_max(9, 9), weights_hit(-128, 255), offsets_hit(9, 9)]),
    Case("bd11", 192, 128, 11, dict(sao_offset="max", weight_range="spec", **_PCM), [sao_max(11, 11), sao_band(), offsets_hit(11, 11)]),
    Case("bd12", 192, 128, 12, dict(sao_offset="max", weight_range="spec", **_PCM), [sao_max(12, 12), weights_hit(-128, 255), offsets_hit(12, 12)]),
    Case("bd12_200x136", 200, 136, 12, dict(extreme_mv_frac=0.5, sao_offset="max"), [mv_hit(-32768, 32767), mv_past_rim(200, 136)]),
    Case("bd12_1288x8", 1288, 8, 12, dict(), [ctb_grid(6, 1288, 8)]),
    Case("bd10_chroma12", 192, 128, 10, dict(bit_depth_chroma=12, sao_offset="max", weight_range="spec", **_PCM),
         [sao_max(10, 12), offsets_hit(10, 12), log2wd(10, 12), tu_flag(capi.TU_PCM, "PCM")]),
    Case("bd12_chroma9", 192, 128, 12, dict(bit_depth_chroma=9, sao_offset="max", weight_range="spec", qp_range=(-9, 51), **_PCM),
         [sao_max(12, 9), offsets_hit(12, 9), log2wd(12, 9), qpy_min(-9)]),
    Case("qp_low8", 192, 128, 8, dict(qp_range=(0, 4)), [tu_qp(0, 0), qpy_min(0)]),
    Case("qp_high8", 192, 128, 8, dict(qp_range=(47, 51), chroma_qp_offsets=(12, 12)), [tu_qp(0, 51), tu_qp(1, 51)]),
    Case("qp_low12", 192, 128, 12, dict(qp_range=(-24, -18), chroma_qp_offsets=(-12, -12)), [tu_qp(0, 0), qpy_min(-24), tu_qp(1, 0)]),
    Case("qp_high12", 192, 128, 12, dict(qp_range=(45, 51), chroma_qp_offsets=(12, 12)), [tu_qp(0, 51 + 24), tu_qp(2, 51 + 24)]),
    Case("lf_offsets_plus12", 192, 128, 8, dict(qp_range=(40, 51), lf_offsets=(12, 12), chroma_qp_offsets=(12, -12)),
         [lf_offsets(12, 12), chroma_qp_offsets(12, -12), tu_qp(0, 51)]),
    Case("lf_offsets_minus12", 192, 128, 10, dict(qp_range=(30, 51), lf_offsets=(-12, -12), chroma_qp_offsets=(-12, 12)),
         [lf_offsets(-12, -12), chroma_qp_offsets(-12, 12)]),
    Case("weights_spec8", 192, 128, 8, dict(weight_range="spec"), [weights_hit(-128, 255), offsets_hit(8, 8), log2wd(8, 8)]),
    Case("extreme_mv8", 192, 128, 8, dict(extreme_mv_frac=0.5, weight_range="spec"), [mv_hit(-32768, 32767), mv_past_rim(192, 128)]),
    Case("extreme_mv10", 192, 128, 10, dict(extreme_mv_frac=0.5), [mv_hit(-32768, 32767), mv_past_rim(192, 128)]),
    Case("smoothing_off_deblock_off", 192, 128, 8, dict(intra_smoothing_off=True, strong_smoothing=False, n_slices=3, slice_deblock_off_frac=1.0),
         [pic_flag(capi.PIC_INTRA_SMOOTHING_OFF, True, "INTRA_SMOOTHING_OFF"), pic_flag(capi.PIC_STRONG_INTRA_SMOOTHING, False, "STRONG_INTRA_SMOOTHING"),
          slices_all(capi.SLICE_DEBLOCK_DISABLED, "deblocking disabled"), ("every bS is 0", lambda pics: all((p.bs_map == 0).all() for p in pics))]),
    Case("no_strong_smoothing10", 256, 192, 10, dict(strong_smoothing=False, size_area=(0.2, 0.6, 0.1, 0.1)),
         [pic_flag(capi.PIC_STRONG_INTRA_SMOOTHING, False, "STRONG_INTRA_SMOOTHING")]),
    Case("bypass_nbf_pcm_lf_off", 192, 128, 8, dict(special_frac=0.2, cbf_prob=0.9, no_bfilter_on_bypass=True, pcm_lf_disable=True),
         [nbf_rdpcm(), pcm_in_nofilt(), pic_flag(capi.PIC_PCM_LF_DISABLE, True, "PCM_LF_DISABLE")]),
    Case("bypass_nbf_pcm_lf_off_12_10", 192, 128, 12, dict(bit_depth_chroma=10, special_frac=0.2, cbf_prob=0.9, no_bfilter_on_bypass=True,
                                                          pcm_lf_disable=True, intra_smoothing_off=True), [nbf_rdpcm(), pcm_in_nofilt()]),
    Case("tiles_slice_filter_flags", 448, 256, 8, dict(tiles=(3, 2), lf_across_tiles=False, n_slices=6, slice_deblock_off_frac=0.5, slice_sao_off_frac=0.5),
         [slice_flag_mix(capi.SLICE_DEBLOCK_DISABLED, "deblocking disabled"), slice_flag_mix(capi.SLICE_SAO_LUMA, "SAO luma"),
          slice_flag_mix(capi.SLICE_SAO_CHROMA, "SAO chroma"), bs_zero_in_disabled_slices()]),
    Case("mono8_tiles_slice_flags", 448, 256, 8, dict(chroma_format_idc=0, tiles=(2, 3), n_slices=5, slice_deblock_off_frac=0.4, slice_sao_off_frac=0.5),
         [no_chroma_tus(), slice_flag_mix(capi.SLICE_SAO_LUMA, "SAO luma"), bs_zero_in_disabled_slices()]),
    Case("skip_sao10", 192, 128, 10, dict(skip_sao=True, sao_offset="max"), [pic_flag(capi.PIC_SKIP_SAO, True, "SKIP_SAO")]),
    # Constrained intra prediction: half the CUs of the P / B pictures are intra, and their inter neighbours are unavailable, so
    # gaps fall anywhere in the border (own column, corner, own row, either reach).  The last case is the source of gaps without
    # it: slice boundaries between the CTB above and the one above-right / above-left.
    Case("cip8_ctb64", 448, 256, 8, dict(size_area=(0.0, 0.5, 0.25, 0.25), **_CIP),
         [gaps(skip=(("corner_missing", "32"), ("corner_only", "32"))), top3_only(), carry32()]),
    Case("cip8_ctb32_small_cus", 320, 192, 8, dict(log2_ctb=5, size_area=(0.0, 0.2, 0.4, 0.4), **_CIP),
         [gaps(skip=(("corner_missing", "32"), ("corner_only", "32"))), top3_only(), carry32()]),
    Case("cip8_ctb16", 208, 120, 8, dict(log2_ctb=4, size_area=(0.0, 0.0, 0.5, 0.5), **_CIP),
         [ctb_grid(4, 208, 120), gaps(kinds=("4", "8y", "8c", "16"), skip=(("corner_only", "8c"), ("corner_only", "16")))]),
    Case("cip10_tiles_slices", 448, 256, 10, dict(tiles=(3, 2), lf_across_tiles=False, n_slices=5, size_area=(0.0, 0.4, 0.3, 0.3), **_CIP),
         [gaps(skip=(("corner_missing", "32"), ("corner_only", "32"))), top3_only(), carry32()]),
    Case("cip12_chroma9", 320, 192, 12, dict(bit_depth_chroma=9, size_area=(0.0, 0.4, 0.3, 0.3), **_CIP),
         [gaps(skip=(("corner_missing", "32"), ("corner_only", "8c"), ("corner_only", "16"), ("corner_only", "32"))), carry32()]),
    Case("cip_mono8", 320, 192, 8, dict(chroma_format_idc=0, size_area=(0.0, 0.5, 0.25, 0.25), **_CIP),
         [no_chroma_tus(), gaps(kinds=("4", "8y", "16", "32"), skip=(("corner_missing", "32"), ("corner_only", "32"))), carry32()]),
    Case("cip8_smoothing_off", 320, 192, 8, dict(intra_smoothing_off=True, size_area=(0.0, 0.5, 0.25, 0.25), **_CIP),
         [pic_flag(capi.PIC_INTRA_SMOOTHING_OFF, True, "INTRA_SMOOTHING_OFF"), gaps(skip=(("corner_missing", "32"),)), top3_only(), carry32()]),
    Case("cip8_strong_smoothing", 448, 256, 8, dict(size_area=(0.3, 0.5, 0.1, 0.1), **_CIP),
         [pic_flag(capi.PIC_STRONG_INTRA_SMOOTHING, True, "STRONG_INTRA_SMOOTHING"), gaps(), carry32(), smoothed_32_on_substituted_border(20)]),
    Case("intra8_24_slices", 416, 240, 8, dict(log2_ctb=5, n_slices=24, pb_intra_frac=1.0),
         [gaps(classes=("corner_missing", "outer_only", "none_off_origin"), skip=(("corner_missing", "8c"), ("outer_only", "32"))), carry32()]),
]
CIP_CASE_IDS = [c.id for c in CASES if c.kw.get("constrained_intra")]

CASE_IDS = [c.id for c in CASES]
BY_ID = {c.id: c for c in CASES}
