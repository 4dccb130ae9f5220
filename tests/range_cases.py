"""The edges of what a picture record may carry, as one shared case list: 4:0:0, 9 / 11 / 12 bit and unequal luma / chroma
depths, QP' from 0 to 51 + QpBdOffset, deblocking and chroma QP offsets at +-12, explicit weights and offsets at the ends of
their range, MVs anywhere in int16, SAO offsets at the legal maximum, the intra-smoothing / boundary-filter / PCM / per-slice
filter switches.  test_cpu_range_edges.py pins the oracle to the reference on every case and test_gpu_range_edges.py the
engine to the oracle.

Every case carries the checks that prove its edge is present in the generated records, so that the list cannot quietly turn
into the easy cases (test_cpu_range_edges.py::test_every_case_reaches_its_edges)."""
from collections import namedtuple

import numpy as np

from libde265_b200 import capi, synth

Case = namedtuple("Case", "id W H bd kw checks")


def make_sequence(W, H, bd, **kw):
    """Reference planes (uploaded to slot 5) and the I -> P -> B -> weighted B pictures of the parity tests' sequence."""
    planes = synth.random_planes(W, H, bd, 99, bit_depth_chroma=kw.get("bit_depth_chroma"), chroma_format_idc=kw.get("chroma_format_idc", 1))
    pics = [synth.make_picture(W, H, "I", seed=11, dst_slot=0, bit_depth=bd, **kw),
            synth.make_picture(W, H, "P", seed=12, dst_slot=1, ref_slots=(0, 5), bit_depth=bd, **kw),
            synth.make_picture(W, H, "B", seed=13, dst_slot=2, ref_slots=(0, 1, 5), bit_depth=bd, **kw),
            synth.make_picture(W, H, "B", seed=14, dst_slot=3, ref_slots=(0, 1, 2), weighted=True, bit_depth=bd, **kw)]
    return planes, pics


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


def ctb_grid(log2, W, H):
    return f"CTB {1 << log2} on a {W}x{H} picture", lambda pics: all(p.params.log2_ctb_size == log2 and (p.params.width, p.params.height) == (W, H)
                                                                     for p in pics)


# ---- the case list: (id, W, H, bd, make_picture kwargs, checks) ----
_PCM = dict(special_frac=0.12, cbf_prob=0.9)

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
]

CASE_IDS = [c.id for c in CASES]
BY_ID = {c.id: c for c in CASES}
