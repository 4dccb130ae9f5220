"""Scaling lists on every residual path, as one shared case list: 8 / 9 / 10 / 12 bit and unequal luma / chroma depths, 4:0:0,
CTB 16 / 32 / 64, factors over 1..255 (and the spec's default lists), qP' from 0 to 51 + QpBdOffset, transform skip of every
size with RDPCM and rotation, constrained intra prediction (so the intra TUs of P / B pictures carry a matrix too).
test_cpu_scaling_lists.py pins the oracle to the reference on every case and test_gpu_scaling_lists.py the engine to the
oracle.

Every case carries the checks that prove its edge is present in the generated records (computed from the records in numpy),
so that the list cannot quietly turn into the easy cases (test_cpu_scaling_lists.py::test_every_case_reaches_its_edges).
The required ones: every (size, matrix ID) pair the format allows used by a coded coefficient, a coefficient with a factor
>= 128 whose exact dequantised value lies beyond +-32767 (the int16 clip), transform skip with a matrix at every size.  Above
qP' 3 the cases also reach values beyond the int32 range: the reference clips the low 32 bits of the 64-bit value
(transform.cc:522-523 calls Clip3(int, int, int)), and the oracle and the engine follow it."""
from collections import namedtuple

import numpy as np

from libde265_b200 import capi, synth
import range_cases

Case = namedtuple("Case", "id W H bd kw checks")
LEVEL_SCALE = (40, 45, 51, 57, 64, 72)
_BASE = dict(synth.SCALING_SIZES)  # nT -> byte offset of its matrix 0


def matrix_id(log2, cidx, inter):
    """The matrix a TU record selects (transform.cc:489-500): 32x32 TUs 0 (intra) / 1 (inter), smaller ones cIdx (+3 inter)."""
    nT = 1 << log2
    return (0 if nT == 32 else cidx) + ((3 if nT < 32 else 1) if inter else 0)


def matrix_coeffs(p):
    """One row per coefficient of the picture's coded TUs that carry a matrix: dict of numpy arrays log2, cidx, matrix, factor,
    level, qp, bd (the TU plane's bit depth), flags, pos and tu (the TU's index)."""
    t = p.tus
    fl = t["flags"].astype(np.int64)
    sel = np.nonzero(((fl & capi.TU_CBF) != 0) & ((fl & capi.TU_SCALING_LIST) != 0) & ((fl & (capi.TU_BYPASS | capi.TU_PCM)) == 0)
                     & (t["n_coeff"] > 0))[0]
    n = t["n_coeff"][sel].astype(np.int64)
    tu = np.repeat(sel, n)
    ci = np.repeat(t["coeff_off"][sel].astype(np.int64) - np.cumsum(n) + n, n) + np.arange(int(n.sum()))
    log2, cidx, flags = t["log2_size"][tu].astype(np.int64), t["cidx"][tu].astype(np.int64), fl[tu]
    nT = 1 << log2
    m = np.where(nT == 32, 0, cidx) + np.where((flags & capi.TU_INTER_MATRIX) != 0, np.where(nT < 32, 3, 1), 0)
    pos = p.coeffs["pos"][ci].astype(np.int64)
    base = np.select([nT == 4, nT == 8, nT == 16], [_BASE[4], _BASE[8], _BASE[16]], _BASE[32])
    factor = p.scaling[base + m * nT * nT + pos].astype(np.int64) if len(tu) else np.zeros(0, np.int64)
    bd = np.where(cidx == 0, p.params.bit_depth_luma, p.params.bit_depth_chroma)
    return dict(log2=log2, cidx=cidx, matrix=m, factor=factor, level=p.coeffs["level"][ci].astype(np.int64), qp=t["qp"][tu].astype(np.int64),
                bd=bd, flags=flags, pos=pos, tu=tu)


def dequant_exact(level, factor, qp, bd, log2):
    """transform.cc:489-525 with Python integers and without the clip: (level * (m * levelScale[qP % 6] << qP / 6) + offset)
    >> bdShift, bdShift = BitDepth + log2(nT) - 5."""
    sh = bd + log2 - 5
    return (level * ((factor * LEVEL_SCALE[qp % 6]) << (qp // 6)) + (1 << (sh - 1))) >> sh


def dequant_reference(level, factor, qp, bd, log2):
    """What the reference stores (transform.cc:522-523): the exact value's low 32 bits (Clip3 takes int), clipped to int16."""
    v = (dequant_exact(level, factor, qp, bd, log2) + (1 << 31)) % (1 << 32) - (1 << 31)
    return min(32767, max(-32768, v))


def _rows(pics):
    rows = [matrix_coeffs(p) for p in pics]
    return {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}


def make_sequence(case):
    """Reference planes (for slot 5) and the case's I -> P -> B -> weighted B pictures (range_cases.make_sequence)."""
    return range_cases.make_sequence(case.W, case.H, case.bd, **case.kw)


# ---- checks: (description, predicate over the sequence's pictures) ----
def all_matrices(chroma=True, max_log2=5):
    """max_log2: the largest luma TU (the CTB's, at most 32x32); a 4:2:0 chroma TU is at most half of it."""
    want = sorted({(1 << l, matrix_id(l, c, inter)) for c in ((0, 1, 2) if chroma else (0,)) for l in range(2, max_log2 + (0 if c else 1))
                   for inter in (False, True)})

    def f(pics):
        r = _rows(pics)
        got = set(zip((1 << r["log2"]).tolist(), r["matrix"].tolist()))
        return all(w in got for w in want)
    return f"every (size, matrix ID) pair {want} used by a coded coefficient", f


def clip_with_big_factor():
    def f(pics):
        r = _rows(pics)
        for i in np.nonzero(r["factor"] >= 128)[0].tolist():
            v = dequant_exact(int(r["level"][i]), int(r["factor"][i]), int(r["qp"][i]), int(r["bd"][i]), int(r["log2"][i]))
            if v > 32767 or v < -32768:
                return True
        return False
    return "a coefficient with factor >= 128 whose exact dequantised value lies beyond the int16 range", f


def beyond_int32():
    def f(pics):
        r = _rows(pics)
        for i in np.nonzero(r["factor"] > 16)[0].tolist():
            v = dequant_exact(int(r["level"][i]), int(r["factor"][i]), int(r["qp"][i]), int(r["bd"][i]), int(r["log2"][i]))
            if not -(1 << 31) <= v < (1 << 31):
                return True
        return False
    return "a coefficient whose exact dequantised value lies beyond the int32 range (the reference keeps its low 32 bits)", f


def tskip_sizes(log2s=(2, 3, 4, 5)):
    def f(pics):
        r = _rows(pics)
        ts = (r["flags"] & capi.TU_TSKIP) != 0
        return all((ts & (r["log2"] == l)).any() for l in log2s)
    return f"transform skip with a matrix at {[1 << l for l in log2s]}", f


def rdpcm_with_matrix():
    def f(pics):
        r = _rows(pics)
        ts = (r["flags"] & capi.TU_TSKIP) != 0
        return all((ts & ((r["flags"] & d) != 0)).any() for d in (capi.TU_RDPCM_H, capi.TU_RDPCM_V))
    return "horizontal and vertical RDPCM on transform-skip TUs with a matrix", f


def rotation_with_matrix():
    """A rotated transform-skip TU with a coefficient whose factor differs from the factor at the rotated position, so the
    lookup before rotation and the lookup after it give different residuals."""
    def f(pics):
        for p in pics:
            r = matrix_coeffs(p)
            rot = ((r["flags"] & capi.TU_ROTATE) != 0) & ((r["flags"] & capi.TU_TSKIP) != 0)
            if not rot.any():
                continue
            other = p.scaling[_BASE[4] + r["matrix"][rot] * 16 + 15 - r["pos"][rot]].astype(np.int64)
            if (other != r["factor"][rot]).any():
                return True
        return False
    return "a rotated transform-skip TU whose factor differs at the rotated position", f


def qp_prime(cidx, qp):
    def f(pics):
        r = _rows(pics)
        return ((r["cidx"] == cidx) & (r["qp"] == qp)).any()
    return f"a coded plane-{cidx} TU with a matrix at qP' = {qp}", f


def factors(lo=1, hi=255):
    def f(pics):
        fa = _rows(pics)["factor"]
        return (fa == lo).any() and (fa == hi).any() and all(p.scaling.min() == lo and p.scaling.max() == hi for p in pics)
    return f"coded coefficients with factors {lo} and {hi}", f


def default_lists():
    d = synth.default_scaling_factors()
    return "the spec's default lists", lambda pics: all((p.scaling == d).all() for p in pics)


def depths(bd_y, bd_c):
    return f"luma / chroma depths {bd_y} / {bd_c}", lambda pics: all((p.params.bit_depth_luma, p.params.bit_depth_chroma) == (bd_y, bd_c) for p in pics)


def no_chroma_tus():
    return "no chroma TU", lambda pics: all((p.tus["cidx"] == 0).all() for p in pics)


def ctb(log2):
    return f"CTB {1 << log2}", lambda pics: all(p.params.log2_ctb_size == log2 for p in pics)


def pb_intra_matrix(log2s=(2, 3, 4, 5)):
    def f(pics):
        r = _rows(pics[1:])
        intra = np.concatenate([(p.tus["flags"][matrix_coeffs(p)["tu"]] & capi.TU_INTRA) != 0 for p in pics[1:]])
        return all((intra & (r["log2"] == l)).any() for l in log2s)
    return f"intra TUs of P / B pictures with a matrix at {[1 << l for l in log2s]}", f


# ---- what the planner makes of the records (b200_plan_picture_host, no GPU): the residual path every matrix TU takes ----
def planner_paths(lib, pics):
    """{path: number of coded TUs with a matrix} over the sequence.  Paths: ("a", "warp" | "8x8" | "4x4") the k_residual
    classes of list A (tu_residual / res8_quarter / res4_lane adding onto the picture), ("b", nT) the intra TUs of list B by size
    (k_intra: res4_lane / res8_quarter / tu_residual into the int16 scratch)."""
    from test_cpu_planner import plan
    out = {}
    for p in pics:
        r = plan(lib, p)
        fl = p.tus["flags"].astype(np.int64)
        mat = ((fl & capi.TU_CBF) != 0) & ((fl & capi.TU_SCALING_LIST) != 0) & ((fl & capi.TU_BYPASS) == 0)
        la, na, n8 = r["la"].astype(np.int64), r["n_aw"], r["n_a8"]
        for name, idx in (("warp", la[:na]), ("8x8", la[na:na + n8]), ("4x4", la[na + n8:])):
            out[("a", name)] = out.get(("a", name), 0) + int(mat[idx].sum())
        lb = r["lb"].astype(np.int64)
        for l in range(2, 6):
            k = ("b", 1 << l)
            out[k] = out.get(k, 0) + int((mat[lb] & (p.tus["log2_size"][lb] == l)).sum())
    return out


def planner_wants(case):
    top = 1 << min(5, case.kw.get("log2_ctb", 6))
    return [("a", "warp"), ("a", "8x8"), ("a", "4x4")] + [("b", n) for n in (4, 8, 16, 32) if n <= top]


# ---- the case list ----
_TS = dict(tskip_max_log2=5, rdpcm_frac=0.3, rotate_frac=0.5)
_MAX = dict(scaling_list="max", size_area=(0.2, 0.4, 0.2, 0.2), special_frac=0.05, qp_range=(22, 51), **_TS)
_CIP = dict(constrained_intra=True, pb_intra_frac=0.5)


def _edges(chroma=True, max_log2=5, flat4=False, wrap=True):
    """The required edges (plus RDPCM and rotation with a matrix, and with `wrap` a value beyond int32); flat4: lists whose
    4x4 matrices and 8x8 list entries are too low for the clip edge and the same at every rotated position (the default lists)."""
    c = [all_matrices(chroma, max_log2), tskip_sizes(tuple(range(2, max_log2 + 1))), rdpcm_with_matrix()]
    return c if flat4 else c + [clip_with_big_factor(), rotation_with_matrix()] + ([beyond_int32()] if wrap else [])


CASES = [
    Case("max8", 320, 192, 8, dict(_MAX), _edges() + [factors(), depths(8, 8)]),
    Case("max9", 320, 192, 9, dict(_MAX), _edges() + [factors(), depths(9, 9)]),
    Case("max10", 320, 192, 10, dict(_MAX), _edges() + [factors(), depths(10, 10)]),
    Case("max12", 320, 192, 12, dict(_MAX), _edges() + [factors(), depths(12, 12)]),
    Case("max10_chroma12", 320, 192, 10, dict(_MAX, bit_depth_chroma=12), _edges() + [depths(10, 12)]),
    Case("max12_chroma9", 320, 192, 12, dict(_MAX, bit_depth_chroma=9), _edges() + [depths(12, 9)]),
    Case("max_mono8", 320, 192, 8, dict(_MAX, chroma_format_idc=0), _edges(chroma=False) + [no_chroma_tus()]),
    Case("max_mono10", 320, 192, 10, dict(_MAX, chroma_format_idc=0), _edges(chroma=False) + [no_chroma_tus()]),
    Case("max8_ctb16", 208, 120, 8, dict(_MAX, log2_ctb=4, size_area=(0.0, 0.0, 0.5, 0.5)), _edges(max_log2=4) + [ctb(4)]),
    Case("max10_ctb32", 320, 192, 10, dict(_MAX, log2_ctb=5, size_area=(0.0, 0.5, 0.3, 0.2)), _edges(wrap=False) + [ctb(5)]),
    Case("qp0_8", 320, 192, 8, dict(_MAX, qp_range=(0, 3), chroma_qp_offsets=(-12, -12)), _edges(wrap=False) + [qp_prime(0, 0), qp_prime(1, 0)]),
    Case("qp0_10", 320, 192, 10, dict(_MAX, qp_range=(-12, -9), chroma_qp_offsets=(-12, -12)), _edges(wrap=False) + [qp_prime(0, 0), qp_prime(2, 0)]),
    Case("qp_max12", 320, 192, 12, dict(_MAX, qp_range=(45, 51), chroma_qp_offsets=(12, 12)), _edges() + [qp_prime(0, 75), qp_prime(1, 75)]),
    Case("qp_max10_chroma12", 320, 192, 10, dict(_MAX, bit_depth_chroma=12, qp_range=(45, 51), chroma_qp_offsets=(12, 12)),
         _edges() + [qp_prime(0, 63), qp_prime(2, 75)]),
    Case("tskip32_rdpcm_rotate10", 320, 192, 10, dict(_MAX, special_frac=0.1, rdpcm_frac=0.5, rotate_frac=0.8), _edges(wrap=False)),
    Case("default10", 320, 192, 10, dict(scaling_list="default", size_area=(0.2, 0.4, 0.2, 0.2), special_frac=0.05, **_TS),
         _edges(flat4=True) + [default_lists()]),
    Case("cip_max8", 320, 192, 8, dict(_MAX, **_CIP), _edges() + [pb_intra_matrix()]),
    Case("cip_max10", 320, 192, 10, dict(_MAX, **_CIP), _edges() + [pb_intra_matrix()]),
]
CASE_IDS = [c.id for c in CASES]
BY_ID = {c.id: c for c in CASES}
