"""The in-loop filters branch by branch, as one shared case list with a classifier of the filters' decisions.

The sequences here steer the samples the filters see: a piecewise-smooth reference (synth.smooth_planes: gentle ramps with
steps on the 8x8 grid sized from tc at the case's QP) predicted with MVs on a 16-sample grid and residuals of one small DC
level, so the deblocking decisions (off / strong / weak / cut off) and the SAO categories all occur, at QP near the ends of
the beta / tc tables, QpC on every part of its table, 8 to 12 bit and unequal depths, no-filter CUs, slices, tiles, and
picture sizes with every CTB remainder.

The classifier (classify_deblock, classify_sao) restates the filters' decisions in numpy and counts the branches they take;
test_cpu_filters.py proves it agrees with the oracle sample for sample before trusting its counts, checks every case
reaches its branches, and pins the oracle to the reference on every case; test_gpu_filters.py runs the engine against the
oracle on every case and every filter kernel."""
from collections import namedtuple

import numpy as np

from libde265_b200 import capi, synth

Case = namedtuple("Case", "id W H bd kw checks")

TAB_BETA = np.array([0] * 16 + [6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 50, 52,
                                54, 56, 58, 60, 62, 64])
TAB_TC = np.array([0] * 18 + [1] * 9 + [2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24])
TAB_QPC = np.array([29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37])
assert len(TAB_BETA) == 52 and len(TAB_TC) == 54

# SAO edge classes: neighbour a = (x + HPOS[c][0], y + VPOS[c][0]), b = (x + HPOS[c][1], y + VPOS[c][1])
HPOS = np.array([[-1, 1], [0, 0], [-1, 1], [1, -1]])
VPOS = np.array([[0, 0], [-1, 1], [-1, 1], [-1, 1]])


def tc_at(qp):
    """tc (8-bit units, at least 1) at QpY ``qp`` and bS 2 with no slice offset."""
    return max(1, int(TAB_TC[min(53, max(0, qp + 2))]))


def make_sequence(W, H, bd, steps=None, pb_intra_frac=0.15, **kw):
    """Reference planes (uploaded to slot 5) and an I -> P -> B sequence on them.  ``steps``: the reference's step heights;
    by default, from tc at the middle of the case's QP range: 0, below the strong filter's 2.5 tc, in the weak filter's
    range and past its 10 tc cut-off, with spikes of 4, 8 and 12 tc that the strong filter's clamps cut.  "random":
    synth.random_planes instead of a smooth reference."""
    qp = kw.get("qp_range", (22, 37))
    tc = tc_at((qp[0] + qp[1]) // 2)
    if steps is None:
        steps = (0, 1, tc, 2 * tc, 4 * tc, 8 * tc, 20 * tc)
    ref_kw = dict(bit_depth_chroma=kw.get("bit_depth_chroma"), chroma_format_idc=kw.get("chroma_format_idc", 1))
    planes = synth.random_planes(W, H, bd, 99, **ref_kw) if steps == "random" else \
        synth.smooth_planes(W, H, bd, 99, steps, spikes=(4 * tc, 8 * tc, 12 * tc), **ref_kw)
    pb = dict(intra_frac=pb_intra_frac, **kw)
    pics = [synth.make_picture(W, H, "I", seed=11, dst_slot=0, bit_depth=bd, **kw),
            synth.make_picture(W, H, "P", seed=12, dst_slot=1, ref_slots=(5,), bit_depth=bd, **pb),
            synth.make_picture(W, H, "B", seed=13, dst_slot=2, ref_slots=(1, 5), bit_depth=bd, **pb)]
    return planes, pics


def with_bs(p, mask):
    """A copy of picture ``p`` whose bS map keeps only the bits in ``mask`` (3: vertical edges, 12: horizontal edges)."""
    return synth.SynthPicture(p.params, p.pus, p.weights, p.tus, p.coeffs, p.slices, p.ctbs, np.ascontiguousarray(p.bs_map & mask), p.qp_map,
                              p.nofilt_map, p.scaling)


def _add(cnt, key, n):
    cnt[key] = cnt.get(key, 0) + int(n)


def _clip(lo, hi, v):
    return np.minimum(np.maximum(v, lo), hi)


class _Geom:
    def __init__(self, p):
        P = p.params
        self.W, self.H, self.log2ctb = P.width, P.height, P.log2_ctb_size
        self.w4, self.h4, self.w8 = (self.W + 3) // 4, (self.H + 3) // 4, (self.W + 7) // 8
        self.wctb = (self.W + (1 << self.log2ctb) - 1) >> self.log2ctb
        self.hctb = (self.H + (1 << self.log2ctb) - 1) >> self.log2ctb
        self.qp = p.qp_map.reshape(-1, self.w8).astype(np.int64)
        self.nf = (p.nofilt_map.reshape(-1, self.w8) & 1) != 0
        self.ctb_slice = p.ctbs["slice_idx"].astype(np.int64)

    def slice_idx(self, xl, yl):  # luma coordinates -> index into the slice table
        return self.ctb_slice[(xl >> self.log2ctb) + (yl >> self.log2ctb) * self.wctb]


def classify_deblock(p, planes, vertical, cnt):
    """The deblocking of the edges of one direction of picture ``p`` applied to ``planes`` (its reconstruction): returns the
    filtered planes and adds the branches taken to ``cnt``.  Luma per 4-line segment: off (d >= beta), strong, the +-2 tc clamp
    deciding each of p0..p2 / q0..q2, one-sided (a no-filter block on one side); per weak line: cut off (|delta| >= 10 tc),
    delta clamped at +-tc, the tc / 2 clamp on p1 / q1, dEp / dEq on neither, one or both sides, one-sided.  tc = 0 with
    bS > 0, beta and tc table indices clipped at 0 and at 51 / 53.  Chroma per line: delta clamped at +-tc, one-sided, QpC
    below 30, on the 30..42 table and from 43."""
    g, P = _Geom(p), p.params
    d = "v" if vertical else "h"
    out = [x.astype(np.int64) for x in planes]
    bs = (p.bs_map.reshape(g.h4, g.w4).astype(np.int64) >> (0 if vertical else 2)) & 3
    uy, ux = np.nonzero(bs)
    keep = (ux % 2 == 0) if vertical else (uy % 2 == 0)
    uy, ux = uy[keep], ux[keep]
    bS = bs[uy, ux]
    xd, yd = ux * 4, uy * 4
    sl = p.slices[g.slice_idx(xd, yd)]
    qpq = g.qp[yd >> 3, xd >> 3]
    qpp = g.qp[yd >> 3, (xd - 1) >> 3] if vertical else g.qp[(yd - 1) >> 3, xd >> 3]
    nfq = g.nf[yd >> 3, xd >> 3]
    nfp = g.nf[yd >> 3, (xd - 1) >> 3] if vertical else g.nf[(yd - 1) >> 3, xd >> 3]
    fP, fQ = ~nfp, ~nfq
    qpl = (qpq + qpp + 1) >> 1

    # ---- luma ----
    bd = P.bit_depth_luma
    bi, ti = qpl + sl["beta_offset"].astype(np.int64), qpl + 2 * (bS - 1) + sl["tc_offset"].astype(np.int64)
    for key, m in (("beta_idx_below_0", bi < 0), ("beta_idx_above_51", bi > 51), ("tc_idx_below_0", ti < 0), ("tc_idx_above_53", ti > 53)):
        _add(cnt, key, m.sum())
    beta = TAB_BETA[_clip(0, 51, bi)] << (bd - 8)
    tc = TAB_TC[_clip(0, 53, ti)] << (bd - 8)
    _add(cnt, "tc_0", (tc == 0).sum())
    k, i = np.arange(4)[None, :, None], np.arange(4)[None, None, :]
    y = out[0]
    if vertical:
        rows = yd[:, None, None] + k
        qi, pi = (rows, xd[:, None, None] + i), (rows, xd[:, None, None] - 1 - i)
    else:
        cols = xd[:, None, None] + k
        qi, pi = (yd[:, None, None] + i, cols), (yd[:, None, None] - 1 - i, cols)
    pv, qv = y[pi], y[qi]  # [segment, line k, distance i]
    dp_ = np.abs(pv[:, :, 2] - 2 * pv[:, :, 1] + pv[:, :, 0])
    dq_ = np.abs(qv[:, :, 2] - 2 * qv[:, :, 1] + qv[:, :, 0])
    dpq0, dpq3 = dp_[:, 0] + dq_[:, 0], dp_[:, 3] + dq_[:, 3]
    dsum = dpq0 + dpq3
    on = dsum < beta
    _add(cnt, f"luma_{d}_off", (~on).sum())

    def strong_line(kk, dpq):
        return (2 * dpq < (beta >> 2)) & (np.abs(pv[:, kk, 3] - pv[:, kk, 0]) + np.abs(qv[:, kk, 0] - qv[:, kk, 3]) < (beta >> 3)) & \
            (np.abs(pv[:, kk, 0] - qv[:, kk, 0]) < ((5 * tc + 1) >> 1))
    strong = on & strong_line(0, dpq0) & strong_line(3, dpq3)
    weak = on & ~strong
    side = (beta + (beta >> 1)) >> 3
    dEp, dEq = (dp_[:, 0] + dp_[:, 3]) < side, (dq_[:, 0] + dq_[:, 3]) < side
    _add(cnt, f"luma_{d}_strong", strong.sum())
    _add(cnt, "luma_strong_one_sided", (strong & (fP != fQ)).sum())
    newp, newq = pv.copy(), qv.copy()
    p0, p1, p2, p3 = (pv[:, :, j] for j in range(4))
    q0, q1, q2, q3 = (qv[:, :, j] for j in range(4))
    t2 = 2 * tc[:, None]
    raw = {"p0": (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3, "p1": (p2 + p1 + p0 + q0 + 2) >> 2, "p2": (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3,
           "q0": (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3, "q1": (p0 + q0 + q1 + q2 + 2) >> 2, "q2": (p0 + q0 + q1 + 3 * q2 + 2 * q3 + 4) >> 3}
    for name, r in raw.items():
        old = pv[:, :, int(name[1])] if name[0] == "p" else qv[:, :, int(name[1])]
        c = _clip(old - t2, old + t2, r)
        f = (fP if name[0] == "p" else fQ)[:, None] & strong[:, None]
        _add(cnt, f"luma_strong_clamp_{name}", (f & (c != r)).sum())
        (newp if name[0] == "p" else newq)[:, :, int(name[1])] = np.where(f, c, old)
    tcl = tc[:, None]
    delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4
    act = weak[:, None] & (np.abs(delta) < 10 * tcl)
    _add(cnt, f"luma_{d}_weak_cutoff", (weak[:, None] & ~act).sum())
    dc = _clip(-tcl, tcl, delta)
    _add(cnt, "luma_weak_delta_clamped", (act & (dc != delta)).sum())
    maxv = (1 << bd) - 1
    fPl, fQl = fP[:, None] & act, fQ[:, None] & act
    newp[:, :, 0] = np.where(fPl, _clip(0, maxv, p0 + dc), newp[:, :, 0])
    newq[:, :, 0] = np.where(fQl, _clip(0, maxv, q0 - dc), newq[:, :, 0])
    rp = (((p2 + p0 + 1) >> 1) - p1 + dc) >> 1
    rq = (((q2 + q0 + 1) >> 1) - q1 - dc) >> 1
    cp, cq = _clip(-(tcl >> 1), tcl >> 1, rp), _clip(-(tcl >> 1), tcl >> 1, rq)
    mp, mq = fPl & dEp[:, None], fQl & dEq[:, None]
    _add(cnt, "luma_weak_p1_clamped", (mp & (cp != rp)).sum())
    _add(cnt, "luma_weak_q1_clamped", (mq & (cq != rq)).sum())
    newp[:, :, 1] = np.where(mp, _clip(0, maxv, p1 + cp), newp[:, :, 1])
    newq[:, :, 1] = np.where(mq, _clip(0, maxv, q1 + cq), newq[:, :, 1])
    ep, eq = dEp[:, None], dEq[:, None]
    for key, m in (("neither", ~ep & ~eq), ("p_only", ep & ~eq), ("q_only", ~ep & eq), ("both", ep & eq)):
        _add(cnt, f"luma_{d}_weak_dE_{key}", (act & m).sum())
    _add(cnt, "luma_weak_one_sided", (act & (fP != fQ)[:, None]).sum())
    y[pi], y[qi] = newp, newq

    # ---- chroma (4:2:0): the chroma 8x8 grid, bS 2 ----
    if P.chroma_format_idc:
        sel = (bS == 2) & ((ux % 4 == 0) & (uy % 2 == 0) if vertical else (ux % 2 == 0) & (uy % 4 == 0))
        bdc, maxc = P.bit_depth_chroma, (1 << P.bit_depth_chroma) - 1
        xc, yc = xd[sel] >> 1, yd[sel] >> 1
        kc = np.arange(4)[None, :]
        for c, off in ((1, P.pps_cb_qp_offset), (2, P.pps_cr_qp_offset)):
            qpi = qpl[sel] + off
            qpc = np.where(qpi < 30, qpi, np.where(qpi >= 43, qpi - 6, TAB_QPC[_clip(0, 12, qpi - 30)]))
            for key, m in (("below_30", qpi < 30), ("table", (qpi >= 30) & (qpi < 43)), ("from_43", qpi >= 43)):
                _add(cnt, f"chroma_qpi_{key}", m.sum())
            tcc = (TAB_TC[_clip(0, 53, qpc + 2 + sl["tc_offset"][sel].astype(np.int64))] << (bdc - 8))[:, None]
            _add(cnt, "chroma_tc_0", (tcc == 0).sum())
            pl = out[c]
            if vertical:
                r = yc[:, None] + kc
                ix = [(r, xc[:, None] + j) for j in (-2, -1, 0, 1)]
            else:
                cl = xc[:, None] + kc
                ix = [(yc[:, None] + j, cl) for j in (-2, -1, 0, 1)]
            cp1, cp0, cq0, cq1 = (pl[t] for t in ix)
            rd = ((cq0 - cp0) * 4 + cp1 - cq1 + 4) >> 3
            dl = _clip(-tcc, tcc, rd)
            fPc, fQc = fP[sel][:, None], fQ[sel][:, None]
            _add(cnt, f"chroma_{d}_lines", fPc.size)
            _add(cnt, "chroma_delta_clamped", ((dl != rd) & (fPc | fQc)).sum())
            _add(cnt, "chroma_one_sided", np.broadcast_to(fPc != fQc, dl.shape).sum())
            pl[ix[1]] = np.where(fPc, _clip(0, maxc, cp0 + dl), cp0)
            pl[ix[2]] = np.where(fQc, _clip(0, maxc, cq0 - dl), cq0)
    return [o.astype(x.dtype) for o, x in zip(out, planes)]


def classify_sao(p, planes, cnt):
    """SAO of picture ``p`` applied to ``planes`` (its deblocked picture): returns the output planes and adds to ``cnt``, per
    sample: edge class x category (e in -2..2; +-1 means one equal neighbour), band hits and hits past band 31 (band position
    29..31), clipping at 0 and at the maximum, no-filter samples and chroma samples whose no-filter luma block is the second of
    the two under their 8-sample group (the first one filtered), and for each reason a neighbour is unavailable (picture border,
    an earlier slice with the current slice's across flag off, a later slice with its own flag off, a tile border) the samples
    whose value that reason alone decides.  "sao_quirk": chroma samples whose value depends on looking up the current slice
    with the CTB's component coordinates (the reference's sao.cc:49) rather than the CTB's own slice."""
    g, P = _Geom(p), p.params
    out = [x.copy() for x in planes]
    if not (P.flags & capi.PIC_SAO_ENABLED) or (P.flags & capi.PIC_SKIP_SAO):
        return out
    ct, sli = p.ctbs, p.slices
    addr = sli["slice_addr_rs"].astype(np.int64)
    across = (sli["flags"] & capi.SLICE_LF_ACROSS_SLICES) != 0
    for c in range(3 if P.chroma_format_idc else 1):
        sh = 1 if c else 0
        v = planes[c].astype(np.int64)
        h, w = v.shape
        bd = P.bit_depth_chroma if c else P.bit_depth_luma
        maxv = (1 << bd) - 1
        ls = g.log2ctb - sh
        S = 1 << ls
        ys, xs = np.mgrid[0:h, 0:w]
        ctb = (xs >> ls) + (ys >> ls) * g.wctb
        ci = ct[ctb]
        on = (sli["flags"][ci["slice_idx"]] & (capi.SLICE_SAO_CHROMA if c else capi.SLICE_SAO_LUMA)) != 0
        typ = np.where(on, (ci["sao_type"].astype(np.int64) >> (2 * c)) & 3, 0)
        nf = g.nf[(ys << sh) >> 3, (xs << sh) >> 3]
        kind = "C" if c else "Y"
        _add(cnt, f"sao_nofilt_{kind}", (nf & (typ != 0)).sum())
        if c:
            bx = (xs << 1) >> 3
            first_ok = ~g.nf[(ys << 1) >> 3, np.maximum(bx - 1, 0)]
            _add(cnt, "sao_nofilt_second_block", (nf & (typ != 0) & (bx % 2 == 1) & first_ok).sum())
        offs = ct["sao_offset"][:, c, :].astype(np.int64)[ctb]  # [h, w, 4]
        # band offset
        pos = ct["sao_band_pos"][:, c].astype(np.int64)[ctb]
        band = v >> (bd - 5)
        kb = (band - pos) & 31
        bhit = (typ == 1) & ~nf & (kb < 4)
        bval = v + np.take_along_axis(offs, np.minimum(kb, 3)[..., None], 2)[..., 0]
        _add(cnt, "sao_band_hit", bhit.sum())
        _add(cnt, "sao_band_wrap", (bhit & (band < pos)).sum())
        _add(cnt, "sao_band_clip_0", (bhit & (bval < 0)).sum())
        _add(cnt, "sao_band_clip_max", (bhit & (bval > maxv)).sum())
        res = np.where(bhit, _clip(0, maxv, bval), v)
        # edge offset
        cls = (ci["sao_eo_class"].astype(np.int64) >> (2 * c)) & 3
        xC, yC = (xs >> ls) << ls, (ys >> ls) << ls
        ctbW, ctbH = np.minimum(S, w - xC), np.minimum(S, h - yC)
        border = (xs == xC) | (ys == yC) | (xs == xC + ctbW - 1) | (ys == yC + ctbH - 1)
        own = addr[ci["slice_idx"]]
        quirk = addr[g.slice_idx(np.minimum(xC, g.W - 1), np.minimum(yC, g.H - 1))]  # component coordinates as luma ones (sao.cc:49)
        sc_across = across[ci["slice_idx"]]
        nb, why = [], {r: np.zeros_like(border) for r in ("pic_border", "earlier_slice", "later_slice", "tile")}
        why_own = {r: np.zeros_like(border) for r in ("earlier_slice", "later_slice")}
        for k in range(2):
            xS, yS = xs + HPOS[cls, k], ys + VPOS[cls, k]
            inside = (xS >= 0) & (yS >= 0) & (xS < w) & (yS < h)
            xSc, ySc = _clip(0, w - 1, xS), _clip(0, h - 1, yS)
            nb.append(v[ySc, xSc])
            cn = ct[(((xSc << sh) >> g.log2ctb) + ((ySc << sh) >> g.log2ctb) * g.wctb)]
            na, nacr = addr[cn["slice_idx"]], across[cn["slice_idx"]]
            why["pic_border"] |= border & ~inside
            for d_, cur in ((why, quirk), (why_own, own)):
                d_["earlier_slice"] |= border & inside & (na < cur) & ~sc_across
                d_["later_slice"] |= border & inside & (na > cur) & ~nacr
            if not (P.flags & capi.PIC_LF_ACROSS_TILES):
                why["tile"] |= border & inside & (cn["tile_id"] != ci["tile_id"])
        e = np.sign(v - nb[0]) + np.sign(v - nb[1])
        eidx = np.where(e < 0, e + 2, e + 1)  # -2, -1, 1, 2 -> offsets 0..3
        eval_ = np.where(e == 0, v, _clip(0, maxv, v + np.take_along_axis(offs, np.clip(eidx, 0, 3)[..., None], 2)[..., 0]))
        edge = (typ == 2) & ~nf

        def applied(reasons):
            bad = np.zeros_like(border)
            for m in reasons.values():
                bad |= m
            return np.where(edge & ~bad, eval_, v)
        final = applied(why)
        for r in why:
            _add(cnt, f"sao_unavail_{r}", (final != applied({q: m for q, m in why.items() if q != r})).sum())
        ok = edge & ~np.logical_or.reduce(list(why.values()))
        for cl_ in range(4):
            for ev in range(-2, 3):
                _add(cnt, f"sao_eo{cl_}_e{ev:+d}", (ok & (cls == cl_) & (e == ev)).sum())
        _add(cnt, "sao_quirk", (final != applied(dict(why, **why_own))).sum())
        res = np.where(typ == 2, final, res)
        out[c] = res.astype(planes[c].dtype)
    return out


def sao_tails(p):
    """The store widths the SAO kernels' last groups take on picture ``p``: ("sao8", plane kind, n) for k_sao8's 16-sample
    segments (n = samples of the segment inside the CTB) and ("sao", plane kind, n) for k_sao's 8-sample groups."""
    g, P = _Geom(p), p.params
    tails = set()
    for c in range(2 if P.chroma_format_idc else 1):
        sh = 1 if c else 0
        w, S = g.W >> sh, 1 << (g.log2ctb - sh)
        kind = "C" if c else "Y"
        for xC in range(0, w, S):
            ctbW = min(S, w - xC)
            tails.update(("sao8", kind, min(16, ctbW - i0)) for i0 in range(0, ctbW, 16))
        tails.update(("sao", kind, min(8, w - x)) for x in range(0, w, 8))
    return tails


# ---- one oracle run of a case, stage by stage, with the classifier's counts ----
Run = namedtuple("Run", "case pics planes stages counts tails")
_RUNS = {}


def run_case(case, orc_factory):
    """Runs the case's sequence through the oracle (``orc_factory()`` makes one): per picture the reconstruction, the picture
    deblocked along vertical edges only and along horizontal edges only (its bS map with the other direction's bits cleared,
    so both start from the reconstruction), deblocked, and final.  The classifier counts the deblocking branches on the
    single-direction pictures and the SAO branches on the deblocked one.  Cached per case id."""
    if case.id in _RUNS:
        return _RUNS[case.id]
    planes, pics = make_sequence(case.W, case.H, case.bd, **case.kw)
    orc = orc_factory()
    orc.upload_slot(5, pics[0].params, planes)
    stages, cnt, tails = [], {}, set()
    for p in pics:
        st = {}
        for name, pic, stop in (("recon", p, capi.STAGE_RECON), ("deblock_v", with_bs(p, 3), capi.STAGE_DEBLOCK),
                                ("deblock_h", with_bs(p, 12), capi.STAGE_DEBLOCK), ("deblock", p, capi.STAGE_DEBLOCK), ("all", p, capi.STAGE_ALL)):
            pic.c.params.stop_after_stage = stop
            orc.reconstruct(pic)
            pic.c.params.stop_after_stage = 0
            st[name] = orc.read_slot(p.params.dst_slot, p.params)
        st["pred_v"] = classify_deblock(p, st["recon"], True, cnt)
        st["pred_h"] = classify_deblock(p, st["recon"], False, cnt)
        st["pred_sao"] = classify_sao(p, st["deblock"], cnt)
        stages.append(st)
        tails |= sao_tails(p)
    orc.close()
    r = Run(case, pics, planes, stages, cnt, tails)
    _RUNS[case.id] = r
    return r


# ---- checks: (description, predicate over a Run) ----
def at_least(n, *keys):
    return f"at least {n} of each of {list(keys)}", lambda r: all(r.counts.get(k, 0) >= n for k in keys)


def tails_reached(want):
    return f"SAO store widths {sorted(want)}", lambda r: set(want) <= r.tails


def sao_changes(n):
    return f"SAO changes at least {n} samples", lambda r: sum(int((st["all"][c] != st["deblock"][c]).sum()) for st in r.stages
                                                               for c in range(len(st["all"]))) >= n


def geometry(log2, W, H):
    return f"CTB {1 << log2} on a {W}x{H} picture", lambda r: all(p.params.log2_ctb_size == log2 and (p.params.width, p.params.height) == (W, H)
                                                                 for p in r.pics)


LUMA_DEBLOCK = ["luma_v_off", "luma_h_off", "luma_v_strong", "luma_h_strong", "luma_v_weak_cutoff", "luma_h_weak_cutoff",
                "luma_weak_delta_clamped"] + [f"luma_{d}_weak_dE_{k}" for d in "vh" for k in ("neither", "p_only", "q_only", "both")]
STRONG_CLAMP = [f"luma_strong_clamp_{s}{i}" for s in "pq" for i in range(3)]
CHROMA_DEBLOCK = ["chroma_v_lines", "chroma_h_lines", "chroma_delta_clamped"]
ONE_SIDED = ["luma_strong_one_sided", "luma_weak_one_sided", "chroma_one_sided"]
SAO_EDGE = [f"sao_eo{c}_e{e:+d}" for c in range(4) for e in range(-2, 3)]
SAO_BAND = ["sao_band_hit", "sao_band_wrap", "sao_band_clip_0", "sao_band_clip_max"]


# ---- the case list ----
_STEER = dict(cbf_prob=0.15, coeff_max=2, mv_step=16, size_area=(0.0, 0.3, 0.4, 0.3))


def _geometry_cases():
    """Widths and heights k * S + r for every r multiple of 8 below the CTB size S (16, 32, 64), the width remainders paired
    with a rotation of the height remainders, in 4:2:0 and 4:0:0 at 8 bit."""
    out = []
    for log2 in (4, 5, 6):
        S = 1 << log2
        rs = list(range(0, S, 8))
        for n, rw in enumerate(rs):
            rh = rs[(n + len(rs) // 2) % len(rs)]
            W, H = 2 * S + rw, S + rh if S > 16 else 2 * S + rh
            for cf in (1, 0):
                checks = [geometry(log2, W, H), at_least(4, "luma_v_strong", "luma_h_strong"), sao_changes(20)]
                out.append(Case(f"geom_ctb{S}_{W}x{H}{'' if cf else '_mono'}", W, H, 8, dict(log2_ctb=log2, chroma_format_idc=cf, **_STEER), checks))
    return out


CASES = [
    Case("steer8", 192, 128, 8, dict(_STEER), [at_least(10, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(1, *STRONG_CLAMP)]),
    Case("steer8_ctb32", 256, 160, 8, dict(log2_ctb=5, **_STEER), [at_least(20, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(5, *STRONG_CLAMP),
                                                                   at_least(10, *SAO_EDGE)]),
    Case("steer10", 192, 128, 10, dict(_STEER), [at_least(10, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(1, *STRONG_CLAMP)]),
    Case("steer12", 192, 128, 12, dict(_STEER), [at_least(10, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(1, *STRONG_CLAMP)]),
    Case("steer12_chroma9", 192, 128, 12, dict(bit_depth_chroma=9, **_STEER), [at_least(10, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(1, *STRONG_CLAMP)]),
    Case("steer10_chroma12", 192, 128, 10, dict(bit_depth_chroma=12, **_STEER), [at_least(10, *LUMA_DEBLOCK, *CHROMA_DEBLOCK), at_least(1, *STRONG_CLAMP)]),
    Case("qp_low8", 192, 128, 8, dict(qp_range=(0, 20), lf_offsets=(-12, -12), **_STEER),
         [at_least(20, "tc_0", "chroma_tc_0", "beta_idx_below_0", "tc_idx_below_0")]),
    Case("qp_high8", 192, 128, 8, dict(qp_range=(44, 51), lf_offsets=(12, 12), chroma_qp_offsets=(12, 12), **_STEER),
         [at_least(20, "beta_idx_above_51", "tc_idx_above_53", "chroma_qpi_from_43", "luma_v_strong", "luma_h_strong")]),
    Case("qpc_table10", 192, 128, 10, dict(qp_range=(26, 42), chroma_qp_offsets=(4, -4), **_STEER),
         [at_least(20, "chroma_qpi_below_30", "chroma_qpi_table", "chroma_qpi_from_43", *CHROMA_DEBLOCK)]),
    Case("nofilt8", 192, 128, 8, dict(special_frac=0.15, pcm_lf_disable=True, **_STEER),
         [at_least(10, *ONE_SIDED, "sao_nofilt_Y", "sao_nofilt_C", "sao_nofilt_second_block")]),
    Case("nofilt10_ctb16", 192, 128, 10, dict(special_frac=0.15, pcm_lf_disable=True, log2_ctb=4, **_STEER),
         [at_least(10, *ONE_SIDED, "sao_nofilt_Y", "sao_nofilt_C", "sao_nofilt_second_block")]),
    Case("sao_band8", 192, 128, 8, dict(log2_ctb=4, sao_band_pos=(28, 32), **_STEER), [at_least(20, *SAO_BAND)]),
    Case("sao_band10", 192, 128, 10, dict(log2_ctb=5, sao_band_pos=(28, 32), **_STEER), [at_least(20, *SAO_BAND)]),
    Case("slices8_ctb32", 256, 192, 8, dict(log2_ctb=5, n_slices=24, **_STEER),
         [at_least(10, "sao_unavail_pic_border", "sao_unavail_earlier_slice", "sao_unavail_later_slice"), at_least(1, "sao_quirk")]),
    Case("slices8_ctb16", 256, 192, 8, dict(log2_ctb=4, n_slices=40, **_STEER),
         [at_least(10, "sao_unavail_pic_border", "sao_unavail_earlier_slice", "sao_unavail_later_slice"), at_least(1, "sao_quirk")]),
    Case("slices10_ctb32", 256, 192, 10, dict(log2_ctb=5, n_slices=24, **_STEER), [at_least(1, "sao_quirk")]),
    Case("tiles8", 320, 192, 8, dict(log2_ctb=5, tiles=(3, 2), lf_across_tiles=False, n_slices=4, **_STEER), [at_least(10, "sao_unavail_tile")]),
    Case("tiles10_ctb16", 192, 128, 10, dict(log2_ctb=4, tiles=(3, 3), lf_across_tiles=False, **_STEER), [at_least(10, "sao_unavail_tile")]),
] + _geometry_cases()

CASE_IDS = [c.id for c in CASES]
BY_ID = {c.id: c for c in CASES}
