"""Record-level model of k_intra's small-TU prediction plans (libde265_b200/csrc/kernels_recon.cuh: intra_border_clamps, tu_desc,
intra_plan_words, g_intra_plan) and the pictures that reach every plan class.  Imports without a GPU: shared by
test_cpu_intra_plans.py (the table against the oracle, the coverage proof) and test_gpu_intra_plans.py (the engine on the same
pictures).

A 4x4 or 8x8 intra TU takes the fast path when its border substitution reduces to clamping the border index into [lo, hi]
(fast_clamps).  Its prediction then follows one of INTRA_PLAN_CLASSES plans, selected by the class

    ((((nT == 8) * 35 + mode) * 4 + (-lo / 4 - 1)) * 4 + (hi / 4 - 1)) * 8 + (smooth | bfilt << 1 | luma << 2)

ENCODABLE holds the classes tu_desc can produce, REACHABLE those a 4:2:0 / 4:0:0 picture whose luma size is a multiple of 8
can produce.  Both are stated as rules below, not listed."""
import collections

import numpy as np

from libde265_b200 import capi, synth

N_MODES = 35
INTRA_PLAN_CLASSES = 2 * N_MODES * 4 * 4 * 8
# the modes an 8x8 TU's border is [1 2 1] smoothed for when its plane is filtered (intrapred.h:185-258): not DC, and more than
# 7 away from both pure directions
SMOOTH_MODES = tuple(m for m in range(N_MODES) if m != 1 and min(abs(m - 26), abs(m - 10)) > 7)
BFILT_MODES = (10, 26)  # the pure directions, whose first column / row luma takes the boundary filter
CLAMP_PAIRS = {4: [(lo, hi) for lo in (-4, -8) for hi in (4, 8)],
               8: [(lo, hi) for lo in (-8, -12, -16) for hi in (8, 12, 16)]}


def encode(nT, mode, lo, hi, smooth, bfilt, luma):
    return (((((nT == 8) * N_MODES + mode) * 4 + (-lo // 4 - 1)) * 4 + (hi // 4 - 1)) * 8 + (int(smooth) | int(bfilt) << 1 | int(luma) << 2))


def decode(cls):
    """(nT, mode, lo, hi, smooth, bfilt, luma) of a class."""
    f, rest = cls & 7, cls >> 3
    hi, rest = 4 * ((rest & 3) + 1), rest >> 2
    lo, rest = -4 * ((rest & 3) + 1), rest >> 2
    return (8 if rest >= N_MODES else 4), rest % N_MODES, lo, hi, bool(f & 1), bool(f & 2), bool(f & 4)


def describe(cls):
    """E.g. '8x8 chroma mode 23 lo -12 hi 16' or '8x8 luma mode 26 lo -8 hi 16 bfilt'."""
    nT, mode, lo, hi, smooth, bfilt, luma = decode(cls)
    flags = (" smooth" if smooth else "") + (" bfilt" if bfilt else "")
    return f"{nT}x{nT} {'luma' if luma else 'chroma'} mode {mode} lo {lo} hi {hi}{flags}"


def _encodable():
    """Every class tu_desc can produce: the clamps of intra_border_clamps at each size (a 4x4 TU has one group of 4 samples per
    reach, an 8x8 TU two), smoothing only on 8x8 TUs in SMOOTH_MODES (either plane: a 4:4:4 picture filters chroma too), the
    boundary filter only on luma in BFILT_MODES (either value: TU_NO_BOUNDARY_FILTER clears it)."""
    out = set()
    for nT, pairs in CLAMP_PAIRS.items():
        for lo, hi in pairs:
            for mode in range(N_MODES):
                for luma in (False, True):
                    for smooth in (False, True):
                        for bfilt in (False, True):
                            if smooth and not (nT == 8 and mode in SMOOTH_MODES):
                                continue
                            if bfilt and not (luma and mode in BFILT_MODES):
                                continue
                            out.add(encode(nT, mode, lo, hi, smooth, bfilt, luma))
    return frozenset(out)


ENCODABLE = _encodable()


def _reachable():
    """The encodable classes a 4:2:0 / 4:0:0 picture with luma width and height multiples of 8 can produce:
    - chroma is never smoothed: only a 4:4:4 picture filters its chroma border;
    - a 4x4 luma TU with its bottom-left group available (lo = -8) has its top-right group available too (hi = 8): it is the
      top-left or bottom-left quarter of an aligned 8x8 block (the other two quarters are decoded before the block below-left
      of them).  The top-left quarter's top-right group lies in the same aligned 8x8 block above as its own top row, one CU or
      one earlier part of the same CU; the bottom-left quarter's is the top-right quarter, decoded before it;
    - an 8x8 luma TU's reach is all or nothing (lo in {-8, -16}, hi in {8, 16}): each reach is 8 samples of one 8x8 CU (the
      smallest CU), inside one CTB, one slice and one tile, entirely inside or outside the picture, and a CU is decoded entirely
      before or after the TU, so no group boundary inside it can separate an available from a missing sample.
    An 8x8 chroma TU's reach spans 16 luma samples, two 8x8 CUs: the picture edge (luma size = 8 mod 16) or constrained intra
    prediction (an intra CU next to an inter CU) can cut it after its first group, so all nine clamp pairs occur."""
    out = set()
    for cls in ENCODABLE:
        nT, mode, lo, hi, smooth, bfilt, luma = decode(cls)
        if smooth and not luma:
            continue
        if luma and nT == 4 and lo == -8 and hi == 4:
            continue
        if luma and nT == 8 and (lo == -12 or hi == 12):
            continue
        out.add(cls)
    return frozenset(out)


REACHABLE = _reachable()


def fast_clamps(tu):
    """intra_border_clamps: (lo, hi) when the TU's own left column, corner and top row are available and each reach is available
    up to a point from its inner end (substitution is then the index clamp into [lo, hi]), else None."""
    q = 1 << (int(tu["log2_size"]) - 2)
    g, av = (1 << q) - 1, int(tu["avail"])
    bl, tr = (av >> q) & g, (av >> (capi.AVAIL_TOP_BIT0 + q)) & g
    own = (av & g) == g and (av >> capi.AVAIL_CORNER_BIT) & 1 and ((av >> capi.AVAIL_TOP_BIT0) & g) == g
    if not own or bl & (bl + 1) or tr & (tr + 1):
        return None
    return -4 * (q + bin(bl).count("1")), 4 * (q + bin(tr).count("1"))


def filter_plane(cidx, pic_flags, chroma_format_idc):
    """Whether the plane's intra borders are smoothed at all (k_intra's filter_plane)."""
    return not (pic_flags & capi.PIC_INTRA_SMOOTHING_OFF) and (cidx == 0 or chroma_format_idc == 3)


def plan_class(tu, pic_flags, chroma_format_idc):
    """tu_desc: the class of an intra TU of at most 8x8 that takes the fast path, else None.  (With the default 16x16-luma
    regions every such TU runs on a region tile; with 8x8 regions an 8x8 chroma TU is a task of its own on the large-TU code.)"""
    flags, log2 = int(tu["flags"]), int(tu["log2_size"])
    if not flags & capi.TU_INTRA or log2 > 3:
        return None
    c = fast_clamps(tu)
    if c is None:
        return None
    nT, mode, cidx = 1 << log2, int(tu["intra_mode"]), int(tu["cidx"])
    smooth = nT == 8 and filter_plane(cidx, pic_flags, chroma_format_idc) and mode in SMOOTH_MODES
    bfilt = cidx == 0 and not flags & capi.TU_NO_BOUNDARY_FILTER and mode in BFILT_MODES
    return encode(nT, mode, c[0], c[1], smooth, bfilt, cidx == 0)


def census(pictures):
    """class -> [TUs with CBF, TUs without CBF] over the pictures' fast-path TUs."""
    out = collections.defaultdict(lambda: [0, 0])
    for p in pictures:
        for tu in p.tus:
            cls = plan_class(tu, p.params.flags, p.params.chroma_format_idc)
            if cls is not None:
                out[cls][0 if tu["flags"] & capi.TU_CBF else 1] += 1
    return dict(out)


# The picture set: luma sizes = 8 mod 16 in both dimensions (8x8 chroma reaches cut by the picture edge after one group), CTB
# 16 / 32 / 64, I pictures and P / B pictures with intra CUs (one with constrained intra prediction and tiles: reaches cut by inter
# CUs and tile columns), bypass CUs with implicit RDPCM (TU_NO_BOUNDARY_FILTER) and intra smoothing off.
# (W, H, type, seed, log2 CTB, kw)
_SMALL_CUS = (0.0, 0.1, 0.5, 0.4)
SPECS = (
    (200, 136, "I", 11, 4, {}),
    (200, 136, "I", 12, 5, {}),
    (456, 264, "I", 13, 6, {}),
    (200, 136, "P", 14, 5, {"intra_frac": 0.6}),
    (456, 264, "B", 15, 6, {"intra_frac": 0.7, "constrained_intra": True, "tiles": (3, 1)}),
    (200, 136, "B", 16, 4, {"intra_frac": 0.8, "no_bfilter_on_bypass": True, "special_frac": 0.2}),
    (456, 264, "I", 19, 5, {"no_bfilter_on_bypass": True, "special_frac": 0.3}),
    (200, 136, "I", 17, 5, {"intra_smoothing_off": True}),
    (456, 264, "I", 18, 6, {"intra_smoothing_off": True}),
) + tuple(  # 8x8 luma TUs with TU_NO_BOUNDARY_FILTER, many with the top-right reach beyond the right edge (x = W - 8, W = 8 mod 16)
    (24, 264, "I", seed, 4 + seed % 3, {"no_bfilter_on_bypass": True, "special_frac": 0.5, "size_area": (0.0, 0.0, 0.0, 1.0)})
    for seed in range(20, 32)
)
# An 8x8 chroma TU (a 16x16 luma block at x, y) whose bottom-left reach the picture's bottom edge cuts after one group lies at
# y = H - 24 and reads it only as the top-left quarter of a 32x32 block (y = 0 mod 32), so H = 24 mod 32; the same goes for the
# top-right reach at x = W - 24.  Its top-right reach is missing at x = W - 16 (W = 16 mod 32).  So each of these tiny
# I pictures of 16x16 CUs has one bottom-right 16x16 block with lo = -12 and hi = 12 (88x88) or hi = 8 (48x88): one or two such
# TUs per picture at most, so many pictures.  cbf_prob 2/3: twice as many TUs with CBF as without, as the coverage asks.
CORNERS = ((88, 88, 5), (48, 88, 6), (48, 88, 5), (88, 88, 6))
N_CORNER_PICTURES = 320
REF_SLOTS = (0, 1)
DST_SLOT = 2


def _cycle_modes(pic, counters, implicit_rdpcm):
    """Reassign the intra mode of every fast-path TU, cycling per (size, plane, lo, hi, CBF, filter context) bucket through the
    modes whose class the bucket can reach, so that rare buckets reach every mode in few pictures.  An 8x8 luma TU of a picture
    with smoothing off cycles through SMOOTH_MODES and a luma TU with TU_NO_BOUNDARY_FILTER through BFILT_MODES: on their other
    modes they take the classes the other pictures reach.  With implicit RDPCM the RDPCM direction of a bypass / transform-skip
    TU follows its mode (transform.cc:425-432), as synth.make_picture derived it."""
    fl, cf = pic.params.flags, pic.params.chroma_format_idc
    tus = pic.tus
    for i in range(len(tus)):
        tu = tus[i]
        flags, log2 = int(tu["flags"]), int(tu["log2_size"])
        if not flags & capi.TU_INTRA or log2 > 3:
            continue
        c = fast_clamps(tu)
        if c is None:
            continue
        luma, nT = int(tu["cidx"]) == 0, 1 << log2
        filt = filter_plane(int(tu["cidx"]), fl, cf)
        nobf = luma and bool(flags & capi.TU_NO_BOUNDARY_FILTER)
        if nT == 8 and luma and not filt:
            modes = SMOOTH_MODES
        elif nobf:
            modes = BFILT_MODES
        else:
            modes = range(N_MODES)
        key = (nT, luma, c, bool(flags & capi.TU_CBF), filt, nobf)
        mode = modes[counters[key] % len(modes)]
        counters[key] += 1
        tus[i]["intra_mode"] = mode
        if implicit_rdpcm and flags & (capi.TU_BYPASS | capi.TU_TSKIP):
            flags &= ~(capi.TU_RDPCM_H | capi.TU_RDPCM_V)
            if mode in BFILT_MODES:
                flags |= capi.TU_RDPCM_H if mode == 10 else capi.TU_RDPCM_V
            tus[i]["flags"] = flags


def coverage_pictures(bd, bd_c=None):
    """The picture set at luma depth bd (chroma bd_c, default bd), modes reassigned by _cycle_modes.  P / B pictures read
    slots REF_SLOTS (reference_planes); every picture writes slot DST_SLOT."""
    counters = collections.Counter()
    out = []
    for W, H, kind, seed, log2_ctb, kw in SPECS:
        refs = () if kind == "I" else REF_SLOTS
        p = synth.make_picture(W, H, kind, seed=seed, bit_depth=bd, bit_depth_chroma=bd_c, dst_slot=DST_SLOT, ref_slots=refs,
                               log2_ctb=log2_ctb, **{"size_area": _SMALL_CUS, **kw})
        _cycle_modes(p, counters, kw.get("no_bfilter_on_bypass", False))
        out.append(p)
    for i in range(N_CORNER_PICTURES):
        W, H, log2_ctb = CORNERS[i % len(CORNERS)]
        p = synth.make_picture(W, H, "I", seed=1000 + i, bit_depth=bd, bit_depth_chroma=bd_c, dst_slot=DST_SLOT, log2_ctb=log2_ctb,
                               size_area=(0.0, 0.0, 1.0, 0.0), cbf_prob=2 / 3)
        _cycle_modes(p, counters, False)
        out.append(p)
    return out


def reference_planes(pic, slot):
    """The samples of reference slot `slot` for picture `pic` (its size and depths)."""
    pp = pic.params
    return synth.random_planes(pp.width, pp.height, pp.bit_depth_luma, 100 + slot, bit_depth_chroma=pp.bit_depth_chroma)


def upload_references(targets, pic):
    """Upload the picture's reference slots to each engine / oracle in `targets` (I pictures: none)."""
    if pic.c.n_pu:
        for s in REF_SLOTS:
            planes = reference_planes(pic, s)
            for t in targets:
                t.upload_slot(s, pic.params, planes)


def oracle_outputs(oracle_mod, pictures, stage):
    """The oracle's DST_SLOT planes of each picture at `stage`."""
    orc = oracle_mod.Oracle()
    out = []
    try:
        for p in pictures:
            upload_references((orc,), p)
            p.c.params.stop_after_stage = stage
            orc.reconstruct(p)
            out.append(orc.read_slot(DST_SLOT, p.params))
    finally:
        for p in pictures:
            p.c.params.stop_after_stage = 0
        orc.close()
    return out


def first_mismatch_class(pic, got, want):
    """Where `got` and `want` differ: the first differing sample in raster order and the first TU in decode order whose block
    differs (a wrong sample spreads to the TUs predicted from it), with its plan class.  None when they are equal."""
    where = None
    for c, (a, b) in enumerate(zip(got, want)):
        d = np.argwhere(a != b)
        if len(d) and where is None:
            y, x = (int(v) for v in d[0])
            where = f"plane {c}: {len(d)} samples differ, first at (x={x}, y={y}): got {a[y, x]} != oracle {b[y, x]}"
    if where is None:
        return None
    for tu in pic.tus:
        c, n, x, y = int(tu["cidx"]), 1 << int(tu["log2_size"]), int(tu["x"]), int(tu["y"])
        if c < len(got) and (got[c][y:y + n, x:x + n] != want[c][y:y + n, x:x + n]).any():
            cls = plan_class(tu, pic.params.flags, pic.params.chroma_format_idc)
            kind = describe(cls) if cls is not None else (f"{n}x{n} intra, not on the fast path" if tu["flags"] & capi.TU_INTRA else f"{n}x{n} inter")
            return f"{where}; first TU in decode order that differs: plane {c} at ({x}, {y}), {kind}"
    return f"{where}; no TU record covers a differing sample"
