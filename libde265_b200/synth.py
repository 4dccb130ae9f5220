"""Seeded synthetic HEVC *command-record* generator (SURVEY.md §8d "synthetic inputs").

No HEVC encoder exists offline, so parity tests at 1080p/4K and bench.py synthesise what the host
parser would have recorded for a picture: a random-but-legal CU/PU/TU quadtree in decode order
(CTB raster, z-order inside, luma -> Cb -> Cr per TU with the 4x4 chroma deferral of
slice.cc:3795-3847), intra modes with z-order availability masks (intrapred.h:436-633), quantised
coefficient lists, motion vectors with random fractional phase (some far outside the picture),
optional explicit weights, transform-skip / transquant-bypass / PCM blocks, a boundary-strength map
derived from the generated structure (deblock.cc:243-383 rules) and SAO parameters per CTB.

Everything is produced with numpy structured arrays whose dtypes mirror include/b200hevc.h, so a
picture can be handed to the engine and to the oracle unchanged.
"""
import ctypes as C

import numpy as np

from . import capi

PU_DT = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "u1"), ("h", "u1"), ("flags", "u1"), ("reserved", "u1"),
                  ("ref_slot", "i1", (2,)), ("wt_idx", "<u2"), ("mv", "<i2", (2, 2)), ("pad", "<u4")])
WT_DT = np.dtype([("w", "<i2", (2, 3)), ("o", "<i2", (2, 3)), ("log2wd_luma", "u1"), ("log2wd_chroma", "u1"), ("pad", "u1", (2,))])
TU_DT = np.dtype([("x", "<u2"), ("y", "<u2"), ("log2_size", "u1"), ("cidx", "u1"), ("flags", "<u2"), ("intra_mode", "u1"),
                  ("qp", "u1"), ("n_coeff", "<u2"), ("coeff_off", "<u4"), ("avail", "<u8")])
CO_DT = np.dtype([("pos", "<u2"), ("level", "<i2")])
SL_DT = np.dtype([("slice_addr_rs", "<u4"), ("beta_offset", "i1"), ("tc_offset", "i1"), ("flags", "u1"), ("pad", "u1")])
CTB_DT = np.dtype([("slice_idx", "<u2"), ("tile_id", "<u2"), ("sao_type", "u1"), ("sao_eo_class", "u1"), ("sao_band_pos", "u1", (3,)),
                   ("sao_offset", "i1", (3, 4)), ("pad", "u1", (3,))])
assert PU_DT.itemsize == 24 and WT_DT.itemsize == 28 and TU_DT.itemsize == 24 and CO_DT.itemsize == 4
assert SL_DT.itemsize == 8 and CTB_DT.itemsize == 24

_TAB_QPC = [29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37]


def _table8_22(q):
    return q if q < 30 else (q - 6 if q >= 43 else _TAB_QPC[q - 30])


def _zorder(x, y):
    """Interleave the low 5 bits of x (even positions) and y (odd positions)."""
    z = 0
    for b in range(5):
        z |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
    return z


_Z = np.array([[_zorder(x, y) for x in range(16)] for y in range(16)], dtype=np.int64)  # [y4][x4] inside a 64x64 CTB


def diag_scan(n):
    """Up-right diagonal scan of an n x n block (H.265 6.5.3): the (x, y) of scan positions 0 .. n*n - 1."""
    return [(s - y, y) for s in range(2 * n - 1) for y in range(min(s, n - 1), -1, -1) if s - y < n]


# H.265 Table 7-6: default ScalingList[1..3][matrixId][i] in up-right diagonal order (Table 7-5: every 4x4 entry is 16)
DEFAULT_LIST_INTRA = (16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 17, 16, 17, 16, 17, 18, 17, 18, 18, 17, 18, 21, 19, 20, 21, 20, 19, 21, 24, 22, 22, 24,
                      24, 22, 22, 24, 25, 25, 27, 30, 27, 25, 25, 29, 31, 35, 35, 31, 29, 36, 41, 44, 41, 36, 47, 54, 54, 47, 65, 70, 65, 88, 88, 115)
DEFAULT_LIST_INTER = (16, 16, 16, 16, 16, 16, 16, 16, 16, 16, 17, 17, 17, 17, 17, 18, 18, 18, 18, 18, 18, 20, 20, 20, 20, 20, 20, 20, 24, 24, 24, 24,
                      24, 24, 24, 24, 25, 25, 25, 25, 25, 25, 25, 28, 28, 28, 28, 28, 28, 33, 33, 33, 33, 33, 41, 41, 41, 41, 54, 54, 54, 71, 71, 91)
SCALING_SIZES = ((4, 0), (8, 6 * 16), (16, 6 * 16 + 6 * 64), (32, 6 * 16 + 6 * 64 + 6 * 256))  # (nT, byte offset of matrix 0)


def scaling_factor(lst, n, dc=16):
    """ScalingFactor of one n x n matrix (H.265 7.4.5) from a 16-entry (n = 4) or 64-entry list in up-right diagonal order:
    the 8x8 list is replicated over (n / 8) x (n / 8) squares for n = 16 / 32, whose position 0 then takes the DC value.
    Flat at x + n * y, the layout of b200_picture.scaling_factors."""
    k = 4 if n == 4 else 8
    m = np.zeros((k, k), np.uint8)
    for i, (x, y) in enumerate(diag_scan(k)):
        m[y, x] = lst[i]
    f = np.kron(m, np.ones((n // k, n // k), np.uint8)).reshape(-1)
    if n >= 16:
        f[0] = dc
    return f


def default_scaling_factors():
    """The spec's default lists (Tables 7-5 / 7-6) expanded with DC 16: matrices 0..2 intra, 3..5 inter at 4x4 to 16x16;
    32x32 matrix 0 intra, 1 inter (the matrix a 32x32 TU record selects), 2..5 unused in 4:2:0 / 4:0:0 and left flat."""
    out = np.full(capi.SCALING_FACTOR_BYTES, 16, np.uint8)
    for n, base in SCALING_SIZES:
        for m in range(6 if n < 32 else 2):
            inter = m >= 3 if n < 32 else m == 1
            out[base + m * n * n:base + (m + 1) * n * n] = scaling_factor((16,) * 16 if n == 4 else DEFAULT_LIST_INTER if inter else DEFAULT_LIST_INTRA, n)
    return out


def max_scaling_factors(rng):
    """Lists drawn over the whole range the syntax allows (1..255): every matrix holds both 1 and 255, and the DC of every 16x16
    and 32x32 matrix differs from the entry its 8x8 list puts at position 0."""
    out = np.zeros(capi.SCALING_FACTOR_BYTES, np.uint8)
    for n, base in SCALING_SIZES:
        k = 16 if n == 4 else 64
        for m in range(6):
            lst = rng.integers(1, 256, k)
            lo, hi = rng.choice(k, 2, replace=False)
            lst[lo], lst[hi] = 1, 255
            dc = int(rng.integers(1, 255))
            dc += dc >= lst[0]  # uniform over 1..255 without lst[0]
            out[base + m * n * n:base + (m + 1) * n * n] = scaling_factor(lst, n, dc)
    return out

# Reference border of a slot (B200_PAD_X / _Y / _CX / _CY of csrc/dev_common.cuh): MC windows further out are moved to this rim.
_PAD_X, _PAD_Y, _PAD_CX, _PAD_CY = 128, 80, 64, 40


class SynthPicture:
    """Holds the numpy arrays of one picture and a ctypes ``capi.Picture`` view of them."""

    def __init__(self, params, pus, weights, tus, coeffs, slices, ctbs, bs_map, qp_map, nofilt_map, scaling=None):
        self.params = params
        self.pus, self.weights, self.tus, self.coeffs = pus, weights, tus, coeffs
        self.slices, self.ctbs, self.bs_map, self.qp_map, self.nofilt_map, self.scaling = slices, ctbs, bs_map, qp_map, nofilt_map, scaling
        p = capi.Picture()
        p.params = params
        p.n_pu, p.n_weights, p.n_tu, p.n_coeff, p.n_slices = len(pus), len(weights), len(tus), len(coeffs), len(slices)

        def ptr(a, t):
            return a.ctypes.data_as(C.POINTER(t)) if a is not None and len(a) else C.cast(None, C.POINTER(t))

        p.pus, p.weights, p.tus, p.coeffs = ptr(pus, capi.PU), ptr(weights, capi.WeightEntry), ptr(tus, capi.TU), ptr(coeffs, capi.Coeff)
        p.slices, p.ctbs = ptr(slices, capi.SliceInfo), ptr(ctbs, capi.CtbInfo)
        p.bs_map, p.qp_map, p.nofilt_map = ptr(bs_map, C.c_uint8), ptr(qp_map, C.c_int8), ptr(nofilt_map, C.c_uint8)
        p.scaling_factors = ptr(scaling, C.c_uint8)
        self.c = p

    def algorithmic_mc_bytes(self):
        """SURVEY §8(d): per PU and used list (W+7)(H+7) luma + 2 (W/2+3)(H/2+3) chroma sample reads (halo-free when
        the phase is integer), 1.5 W H sample writes per PU, + the command record."""
        bps = 2 if self.params.bit_depth_luma > 8 else 1
        pu = self.pus
        if not len(pu):
            return 0
        w, h = pu["w"].astype(np.int64), pu["h"].astype(np.int64)
        total = (3 * w * h // 2).sum() * bps + len(pu) * PU_DT.itemsize
        for l in range(2):
            used = (pu["flags"] & (1 << l)) != 0
            fx, fy = (pu["mv"][:, l, 0] & 3) != 0, (pu["mv"][:, l, 1] & 3) != 0
            cfx, cfy = (pu["mv"][:, l, 0] & 7) != 0, (pu["mv"][:, l, 1] & 7) != 0
            lum = (w + 7 * fx) * (h + 7 * fy)
            chr_ = 2 * (w // 2 + 3 * cfx) * (h // 2 + 3 * cfy)
            total += ((lum + chr_) * used).sum() * bps
        return int(total)


def make_picture(width, height, pic_type="B", seed=1, bit_depth=8, dst_slot=0, ref_slots=(), log2_ctb=6, intra_frac=None,
                 weighted=False, deblock=True, sao=True, special_frac=0.01, cbf_prob=0.6, n_slices=1, scaling_list=False,
                 size_area=(0.10, 0.25, 0.35, 0.30), qp_range=(22, 37), far_mv_frac=0.01, tiles=(1, 1), lf_across_tiles=True,
                 rdpcm_frac=0.0, rotate_frac=0.0, tskip_max_log2=2, chroma_format_idc=1, bit_depth_chroma=None, chroma_qp_offsets=None,
                 lf_offsets=None, weight_range="narrow", sao_offset="random", extreme_mv_frac=0.0, strong_smoothing=True,
                 intra_smoothing_off=False, no_bfilter_on_bypass=False, pcm_lf_disable=False, slice_deblock_off_frac=0.0,
                 slice_sao_off_frac=0.0, skip_sao=False, constrained_intra=False, coeff_max=None, mv_step=None,
                 sao_band_pos=(0, 32)):
    """Generate one picture.  ``size_area`` = fraction of the picture area coded as 64/32/16/8 CUs.
    ``tiles`` = (columns, rows) of uniformly spaced tiles (pps.cc uniform_spacing rule): CTBs are then coded in tile-scan
    order and intra availability stops at tile borders (intrapred.h:488-503); ``lf_across_tiles`` False also removes the
    deblocking edges on tile borders (deblock.cc:185-230) and lets SAO treat the neighbour tile as unavailable (sao.cc:157).
    ``rdpcm_frac`` / ``rotate_frac``: share of the transform-skip / bypass TUs that use RDPCM (RExt implicit/explicit rdpcm,
    transform.cc:425-432,566-578) resp. coefficient rotation (4x4 TUs of intra CUs, transform.cc:402-404);
    ``tskip_max_log2``: largest transform-skip TU (RExt log2_max_transform_skip_block_size).

    Range knobs (each, at its default, draws no random number and changes nothing):
    ``chroma_format_idc`` 0 (4:0:0: no chroma TUs, luma-only PCM) or 1; ``bit_depth_chroma`` (default: ``bit_depth``) for the
    chroma PCM samples, QpBdOffsetC, log2wd_chroma, the chroma weight offsets and the SAO chroma offsets; ``qp_range`` may
    start at -QpBdOffsetY; ``chroma_qp_offsets`` = (pps_cb, pps_cr); ``lf_offsets`` = (beta, tc) of every slice (the
    slice_*_offset_div2 values times 2); ``weight_range`` "spec": weights (1 << denom) + [-128, 127] and offsets
    [-128, 127] << (bd - 8) per plane, with the extremes -128 (one past the syntax's floor) and 255 always present;
    ``sao_offset`` "max": every SAO offset at +-((1 << (min(bd, 10) - 5)) - 1) << log2_sao_offset_scale, scale drawn in
    [0, bd - 10]; ``extreme_mv_frac``: share of the PUs touching the picture border whose MV components are -32768 / 32767 or
    land just inside / outside the rim of the slot's reference border (any phase); ``strong_smoothing`` /
    ``intra_smoothing_off``: the SPS flags; ``no_bfilter_on_bypass``: implicit RDPCM enabled (TU_NO_BOUNDARY_FILTER on the
    intra TUs of bypass CUs, implicit RDPCM on their horizontal / vertical bypass and transform-skip TUs, as
    integration/libde265_hooks.cc records them); ``pcm_lf_disable``: pcm_loop_filter_disable (PCM CUs in ``nofilt_map``);
    ``slice_deblock_off_frac`` / ``slice_sao_off_frac``: share of the slices with deblocking off (their edges get bS 0) resp.
    each SAO plane flag off; ``skip_sao``: PIC_SKIP_SAO; ``constrained_intra``: constrained_intra_pred_flag, a neighbour group
    of an intra TU counts as available only if its CU is intra (intrapred.h:557-616, as integration/libde265_hooks.cc records
    it): only the ``avail`` masks change; ``scaling_list`` True: factors drawn over 1..63 (half of them 16), "default": the
    spec's default lists (default_scaling_factors), "max": lists over 1..255 (max_scaling_factors) — each sets
    PIC_SCALING_LIST and marks every coded non-bypass TU with its matrix.

    Filter-steering knobs (same rule: at the default nothing changes): ``coeff_max`` codes every coded TU as one nonzero DC level in
    [-coeff_max, coeff_max], so residuals shift whole blocks (a flat step at transform edges) instead of adding texture;
    ``mv_step``: every MV is a multiple of ``mv_step`` luma samples in each component (-2 .. 2 steps), so a reference with
    steps on its 8x8 grid keeps them on the picture's 8x8 grid when mv_step is a multiple of 8; ``sao_band_pos`` = [lo, hi) of
    the SAO band positions (29..31 put two or three of the four bands past band 31, onto bands 0..2)."""
    assert width % 8 == 0 and height % 8 == 0
    assert chroma_format_idc in (0, 1)
    rng = np.random.default_rng(seed)
    S = 1 << log2_ctb
    wctb, hctb = (width + S - 1) // S, (height + S - 1) // S
    w4, h4, w8, h8 = (width + 3) // 4, (height + 3) // 4, (width + 7) // 8, (height + 7) // 8
    bd_c = bit_depth if bit_depth_chroma is None else bit_depth_chroma
    bdoff, bdoff_c = 6 * (bit_depth - 8), 6 * (bd_c - 8)
    if intra_frac is None:
        intra_frac = 1.0 if pic_type == "I" else 0.08
    if pic_type != "I" and not ref_slots:
        raise ValueError("P/B pictures need ref_slots")
    if qp_range[0] < -bdoff or qp_range[1] > 51:
        raise ValueError(f"qp_range {qp_range}: QpY lies in [-{bdoff}, 51] at {bit_depth} bit")
    cb_off, cr_off = int(rng.integers(-3, 4)), int(rng.integers(-3, 4))
    if chroma_qp_offsets is not None:
        cb_off, cr_off = chroma_qp_offsets

    params = capi.PicParams()
    params.width, params.height = width, height
    params.chroma_format_idc = chroma_format_idc
    params.bit_depth_luma, params.bit_depth_chroma = bit_depth, bd_c
    params.log2_ctb_size = log2_ctb
    flags = (capi.PIC_STRONG_INTRA_SMOOTHING if strong_smoothing else 0) | (capi.PIC_LF_ACROSS_TILES if lf_across_tiles else 0)
    if sao:
        flags |= capi.PIC_SAO_ENABLED
    if not deblock:
        flags |= capi.PIC_SKIP_DEBLOCK
    if scaling_list:
        flags |= capi.PIC_SCALING_LIST
    if intra_smoothing_off:
        flags |= capi.PIC_INTRA_SMOOTHING_OFF
    if pcm_lf_disable:
        flags |= capi.PIC_PCM_LF_DISABLE
    if skip_sao:
        flags |= capi.PIC_SKIP_SAO
    params.flags = flags
    params.pps_cb_qp_offset, params.pps_cr_qp_offset = cb_off, cr_off
    params.dst_slot = dst_slot
    params.poc = seed

    # ---- tiles: uniform spacing; CTB coding order = tiles in raster order, CTBs in raster order inside a tile ----
    n_ctb = wctb * hctb
    tcols, trows = max(1, min(tiles[0], wctb)), max(1, min(tiles[1], hctb))
    col_bd = [(i * wctb) // tcols for i in range(tcols + 1)]
    row_bd = [(j * hctb) // trows for j in range(trows + 1)]
    ctb_tile = np.zeros(n_ctb, np.int32)
    ctb_order = []  # raster addresses in coding (tile-scan) order
    for tj in range(trows):
        for ti in range(tcols):
            for cy in range(row_bd[tj], row_bd[tj + 1]):
                for cx in range(col_bd[ti], col_bd[ti + 1]):
                    ctb_tile[cx + cy * wctb] = ti + tj * tcols
                    ctb_order.append(cx + cy * wctb)
    ts_of = np.zeros(n_ctb, np.int64)
    ts_of[np.array(ctb_order)] = np.arange(n_ctb)

    # ---- slices: contiguous CTB ranges in coding order ----
    n_slices = max(1, min(n_slices, n_ctb))
    bounds = [0] + sorted(rng.choice(np.arange(1, n_ctb), size=n_slices - 1, replace=False).tolist()) + [n_ctb] if n_slices > 1 else [0, n_ctb]
    slices = np.zeros(n_slices, SL_DT)
    ctb_slice = np.zeros(n_ctb, np.int32)
    for i in range(n_slices):
        slices[i]["slice_addr_rs"] = ctb_order[bounds[i]]
        slices[i]["beta_offset"] = 2 * int(rng.integers(-3, 4))
        slices[i]["tc_offset"] = 2 * int(rng.integers(-3, 4))
        if lf_offsets is not None:
            slices[i]["beta_offset"], slices[i]["tc_offset"] = lf_offsets
        f = capi.SLICE_SAO_LUMA | capi.SLICE_SAO_CHROMA
        if n_slices == 1 or rng.random() < 0.5:
            f |= capi.SLICE_LF_ACROSS_SLICES
        if slice_deblock_off_frac and rng.random() < slice_deblock_off_frac:
            f |= capi.SLICE_DEBLOCK_DISABLED
        if slice_sao_off_frac:
            if rng.random() < slice_sao_off_frac:
                f &= ~capi.SLICE_SAO_LUMA
            if rng.random() < slice_sao_off_frac:
                f &= ~capi.SLICE_SAO_CHROMA
        slices[i]["flags"] = f
        ctb_slice[np.array(ctb_order[bounds[i]:bounds[i + 1]])] = i

    # ---- weights ----
    weights = np.zeros(0, WT_DT)
    if weighted and pic_type != "I":
        nw = 4
        weights = np.zeros(nw, WT_DT)
        shift1, shift1_c = max(2, 14 - bit_depth), max(2, 14 - bd_c)
        o_scale = np.array([1 << (bit_depth - 8), 1 << (bd_c - 8), 1 << (bd_c - 8)])  # per plane: luma, Cb, Cr
        for i in range(nw):
            if weight_range == "spec":  # pred_weight_table: delta weights and offsets in [-128, 127] (offsets in 8-bit units)
                dl, dc = int(rng.integers(0, 8)), int(rng.integers(0, 8))
                weights[i]["w"] = rng.integers(-128, 128, size=(2, 3)) + np.array([1 << dl, 1 << dc, 1 << dc])
                weights[i]["o"] = rng.integers(-128, 128, size=(2, 3)) * o_scale
            else:
                assert weight_range == "narrow"
                weights[i]["w"] = rng.integers(-40, 120, size=(2, 3))
                weights[i]["o"] = rng.integers(-20, 21, size=(2, 3)) * o_scale
                dl, dc = int(rng.integers(0, 8)), int(rng.integers(0, 8))
            weights[i]["log2wd_luma"] = dl + shift1
            weights[i]["log2wd_chroma"] = dc + shift1_c
        if weight_range == "spec":  # the extremes on every plane and list: entry 0 lowest, entry 1 highest, entries 2/3 mixed
            weights[0]["w"], weights[0]["o"] = -128, -128 * o_scale
            weights[1]["w"], weights[1]["o"] = 255, 127 * o_scale
            weights[2]["w"][0], weights[2]["w"][1] = [255, -128, 255], [-128, 255, -128]
            weights[3]["o"][0], weights[3]["o"][1] = [127, -128, 127] * o_scale, [-128, 127, -128] * o_scale

    scaling = None
    if scaling_list == "default":
        scaling = default_scaling_factors()
    elif scaling_list == "max":
        scaling = max_scaling_factors(rng)
    elif scaling_list:
        assert scaling_list is True, scaling_list
        scaling = rng.integers(1, 64, size=capi.SCALING_FACTOR_BYTES).astype(np.uint8)
        scaling[rng.random(capi.SCALING_FACTOR_BYTES) < 0.5] = 16

    # ---- per-4x4 maps used for availability / deblocking ----
    is_intra = np.zeros((h4, w4), np.bool_)
    nz = np.zeros((h4, w4), np.bool_)          # TU has non-zero luma coefficients
    tu_edge_v = np.zeros((h4, w4), np.bool_)   # left border of the unit is a transform edge
    tu_edge_h = np.zeros((h4, w4), np.bool_)
    pu_edge_v = np.zeros((h4, w4), np.bool_)
    pu_edge_h = np.zeros((h4, w4), np.bool_)
    mvmap = np.zeros((h4, w4, 6), np.int32)    # ref0, ref1 (-1 unused), mv0x, mv0y, mv1x, mv1y
    mvmap[:, :, 0:2] = -1
    qp_map = np.zeros((h8, w8), np.int8)
    nofilt = np.zeros((h8, w8), np.uint8)

    pus, tus, co_pos, co_lvl = [], [], [], []
    n_coeff_total = [0]

    def gen_coeffs(nT, qp, special):
        """Returns (positions, levels) of a TU: mostly sparse low-frequency, sometimes dense / extreme (one DC level with
        ``coeff_max``)."""
        if coeff_max is not None:
            lv = int(rng.integers(1, coeff_max + 1)) * (1 if rng.random() < 0.5 else -1)
            return np.zeros(1, np.uint16), np.array([lv], np.int16)
        r = rng.random()
        if r < 0.70:
            n = int(rng.integers(1, max(2, nT)))  # sparse
            lim = max(2, nT // 2)
            xs = np.minimum(rng.geometric(0.45, n) - 1, lim - 1)
            ys = np.minimum(rng.geometric(0.45, n) - 1, lim - 1)
            pos = np.unique(xs + ys * nT)
            lv = rng.integers(-12, 13, len(pos))
        elif r < 0.95:
            n = int(rng.integers(nT, nT * nT // 2 + 1))
            pos = rng.choice(nT * nT, size=n, replace=False)
            lv = rng.integers(-200, 201, n)
        else:
            n = nT * nT
            pos = np.arange(n)
            lv = rng.integers(-2048, 2049, n) if rng.random() < 0.7 else rng.integers(-32768, 32768, n)
        lv = np.where(lv == 0, 1, lv)
        return pos.astype(np.uint16), lv.astype(np.int16)

    def avail_mask(xB, yB, nT, cidx, ctb_addr, cur_slice):
        """intrapred.h:436-633: picture bounds, slice and tile of the neighbouring CTB, coding order of the min-TB."""
        sh = 1 if cidx else 0
        xL, yL = xB << sh, yB << sh
        cur_z = (int(ts_of[ctb_addr]) << 8) + int(_Z[(yL & (S - 1)) >> 2, (xL & (S - 1)) >> 2])

        def ok(xn, yn):  # luma coordinates of the neighbour sample
            if xn < 0 or yn < 0 or xn >= width or yn >= height:
                return False
            ca = (xn >> log2_ctb) + (yn >> log2_ctb) * wctb
            if ctb_slice[ca] != cur_slice or ctb_tile[ca] != ctb_tile[ctb_addr]:
                return False
            if (int(ts_of[ca]) << 8) + int(_Z[(yn & (S - 1)) >> 2, (xn & (S - 1)) >> 2]) > cur_z:
                return False
            return not constrained_intra or bool(is_intra[yn >> 2, xn >> 2])

        m = 0
        n_bottom = min(2 * nT, ((height - (yB << sh)) + sh) >> sh)
        n_right = min(2 * nT, ((width - (xB << sh)) + sh) >> sh)
        for k in range(nT // 2):  # left groups: rows 4k..4k+3, tested at the group's last row
            y = 4 * k + 3
            if y < n_bottom and ok((xB - 1) << sh, (yB + y) << sh):
                m |= 1 << k
        if ok((xB - 1) << sh, (yB - 1) << sh):
            m |= 1 << capi.AVAIL_CORNER_BIT
        top_right_ok = (xL + (nT << sh)) < width
        for k in range(nT // 2):  # top groups: columns 4k..4k+3, tested at the group's first column
            x = 4 * k
            if x >= n_right or (x >= nT and not top_right_ok):
                continue
            if ok((xB + x) << sh, (yB - 1) << sh):
                m |= 1 << (capi.AVAIL_TOP_BIT0 + k)
        return m

    def emit_tu(x, y, log2, cidx, flags, mode, qp, avail, pos=None, lv=None):
        n = 0 if pos is None else len(pos)
        tus.append((x, y, log2, cidx, flags, mode, qp, n, n_coeff_total[0], avail))
        if n:
            co_pos.append(pos)
            co_lvl.append(lv)
            n_coeff_total[0] += n

    def qp_primes(qpy):
        qpi_cb = min(max(qpy + cb_off, -bdoff_c), 57)
        qpi_cr = min(max(qpy + cr_off, -bdoff_c), 57)
        return qpy + bdoff, max(0, _table8_22(qpi_cb) + bdoff_c), max(0, _table8_22(qpi_cr) + bdoff_c)

    def tu_block(x, y, log2, cidx, intra, mode, qp, bypass, ctb_addr, cur_slice, cu_intra):
        """One decode_TU call; returns True when coefficients were coded."""
        nT = 1 << log2
        flags = 0
        avail = 0
        if intra:
            flags |= capi.TU_INTRA
            avail = avail_mask(x, y, nT, cidx, ctb_addr, cur_slice)
            if no_bfilter_on_bypass and bypass:
                flags |= capi.TU_NO_BOUNDARY_FILTER
        cbf = rng.random() < cbf_prob
        pos = lv = None
        if cbf:
            flags |= capi.TU_CBF
            pos, lv = gen_coeffs(nT, qp, False)
            if bypass:
                flags |= capi.TU_BYPASS
                lv = np.clip(lv, -255, 255).astype(np.int16)
            elif log2 <= tskip_max_log2 and rng.random() < special_frac * 4:
                flags |= capi.TU_TSKIP
            if no_bfilter_on_bypass and intra and (flags & (capi.TU_BYPASS | capi.TU_TSKIP)) and mode in (10, 26):
                flags |= capi.TU_RDPCM_H if mode == 10 else capi.TU_RDPCM_V  # implicit RDPCM (transform.cc:425-432)
            elif flags & (capi.TU_BYPASS | capi.TU_TSKIP):
                if rng.random() < rdpcm_frac:
                    flags |= capi.TU_RDPCM_H if rng.random() < 0.5 else capi.TU_RDPCM_V
                if nT == 4 and cu_intra and rng.random() < rotate_frac:
                    flags |= capi.TU_ROTATE
            if nT == 4 and cidx == 0 and cu_intra and not (flags & (capi.TU_BYPASS | capi.TU_TSKIP)):
                flags |= capi.TU_DST
            if scaling_list and not bypass:
                flags |= capi.TU_SCALING_LIST | (0 if cu_intra else capi.TU_INTER_MATRIX)
        if intra or cbf:
            emit_tu(x, y, log2, cidx, flags, mode, qp, avail, pos, lv)
        return cbf

    def transform_tree(x, y, log2, depth, cu, blk_idx, xbase, ybase):
        """read_transform_tree / read_transform_unit ordering (slice.cc:3584-3870)."""
        intra, lmode_of, cmode, qps, bypass, ctb_addr, cur_slice, max_depth, _nxn = cu
        size = 1 << log2
        split = log2 > 5 or (log2 > 2 and depth < max_depth and rng.random() < (0.5 if intra else 0.35))
        if cu[0] and cu[8] and depth == 0:  # intra NxN: forced split at depth 0
            split = True
        if split:
            h = size >> 1
            for i, (dx, dy) in enumerate(((0, 0), (h, 0), (0, h), (h, h))):
                transform_tree(x + dx, y + dy, log2 - 1, depth + 1, cu, i, x, y)
            return
        tu_edge_v[y >> 2:(y + size) >> 2, x >> 2] = True
        tu_edge_h[y >> 2, x >> 2:(x + size) >> 2] = True
        cbf_l = tu_block(x, y, log2, 0, intra, lmode_of(x, y), qps[0], bypass, ctb_addr, cur_slice, intra)
        if cbf_l:
            nz[y >> 2:(y + size) >> 2, x >> 2:(x + size) >> 2] = True
        if not chroma_format_idc:  # 4:0:0: no chroma TUs
            return
        if log2 > 2:
            tu_block(x >> 1, y >> 1, log2 - 1, 1, intra, cmode, qps[1], bypass, ctb_addr, cur_slice, intra)
            tu_block(x >> 1, y >> 1, log2 - 1, 2, intra, cmode, qps[2], bypass, ctb_addr, cur_slice, intra)
        elif blk_idx == 3:
            tu_block(xbase >> 1, ybase >> 1, 2, 1, intra, cmode, qps[1], bypass, ctb_addr, cur_slice, intra)
            tu_block(xbase >> 1, ybase >> 1, 2, 2, intra, cmode, qps[2], bypass, ctb_addr, cur_slice, intra)

    def rand_mv():
        if mv_step is not None:
            return 4 * mv_step * int(rng.integers(-2, 3)), 4 * mv_step * int(rng.integers(-2, 3))
        r = rng.random()
        if r < far_mv_frac:
            return int(rng.integers(-4 * width, 4 * width)), int(rng.integers(-4 * height, 4 * height))
        if r < 0.15:
            return 4 * int(rng.integers(-16, 17)), 4 * int(rng.integers(-16, 17))  # integer position
        return int(rng.integers(-256, 257)), int(rng.integers(-256, 257))

    def extreme_mv(pos, size, extent, pad, cpad):
        """One MV component of a PU at `pos`: an int16 extreme, or the MC window (first tap: pos + int - 3 in luma,
        pos / 2 + int - 1 in chroma) one sample before / on / after the rim of the slot's reference border, any phase."""
        r = int(rng.integers(0, 6))
        if r < 2:
            return (-32768, 32767)[r]
        side, d = int(rng.integers(0, 2)), int(rng.integers(-1, 2))
        if r < 4:  # luma rims: -pad and extent + pad - 23 (the last window origin that fits)
            t = (-pad if side == 0 else extent + pad - 23) + d
            mv = 4 * (t + 3 - pos) + int(rng.integers(0, 4))
        else:  # chroma rims: -cpad and extent / 2 + cpad - 11
            t = (-cpad if side == 0 else extent // 2 + cpad - 11) + d
            mv = 8 * (t + 1 - (pos >> 1)) + int(rng.integers(0, 8))
        return int(np.clip(mv, -32768, 32767))

    def emit_pu(x, y, w, h):
        small = (w + h) == 12  # 8x4 / 4x8: uni-prediction only
        bi = pic_type == "B" and not small and rng.random() < 0.5
        lists = (0, 1) if bi else ((0,) if pic_type == "P" or rng.random() < 0.5 else (1,))
        flags, ref, mv = 0, [-1, -1], [[0, 0], [0, 0]]
        for l in lists:
            flags |= 1 << l
            ref[l] = int(ref_slots[int(rng.integers(0, len(ref_slots)))])
            if rng.random() < 0.003:
                ref[l] = -1  # missing reference -> mid-grey
            mv[l] = list(rand_mv())
            if extreme_mv_frac and (x == 0 or y == 0 or x + w >= width or y + h >= height) and rng.random() < extreme_mv_frac:
                mv[l] = [extreme_mv(x, w, width, _PAD_X, _PAD_CX), extreme_mv(y, h, height, _PAD_Y, _PAD_CY)]
        wt = 0
        if len(weights):
            flags |= capi.PU_WEIGHTED
            wt = int(rng.integers(0, len(weights)))
        pus.append((x, y, w, h, flags, 0, ref, wt, mv, 0))
        pu_edge_v[y >> 2:(y + h) >> 2, x >> 2] = True
        pu_edge_h[y >> 2, x >> 2:(x + w) >> 2] = True
        mvmap[y >> 2:(y + h) >> 2, x >> 2:(x + w) >> 2] = [ref[0], ref[1], mv[0][0], mv[0][1], mv[1][0], mv[1][1]]

    def coding_unit(x, y, log2, ctb_addr, cur_slice):
        size = 1 << log2
        qpy = int(rng.integers(qp_range[0], qp_range[1] + 1))
        qp_map[y >> 3:(y + size) >> 3, x >> 3:(x + size) >> 3] = qpy
        intra = rng.random() < intra_frac
        bypass = rng.random() < special_frac
        qps = qp_primes(qpy)
        if bypass:
            nofilt[y >> 3:(y + size) >> 3, x >> 3:(x + size) >> 3] = 1
        if intra and log2 <= 5 and rng.random() < special_frac:  # PCM CU
            is_intra[y >> 2:(y + size) >> 2, x >> 2:(x + size) >> 2] = True
            tu_edge_v[y >> 2:(y + size) >> 2, x >> 2] = True
            tu_edge_h[y >> 2, x >> 2:(x + size) >> 2] = True
            if pcm_lf_disable:  # the host folds pcm_loop_filter_disable into the no-filter map
                nofilt[y >> 3:(y + size) >> 3, x >> 3:(x + size) >> 3] = 1
            for c in range(3 if chroma_format_idc else 1):
                s = size if c == 0 else size >> 1
                n = s * s
                lv = rng.integers(0, 1 << (bd_c if c else bit_depth), n).astype(np.int16)
                emit_tu(x >> (1 if c else 0), y >> (1 if c else 0), log2 - (1 if c else 0), c, capi.TU_PCM, 0, 0, 0, np.arange(n, dtype=np.uint16), lv)
            return
        if intra:
            is_intra[y >> 2:(y + size) >> 2, x >> 2:(x + size) >> 2] = True
            nxn = log2 == 3 and rng.random() < 0.4
            if nxn:
                modes = [int(rng.integers(0, 35)) for _ in range(4)]
                h = size >> 1
                lmode_of = lambda tx, ty: modes[(1 if tx >= x + h else 0) + (2 if ty >= y + h else 0)]
                base = modes[0]
            else:
                m0 = int(rng.integers(0, 35))
                lmode_of = lambda tx, ty: m0
                base = m0
            cmode = [0, 26, 10, 1, base][int(rng.integers(0, 5))]
            cu = (True, lmode_of, cmode, qps, bypass, ctb_addr, cur_slice, 2 if log2 > 3 else 1, nxn)
            transform_tree(x, y, log2, 0, cu, 0, x, y)
            return
        # inter CU: PartMode
        r = rng.random()
        if log2 == 3:
            part = "2Nx2N" if r < 0.84 else ("2NxN" if r < 0.92 else "Nx2N")
        else:
            part = "2Nx2N" if r < 0.6 else ["2NxN", "Nx2N", "2NxnU", "2NxnD", "nLx2N", "nRx2N"][int(rng.integers(0, 6))]
        h2, q = size >> 1, size >> 2
        rects = {"2Nx2N": [(0, 0, size, size)], "2NxN": [(0, 0, size, h2), (0, h2, size, h2)], "Nx2N": [(0, 0, h2, size), (h2, 0, h2, size)],
                 "2NxnU": [(0, 0, size, q), (0, q, size, size - q)], "2NxnD": [(0, 0, size, size - q), (0, size - q, size, q)],
                 "nLx2N": [(0, 0, q, size), (q, 0, size - q, size)], "nRx2N": [(0, 0, size - q, size), (size - q, 0, q, size)]}[part]
        for dx, dy, w, h in rects:
            emit_pu(x + dx, y + dy, w, h)
        if rng.random() < 0.7:  # rqt_root_cbf
            cu = (False, lambda tx, ty: 0, 0, qps, bypass, ctb_addr, cur_slice, 2, False)
            transform_tree(x, y, log2, 0, cu, 0, x, y)
        else:
            tu_edge_v[y >> 2:(y + size) >> 2, x >> 2] = True
            tu_edge_h[y >> 2, x >> 2:(x + size) >> 2] = True

    # cumulative split probabilities from the area shares: p(split at size s) = area coded below s / area reaching s
    a64, a32, a16, a8 = size_area
    tot = a64 + a32 + a16 + a8
    a64, a32, a16, a8 = a64 / tot, a32 / tot, a16 / tot, a8 / tot
    p_split = {6: 1 - a64, 5: (a16 + a8) / max(1e-9, a32 + a16 + a8), 4: a8 / max(1e-9, a16 + a8), 3: 0.0}

    def coding_quadtree(x, y, log2, ctb_addr, cur_slice):
        size = 1 << log2
        if x >= width or y >= height:
            return
        must = x + size > width or y + size > height
        if log2 > 3 and (must or rng.random() < p_split[log2]):
            h = size >> 1
            for dx, dy in ((0, 0), (h, 0), (0, h), (h, h)):
                coding_quadtree(x + dx, y + dy, log2 - 1, ctb_addr, cur_slice)
        else:
            coding_unit(x, y, log2, ctb_addr, cur_slice)

    for ca in ctb_order:
        coding_quadtree((ca % wctb) * S, (ca // wctb) * S, log2_ctb, ca, int(ctb_slice[ca]))

    pus_a = np.array([(a, b, c, d, e, f, tuple(g), h, tuple(map(tuple, i)), j) for a, b, c, d, e, f, g, h, i, j in pus], PU_DT) if pus else np.zeros(0, PU_DT)
    tus_a = np.array(tus, TU_DT) if tus else np.zeros(0, TU_DT)
    coeffs = np.zeros(n_coeff_total[0], CO_DT)
    if co_pos:
        coeffs["pos"] = np.concatenate(co_pos)
        coeffs["level"] = np.concatenate(co_lvl)

    # ---- boundary strength (deblock.cc:243-383) on the generated structure ----
    bs = np.zeros((h4, w4), np.uint8)
    if deblock:
        for vertical in (True, False):
            te, pe = (tu_edge_v, pu_edge_v) if vertical else (tu_edge_h, pu_edge_h)
            edge = te | pe
            if vertical:
                edge[:, 0] = False
                if not lf_across_tiles:  # filterLeftCbEdge = 0 on tile borders (deblock.cc:196-203)
                    for cb in col_bd[1:-1]:
                        edge[:, (cb * S) >> 2] = False
            else:
                edge[0, :] = False
                if not lf_across_tiles:
                    for rb in row_bd[1:-1]:
                        edge[(rb * S) >> 2, :] = False

            def shift(a):  # value of the P-side unit (left / above)
                r = np.empty_like(a)
                if vertical:
                    r[:, 1:] = a[:, :-1]
                    r[:, 0] = a[:, 0]
                else:
                    r[1:] = a[:-1]
                    r[0] = a[0]
                return r

            ip, nzp, mp = shift(is_intra), shift(nz), shift(mvmap)
            mq = mvmap
            rp0, rp1, rq0, rq1 = mp[..., 0], mp[..., 1], mq[..., 0], mq[..., 1]

            def big(i, j):  # |mvP_i - mvQ_j| >= 4 in x or y (unused lists count as mv 0)
                px = np.where(mp[..., i] >= 0, mp[..., 2 + 2 * i], 0)
                py = np.where(mp[..., i] >= 0, mp[..., 3 + 2 * i], 0)
                qx = np.where(mq[..., j] >= 0, mq[..., 2 + 2 * j], 0)
                qy = np.where(mq[..., j] >= 0, mq[..., 3 + 2 * j], 0)
                return (np.abs(px - qx) >= 4) | (np.abs(py - qy) >= 4)

            same = ((rp0 == rq0) & (rp1 == rq1)) | ((rp0 == rq1) & (rp1 == rq0))
            straight = big(0, 0) | big(1, 1)
            cross = big(0, 1) | big(1, 0)
            mvdiff = np.where(rp0 != rp1, np.where(rp0 == rq0, straight, cross), straight & cross)
            b = np.where(ip | is_intra, 2, np.where(te & (nzp | nz), 1, np.where(~same | mvdiff, 1, 0)))
            b = np.where(edge, b, 0).astype(np.uint8)
            bs |= b if vertical else (b << 2)
        if slice_deblock_off_frac:  # deblock.cc:215: a slice with deblocking off marks no edge of its CUs (the Q side)
            off = (slices["flags"] & capi.SLICE_DEBLOCK_DISABLED) != 0
            ys, xs = np.mgrid[0:h4, 0:w4]
            bs[off[ctb_slice[((xs * 4) >> log2_ctb) + ((ys * 4) >> log2_ctb) * wctb]]] = 0

    # ---- SAO ----
    ctbs = np.zeros(n_ctb, CTB_DT)
    ctbs["slice_idx"] = ctb_slice
    ctbs["tile_id"] = ctb_tile
    if sao:
        lim, lim_c = 7 if bit_depth == 8 else 31, 7 if bd_c == 8 else 31
        for i in range(n_ctb):
            tl, tc = int(rng.integers(0, 3)), int(rng.integers(0, 3))
            cl, cc = int(rng.integers(0, 4)), int(rng.integers(0, 4))
            ctbs[i]["sao_type"] = tl | (tc << 2) | (tc << 4)
            ctbs[i]["sao_eo_class"] = cl | (cc << 2) | (cc << 4)
            ctbs[i]["sao_band_pos"] = rng.integers(sao_band_pos[0], sao_band_pos[1], 3)
            if lim == lim_c:
                off = rng.integers(-lim, lim + 1, (3, 4))
            else:
                off = rng.integers(-np.array([[lim], [lim_c], [lim_c]]), np.array([[lim], [lim_c], [lim_c]]) + 1, (3, 4))
            if sao_offset == "max":  # SaoOffsetVal at the largest magnitude the depth allows (sao_offset_abs << log2_sao_offset_scale)
                for c, bd in enumerate((bit_depth, bd_c, bd_c)):
                    mag = ((1 << (min(bd, 10) - 5)) - 1) << int(rng.integers(0, max(0, bd - 10) + 1))
                    off[c] = np.where(off[c] < 0, -mag, mag)
            else:
                assert sao_offset == "random"
            for c, t in enumerate((tl, tc, tc)):
                if t == 2:  # edge offsets: first two >= 0, last two <= 0
                    off[c] = [abs(off[c][0]), abs(off[c][1]), -abs(off[c][2]), -abs(off[c][3])]
            ctbs[i]["sao_offset"] = off

    return SynthPicture(params, pus_a, weights, tus_a, coeffs, slices, ctbs, np.ascontiguousarray(bs.reshape(-1)),
                        np.ascontiguousarray(qp_map.reshape(-1)), np.ascontiguousarray(nofilt.reshape(-1)), scaling)


def random_planes(width, height, bit_depth, seed, bit_depth_chroma=None, chroma_format_idc=1):
    """Random reference picture (xorshift-like seeded noise with some smooth structure).  4:0:0: the luma plane only (the
    same samples as the 4:2:0 picture's luma); chroma samples lie in [0, 2^bit_depth_chroma)."""
    rng = np.random.default_rng(seed)
    dt = np.uint16 if bit_depth > 8 else np.uint8
    planes = []
    for c in range(3 if chroma_format_idc else 1):
        maxv = (1 << (bit_depth if c == 0 or bit_depth_chroma is None else bit_depth_chroma)) - 1
        w, h = (width, height) if c == 0 else (width // 2, height // 2)
        base = rng.integers(0, maxv + 1, (h // 8 + 1, w // 8 + 1))
        img = np.kron(base, np.ones((8, 8), np.int64))[:h, :w] + rng.integers(-40, 41, (h, w))
        ext = rng.random((h, w)) < 0.02  # sprinkle extremes (0 / max) to exercise the int16 wrap of App. A.1
        img = np.where(ext, rng.integers(0, 2, (h, w)) * maxv, img)
        planes.append(np.ascontiguousarray(np.clip(img, 0, maxv).astype(dt)))
    return planes


def smooth_planes(width, height, bit_depth, seed, steps, bit_depth_chroma=None, chroma_format_idc=1, spikes=()):
    """Piecewise-smooth reference picture: a gentle ramp over the whole plane (from below 0 to above the maximum, so both
    clip levels occur) plus a level per 8x8 block that changes from block to block by one of ``steps`` (8-bit units, scaled
    by 2^(bd - 8); random sign, drawn towards 0 so the levels stay bounded), and on a quarter of the blocks a small texture.
    The steps sit on the 8x8 grid where deblocking edges lie; choosing them relative to tc and beta at the case's QP makes
    the filters' off / strong / weak / cut-off outcomes all occur.  ``spikes``: heights (8-bit units) of single-sample spikes
    on a quarter of the samples at x % 4 and y % 4 in {1, 2}: the deblocking decisions read lines 0 and 3 of an edge segment
    only, so a spike on line 1 or 2 is filtered as the calm lines decide, and the strong filter's +-2 tc clamps decide the
    result (MVs on a 16-sample grid keep the spikes on those lines)."""
    rng = np.random.default_rng(seed)
    dt = np.uint16 if bit_depth > 8 else np.uint8
    steps = np.asarray(steps, np.int64)
    planes = []
    for c in range(3 if chroma_format_idc else 1):
        bd = bit_depth if c == 0 or bit_depth_chroma is None else bit_depth_chroma
        maxv, sc = (1 << bd) - 1, 1 << (bd - 8)
        w, h = (width, height) if c == 0 else (width // 2, height // 2)
        bw, bh = (w + 7) // 8, (h + 7) // 8

        def walk(n):  # block levels along one axis: steps from the set, signs pulled back towards 0
            lv = np.zeros(n, np.int64)
            for i in range(1, n):
                d = int(steps[rng.integers(0, len(steps))]) * sc
                lv[i] = lv[i - 1] + (-d if (lv[i - 1] > 0) == (rng.random() < 0.75) else d)
            return lv
        blocks = walk(bw)[None, :] + walk(bh)[:, None]
        ang = rng.uniform(0, 2 * np.pi)
        ys, xs = np.mgrid[0:h, 0:w]
        t = (xs * np.cos(ang) + ys * np.sin(ang)) / max(1.0, abs(w * np.cos(ang)) + abs(h * np.sin(ang)))
        t -= t.min()
        ramp = (-0.1 + 1.2 * t / max(t.max(), 1e-9)) * maxv
        tex = np.kron(rng.random((bh, bw)) < 0.25, np.ones((8, 8), bool))[:h, :w] * rng.integers(-2 * sc, 2 * sc + 1, (h, w))
        img = np.rint(ramp).astype(np.int64) + np.kron(blocks, np.ones((8, 8), np.int64))[:h, :w] + tex
        if len(spikes):
            at = (rng.random((h, w)) < 0.25) & np.isin(ys % 4, (1, 2)) & np.isin(xs % 4, (1, 2))
            img += at * rng.choice(np.asarray(spikes, np.int64) * sc, (h, w)) * rng.choice([-1, 1], (h, w))
        planes.append(np.ascontiguousarray(np.clip(img, 0, maxv).astype(dt)))
    return planes
