"""k_intra's small-TU prediction plans without a GPU: the table engine.cu builds (intra_plan_words in
libde265_b200/csrc/kernels_recon.cuh, compiled for the host by tests/intra_plan_emul.cu) executed class by class with a plain
restatement of tu_intra_fast's consumer, against the oracle's border / filter / prediction (pinned to the reference by
test_oracle_vs_ref.py); the clamp rule the fast path rests on, over every availability mask; and proof from the records that
the pictures test_gpu_intra_plans.py runs reach every reachable class, and the boundary filter's clip on both sides."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import intra_plan_cases as ipc
from libde265_b200 import capi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libintra_plan_emul.so")
SRC = os.path.join(HERE, "intra_plan_emul.cu")
CSRC = os.path.join(ROOT, "libde265_b200", "csrc")

u16p = C.POINTER(C.c_uint16)


def build_emulator():
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("kernels_recon.cuh", "kernels_residual.cuh", "dev_common.cuh")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", SO, SRC])


@pytest.fixture(scope="module")
def table():
    """g_intra_plan as init_tables fills it: [class][slot * 32 + lane]."""
    build_emulator()
    lib = C.CDLL(SO)
    lib.intra_plan_words.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_uint32)]
    assert lib.intra_plan_classes() == ipc.INTRA_PLAN_CLASSES
    ts = lib.intra_plan_tile_stride()
    out = np.zeros((ipc.INTRA_PLAN_CLASSES, 64), np.uint32)
    w = (C.c_uint32 * 2)()
    for cls in sorted(ipc.ENCODABLE):
        for lane in range(32):
            assert lib.intra_plan_words(cls, lane, w) == 0
            out[cls, lane], out[cls, lane + 32] = w[0], w[1]
    return out, ts


@pytest.fixture(scope="module")
def orc(oracle_mod):
    lib = oracle_mod.oracle()
    lib.orc_intra_border.argtypes = [u16p, u16p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_int]
    lib.orc_intra_filter.argtypes = [u16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.orc_intra_pred.argtypes = [u16p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, u16p, C.c_int, C.c_int]
    return lib


def avail_mask(nT, lo, hi, bl=None, tr=None):
    """The mask with the TU's own column, corner and row available and the bottom-left / top-right groups that give [lo, hi]
    (or the explicit group bits bl / tr)."""
    q = nT // 4
    bl = (1 << ((-lo - nT) // 4)) - 1 if bl is None else bl
    tr = (1 << ((hi - nT) // 4)) - 1 if tr is None else tr
    g = (1 << q) - 1
    return g | bl << q | 1 << capi.AVAIL_CORNER_BIT | g << capi.AVAIL_TOP_BIT0 | tr << (capi.AVAIL_TOP_BIT0 + q)


PLANE = 80  # plane of the oracle's border gather: the TU at (XB, YB), every reach inside up to nT = 32
XB = YB = 8


def plane_with_border(raw, nT):
    """A plane whose neighbour samples of the TU at (XB, YB) are raw[i + 2nT] = border[i], i in [-2nT, 2nT]; mid-grey elsewhere."""
    p = np.full((PLANE, PLANE), 77, np.uint16)
    for r in range(2 * nT):
        p[YB + r, XB - 1] = raw[2 * nT - r - 1]
    p[YB - 1, XB - 1] = raw[2 * nT]
    p[YB - 1, XB:XB + 2 * nT] = raw[2 * nT + 1:]
    return p


def oracle_border(orc, plane, nT, avail, bd):
    """orc_intra_border: a 129 + 2 sample buffer whose index 66 is border[0]."""
    buf = np.zeros(4 * 32 + 5, np.uint16)
    ptr = C.cast(buf.ctypes.data + 2 * 66, u16p)
    orc.orc_intra_border(ptr, plane.ctypes.data_as(u16p), PLANE, XB, YB, nT, avail, bd)
    return buf, ptr


def oracle_prediction(orc, cls, raw, bd):
    nT, mode, lo, hi, smooth, bfilt, luma = ipc.decode(cls)
    plane = plane_with_border(raw, nT)
    buf, ptr = oracle_border(orc, plane, nT, avail_mask(nT, lo, hi), bd)
    if smooth:
        orc.orc_intra_filter(ptr, nT, 0 if luma else 1, mode, 1, bd)
    dst = np.zeros((nT, nT), np.uint16)
    orc.orc_intra_pred(dst.ctypes.data_as(u16p), nT, nT, 0 if luma else 1, mode, ptr, bd, 0 if bfilt else 1)
    return dst.astype(np.int64)


SENTINEL = 1 << 20  # above every sample value: any sample read outside [lo, hi] shows in the result


def plan_tile(raws, nT, lo, hi, ts):
    """Region tiles (one row per border) as tu_intra_fast sees them, flattened from the TU's sample (-1, -1): border[i] at
    -i * ts for i < 0 and at i for i >= 0, only for i in [lo, hi]; everything else the sentinel.  Also the mask of legal offsets."""
    n = (2 * nT + 1) * ts + 2 * nT + 1
    tile = np.full((len(raws), n), SENTINEL, np.int64)
    legal = np.zeros(n, bool)
    for i in range(lo, hi + 1):
        off = -i * ts if i < 0 else i
        tile[:, off] = [r[i + 2 * nT] for r in raws]
        legal[off] = True
    return tile, legal


def consume(cls, words, tile, bd):
    """tu_intra_fast restated: the prediction (rows of `tile`, nT, nT) the words give, and the tile offsets they read."""
    nT, mode, lo, hi, smooth, bfilt, luma = ipc.decode(cls)
    log2 = nT.bit_length() - 1
    NP = 1 if nT == 4 else 2  # pixel slots per lane (4x4: lanes 16..31 idle)
    w = [int(v) for v in words]  # w[lane + 32 * p]
    reads = set()

    def T(u):
        reads.add(u & 1023)
        return tile[:, u & 1023]

    def F(u):  # [1 2 1] taps
        return (T(u) + 2 * T(u >> 10) + T(u >> 20) + 2) >> 2

    out = np.zeros((tile.shape[0], nT, nT), np.int64)
    f = [F(w[lane]) for lane in range(32)] if mode == 0 else None  # planar: lane s filters border[s - nT - 1]
    dc = (sum(T(w[lane] >> 22) for lane in range(2 * nT)) + nT) >> (log2 + 1) if mode == 1 else None
    for p in range(NP):
        for lane in range(32):
            o, u = lane + 32 * p, w[lane + 32 * p]
            x, y = o & (nT - 1), (o >> log2) & (nT - 1)
            if mode == 0:
                tr, bl, left, top = f[2 * nT + 2], f[0], f[nT - y], f[nT + 2 + x]
                px = ((nT - 1 - x) * left + (x + 1) * tr + (nT - 1 - y) * top + (y + 1) * bl + nT) >> (log2 + 1)
            elif mode == 1:
                kind, a = (u >> 20) & 3, T(u)
                b = T(u >> 10) if kind == 2 else dc
                px = (a + b + 2 * dc + 2) >> 2 if kind else dc
            elif nT == 8 and smooth:
                px = F(u)
            else:
                r1, r2, fact = T(u), T(u >> 10), (u >> 20) & 31
                px = ((32 - fact) * r1 + fact * r2 + 16) >> 5
                if bfilt and u >> 31:
                    reads.add(0)
                    px = np.clip(r1 + ((r2 - tile[:, 0]) >> 1), 0, (1 << bd) - 1)
            if o < nT * nT:
                out[:, y, x] = px
    return out, reads


def borders(nT, bd, rng):
    """Random twice, 0 / max alternating both ways, and the two that drive the boundary filter below 0 and above max: flat 0
    with the corner at max, flat max with the corner at 0."""
    n, m = 4 * nT + 1, (1 << bd) - 1
    alt = np.arange(n) % 2 * m
    low, high = np.zeros(n, np.int64), np.full(n, m, np.int64)
    low[2 * nT], high[2 * nT] = m, 0
    return [rng.integers(0, m + 1, n), rng.integers(0, m + 1, n), alt, m - alt, low, high]


def test_encodable_and_reachable_sets():
    assert len(ipc.ENCODABLE) == 1008
    assert len(ipc.REACHABLE) == 730  # 767 less the 37 classes of 4x4 luma with lo -8, hi 4 (see intra_plan_cases._reachable)
    assert ipc.REACHABLE <= ipc.ENCODABLE
    assert all(ipc.decode(ipc.encode(*ipc.decode(c)[:4], *ipc.decode(c)[4:])) == ipc.decode(c) for c in ipc.ENCODABLE)


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_plan_table_against_the_oracle(table, orc, bd):
    """Every encodable class, all 32 lanes x 2 slots, six borders: the words executed as tu_intra_fast executes them equal the
    oracle's prediction, and read no tile sample outside [lo, hi]."""
    words, ts = table
    rng = np.random.default_rng(bd)
    bad = []
    for cls in sorted(ipc.ENCODABLE):
        nT, mode, lo, hi = ipc.decode(cls)[:4]
        raws = borders(nT, bd, rng)
        want = np.stack([oracle_prediction(orc, cls, r, bd) for r in raws])
        tile, legal = plan_tile(raws, nT, lo, hi, ts)
        got, reads = consume(cls, words[cls], tile, bd)
        stray = sorted(o for o in reads if not legal[o])
        if stray:
            bad.append(f"{ipc.describe(cls)}: reads tile offsets {stray[:4]} outside [lo, hi]")
        elif not (got == want).all():
            k, y, x = (int(v) for v in np.argwhere(got != want)[0])
            bad.append(f"{ipc.describe(cls)}: border {k} pixel (x={x}, y={y}) plan {got[k, y, x]} != oracle {want[k, y, x]}")
    assert not bad, f"{len(bad)} classes differ:\n" + "\n".join(bad[:20])


@pytest.mark.parametrize("nT", [4, 8, 16, 32])
def test_clamp_rule_every_mask(orc, nT):
    """Where fast_clamps (intra_border_clamps) holds, the substituted border equals the raw border with its index clamped into
    [lo, hi].  nT 4 / 8: every mask; 16 / 32: the own column, corner and row available, every bottom-left / top-right pattern."""
    q, bd = nT // 4, 10
    raw = np.random.default_rng(nT).integers(0, 1 << bd, 4 * nT + 1)
    plane = plane_with_border(raw, nT)
    idx = np.arange(-2 * nT, 2 * nT + 1)
    if nT <= 8:
        bits = list(range(2 * q)) + [capi.AVAIL_CORNER_BIT] + [capi.AVAIL_TOP_BIT0 + k for k in range(2 * q)]
        masks = [sum(1 << b for i, b in enumerate(bits) if (m >> i) & 1) for m in range(1 << len(bits))]
    else:
        masks = [avail_mask(nT, 0, 0, bl, tr) for bl in range(1 << q) for tr in range(1 << q)]
    n_fast = 0
    for m in masks:
        c = ipc.fast_clamps({"log2_size": nT.bit_length() - 1, "avail": m})
        if c is None:
            continue
        n_fast += 1
        buf, _ = oracle_border(orc, plane, nT, m, bd)
        got = buf[66 - 2 * nT:66 + 2 * nT + 1].astype(np.int64)
        want = raw[np.clip(idx, *c) + 2 * nT]
        assert (got == want).all(), f"nT {nT} mask {m:#x} clamps {c}: border differs at index {idx[np.argmax(got != want)]}"
    assert n_fast == (q + 1) ** 2  # every (bottom-left, top-right) prefix pair


@pytest.mark.parametrize("bd,bd_c", [(8, None), (10, None), (12, None), (12, 9)], ids=["8", "10", "12", "12_9"])
def test_coverage_pictures_reach_every_reachable_class(bd, bd_c):
    """Every class in REACHABLE at least twice with CBF and once without, and no other class."""
    cen = ipc.census(ipc.coverage_pictures(bd, bd_c))
    missing = sorted(c for c in ipc.REACHABLE if cen.get(c, [0, 0])[0] < 2 or cen.get(c, [0, 0])[1] < 1)
    assert not missing, f"{len(missing)} of {len(ipc.REACHABLE)} reachable classes not reached twice with CBF and once without:\n" + \
        "\n".join(f"{ipc.describe(c)}: {cen.get(c, [0, 0])}" for c in missing)
    unexpected = sorted(set(cen) - ipc.REACHABLE)
    assert not unexpected, "classes outside REACHABLE: " + ", ".join(ipc.describe(c) for c in unexpected)
    print(f"{len(ipc.REACHABLE)} reachable classes, all reached")


@pytest.mark.parametrize("bd", [8, 10])
def test_boundary_filter_clips_on_both_sides(oracle_mod, bd):
    """In the pre-deblocking samples the predictions read, the unclipped boundary-filter value of the fast-path TUs leaves
    [0, max] below and above, for 4x4 and 8x8 and modes 10 and 26."""
    pics = ipc.coverage_pictures(bd)
    recs = ipc.oracle_outputs(oracle_mod, pics, capi.STAGE_RECON)
    m = (1 << bd) - 1
    seen = {(nT, mode): [0, 0] for nT in (4, 8) for mode in ipc.BFILT_MODES}
    for p, rec in zip(pics, recs):
        Y = rec[0].astype(np.int64)
        for tu in p.tus:
            cls = ipc.plan_class(tu, p.params.flags, p.params.chroma_format_idc)
            if cls is None or not ipc.decode(cls)[5]:
                continue
            nT, mode = ipc.decode(cls)[:2]
            x0, y0 = int(tu["x"]), int(tu["y"])
            if mode == 26:
                v = Y[y0 - 1, x0] + ((Y[y0:y0 + nT, x0 - 1] - Y[y0 - 1, x0 - 1]) >> 1)
            else:
                v = Y[y0, x0 - 1] + ((Y[y0 - 1, x0:x0 + nT] - Y[y0 - 1, x0 - 1]) >> 1)
            seen[(nT, mode)][0] += int((v < 0).sum())
            seen[(nT, mode)][1] += int((v > m).sum())
    assert all(lo and hi for lo, hi in seen.values()), f"{bd} bit: pixels below 0 / above {m} per (nT, mode): {seen}"
