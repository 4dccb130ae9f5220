"""Restatement of the RGB export's arithmetic (libde265_b200/csrc/export.cuh) in numpy: the integer formula, exactly, and the
float64 definition it approximates.  Shared by test_cpu_export.py and test_gpu_export.py."""
import math

import numpy as np

MATRICES = {1: (0.299, 0.114), 2: (0.2126, 0.0722), 3: (0.2627, 0.0593)}  # B200_EXPORT_RGB_BT601 / 709 / 2020: (Kr, Kb)
RGB_NAMES = {"bt601": 1, "bt709": 2, "bt2020": 3}


def ranges(full_range, bd_y, bd_c):
    """(oY, rangeY, oC, rangeC)"""
    if full_range:
        return 0, (1 << bd_y) - 1, 1 << (bd_c - 1), (1 << bd_c) - 1
    return 16 << (bd_y - 8), 219 << (bd_y - 8), 1 << (bd_c - 1), 224 << (bd_c - 8)


def weights(matrix):
    """k per (channel, input): rows R, G, B; columns Y, Cb, Cr."""
    kr, kb = MATRICES[matrix]
    kg = 1.0 - kr - kb
    return ((1.0, 0.0, 2.0 * (1.0 - kr)),
            (1.0, -2.0 * kb * (1.0 - kb) / kg, -2.0 * kr * (1.0 - kr) / kg),
            (1.0, 2.0 * (1.0 - kb), 0.0))


def coefs(matrix, full_range, bd_y, bd_c):
    """The integer coefficients, in export_emul_coefs's order: y, r_cr, g_cb, g_cr, b_cb, oy, oc."""
    oy, ry, oc, rc = ranges(full_range, bd_y, bd_c)
    k = weights(matrix)
    q = lambda kk, r: int(math.floor(65536.0 * 255.0 * kk / r + 0.5))  # noqa: E731
    return [q(1.0, ry), q(k[0][2], rc), q(k[1][1], rc), q(k[1][2], rc), q(k[2][1], rc), oy, oc]


def rgb_int(matrix, full_range, bd_y, bd_c, y, cb, cr):
    """uint8 array (..., 3) from sample arrays of one shape: the integer formula."""
    cy, r_cr, g_cb, g_cr, b_cb, oy, oc = coefs(matrix, full_range, bd_y, bd_c)
    ty = cy * (np.asarray(y, np.int64) - oy) + (1 << 15)
    u, v = np.asarray(cb, np.int64) - oc, np.asarray(cr, np.int64) - oc
    out = [(ty + r_cr * v) >> 16, (ty + g_cb * u + g_cr * v) >> 16, (ty + b_cb * u) >> 16]
    return np.clip(np.stack(out, -1), 0, 255).astype(np.uint8)


def rgb_float(matrix, full_range, bd_y, bd_c, y, cb, cr):
    """float64 array (..., 3): the definition, clamped to [0, 255] and not rounded."""
    oy, ry, oc, rc = ranges(full_range, bd_y, bd_c)
    yn = (np.asarray(y, np.float64) - oy) / ry
    u, v = (np.asarray(cb, np.float64) - oc) / rc, (np.asarray(cr, np.float64) - oc) / rc
    out = [255.0 * (k[0] * yn + k[1] * u + k[2] * v) for k in weights(matrix)]
    return np.clip(np.stack(out, -1), 0.0, 255.0)


def rgb_planes(matrix, full_range, bd_y, bd_c, planes, crop=None):
    """(3, h, w) uint8 from read_slot-style planes [Y, Cb, Cr] (or [Y]: 4:0:0, chroma at the mid-point): nearest chroma."""
    Y = planes[0]
    x, y, w, h = crop if crop is not None else (0, 0, Y.shape[1], Y.shape[0])
    ys = Y[y:y + h, x:x + w]
    if len(planes) == 1:
        cb = cr = np.full(ys.shape, 1 << (bd_c - 1), np.int64)
    else:
        rows, cols = (np.arange(y, y + h) >> 1)[:, None], (np.arange(x, x + w) >> 1)[None, :]
        cb, cr = planes[1][rows, cols], planes[2][rows, cols]
    return np.moveaxis(rgb_int(matrix, full_range, bd_y, bd_c, ys, cb, cr), -1, 0)
