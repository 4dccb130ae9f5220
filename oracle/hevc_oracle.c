/*
 * hevc_oracle.c — CPU restatement of libde265's scalar reconstruction path.
 * TEST INFRASTRUCTURE ONLY — see hevc_oracle.h for the usage rules and how parity is pinned.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * /root/reference/libde265/).  This is a restatement written from the behaviour of
 * the reference, not a copy: one generic code path per operation instead of the
 * reference's per-size / per-phase / per-bit-depth instantiations.
 */
#include "hevc_oracle.h"

#include <stdlib.h>
#include <string.h>

#define MAXI(a, b) ((a) > (b) ? (a) : (b))
#define MINI(a, b) ((a) < (b) ? (a) : (b))

static inline int clip3(int lo, int hi, int v) { return v < lo ? lo : v > hi ? hi : v; }
static inline int clip_bd(int v, int bd) { int m = (1 << bd) - 1; return v < 0 ? 0 : v > m ? m : v; }
static inline int iabs(int v) { return v < 0 ? -v : v; }
static inline int ilog2(int v) { int n = 0; while (v > 1) { n++; v >>= 1; } return n; }

/* ------------------------------------------------------------------------------------------
 * Residual: dequant, inverse DCT/DST, transform skip, bypass
 * ---------------------------------------------------------------------------------------- */

/* transform.cc:358 */
static const int level_scale[6] = {40, 45, 51, 57, 64, 72};

void orc_dequant(int16_t* coeff_buf, const int16_t* levels, const uint16_t* pos, int n,
                 int qP, int bit_depth, int log2_nT, const uint8_t* sclist)
{
  /* transform.cc:452 bdShift = BitDepth + Log2(nT) - 5 ; without scaling list m=16 is folded
   * into bdShift-4 (transform.cc:461-468); the int32 and int64 paths (:473-487) agree. */
  int bd_shift = bit_depth + log2_nT - 5;
  if (!sclist) bd_shift -= 4;
  const int64_t offset = (int64_t)1 << (bd_shift - 1);
  for (int i = 0; i < n; i++) {
    int m = sclist ? sclist[pos[i]] : 1;
    int64_t fact = (int64_t)(m * level_scale[qP % 6]) << (qP / 6);
    /* transform.cc:522-523 hands the 64-bit value to Clip3(int, int, int) (util.h:89): its low 32 bits are clipped.  Only a
     * scaling factor above 16 can push the value past the int32 range. */
    int32_t v = (int32_t)(uint32_t)(((int64_t)levels[i] * fact + offset) >> bd_shift);
    if (v < -32768) v = -32768;
    if (v > 32767) v = 32767;
    coeff_buf[pos[i]] = (int16_t)v;
  }
}

/* First column of the 32-point HEVC core transform (fallback-dct.cc:512-545).  The full matrix
 * is generated from these 32 distinct magnitudes: mat[k][n] = c[k] sign-folded by the cosine
 * symmetry, i.e. mat[k][n] = C((2n+1)*k mod 128) with C(j) = round-table of 64*sqrt2*cos(j*pi/64). */
static const int8_t dct_col0[32] = {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67,
                                    64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4};
static int8_t dct_mat[32][32];
static int dct_mat_ready = 0;

static void build_dct_mat(void)
{
  if (dct_mat_ready) return;
  /* mat[k][n] = c(k) * cos((2n+1) k pi / 64) quantised exactly like the standard's table: the
   * table satisfies mat[k][n] = +-dct_col0[j] where j = ((2n+1)*k) mod 128 folded into [0,32]. */
  for (int k = 0; k < 32; k++)
    for (int n = 0; n < 32; n++) {
      int j = ((2 * n + 1) * k) % 128; /* angle in units of pi/64 */
      int sign = 1;
      if (j > 64) j = 128 - j;          /* cos(2pi - a) = cos(a) */
      if (j > 32) { j = 64 - j; sign = -1; } /* cos(pi - a) = -cos(a) */
      int v = (j == 32) ? 0 : dct_col0[j];
      if (k == 0) v = 64;
      dct_mat[k][n] = (int8_t)(sign * v);
    }
  dct_mat_ready = 1;
}

void orc_idct_add(orc_pixel* dst, ptrdiff_t stride, int nT, const int16_t* coeffs, int bit_depth)
{
  /* fallback-dct.cc:550-691: column pass with rounding 64>>7 clipped to int16 (:640), row pass
   * with shift 20-bitDepth NOT clipped (:680), then add + clip to the pixel range (:685). */
  build_dct_mat();
  const int post_shift = 20 - bit_depth;
  const int rnd2 = 1 << (post_shift - 1);
  const int fact = 32 / nT;
  int16_t g[32 * 32];
  /* zero rows / columns beyond the last significant coefficient contribute nothing; skipping them is the reference's own
   * optimisation (fallback-dct.cc:614-617,667-670) */
  int max_row = 0, max_col = 0;
  for (int j = 0; j < nT; j++)
    for (int c = 0; c < nT; c++)
      if (coeffs[c + j * nT]) { if (j > max_row) max_row = j; if (c > max_col) max_col = c; }
  for (int c = 0; c < nT; c++)
    for (int i = 0; i < nT; i++) {
      int sum = 0;
      if (c <= max_col)
        for (int j = 0; j <= max_row; j++) sum += dct_mat[fact * j][i] * coeffs[c + j * nT];
      g[c + i * nT] = (int16_t)clip3(-32768, 32767, (sum + 64) >> 7);
    }
  for (int y = 0; y < nT; y++)
    for (int i = 0; i < nT; i++) {
      int sum = 0;
      for (int j = 0; j <= max_col; j++) sum += dct_mat[fact * j][i] * g[y * nT + j];
      int out = (sum + rnd2) >> post_shift;
      dst[y * stride + i] = (orc_pixel)clip_bd(dst[y * stride + i] + out, bit_depth);
    }
}

/* fallback-dct.cc:260-265 */
static const int8_t dst_mat[4][4] = {{29, 55, 74, 84}, {74, 74, 0, -74}, {84, -29, -74, 55}, {55, -84, 74, -29}};

void orc_dst4_add(orc_pixel* dst, ptrdiff_t stride, const int16_t* coeffs, int bit_depth)
{
  /* fallback-dct.cc:269-407: as the DCT but the row pass IS clipped to int16 before the add (:318) */
  const int post_shift = 20 - bit_depth;
  const int rnd2 = 1 << (post_shift - 1);
  int16_t g[4][4];
  for (int c = 0; c < 4; c++)
    for (int i = 0; i < 4; i++) {
      int sum = 0;
      for (int j = 0; j < 4; j++) sum += dst_mat[j][i] * coeffs[c + j * 4];
      g[i][c] = (int16_t)clip3(-32768, 32767, (sum + 64) >> 7);
    }
  for (int y = 0; y < 4; y++)
    for (int i = 0; i < 4; i++) {
      int sum = 0;
      for (int j = 0; j < 4; j++) sum += dst_mat[j][i] * g[y][j];
      int out = clip3(-32768, 32767, (sum + rnd2) >> post_shift);
      dst[y * stride + i] = (orc_pixel)clip_bd(dst[y * stride + i] + out, bit_depth);
    }
}

static void add_residual(orc_pixel* dst, ptrdiff_t stride, const int32_t* r, int nT, int bd)
{
  /* fallback-dct.h:65-73 */
  for (int y = 0; y < nT; y++)
    for (int x = 0; x < nT; x++) dst[y * stride + x] = (orc_pixel)clip_bd(dst[y * stride + x] + r[y * nT + x], bd);
}

void orc_tskip_add(orc_pixel* dst, ptrdiff_t stride, int nT, const int16_t* coeffs, int bit_depth, int rdpcm)
{
  /* transform.cc:548-596: bdShift = 20-bitDepth, tsShift = 5+log2(nT);
   * fallback-dct.cc:81-91 (plain), :187-214 (rdpcm running sums) */
  const int bd_shift = 20 - bit_depth, ts_shift = 5 + ilog2(nT), rnd = 1 << (bd_shift - 1);
  int32_t r[32 * 32];
  for (int y = 0; y < nT; y++)
    for (int x = 0; x < nT; x++) {
      int32_t c = (int32_t)((uint32_t)(int32_t)coeffs[x + y * nT] << ts_shift);
      r[x + y * nT] = (c + rnd) >> bd_shift;
    }
  if (rdpcm == 1) {
    for (int y = 0; y < nT; y++) for (int x = 1; x < nT; x++) r[x + y * nT] += r[x - 1 + y * nT];
  } else if (rdpcm == 2) {
    for (int x = 0; x < nT; x++) for (int y = 1; y < nT; y++) r[x + y * nT] += r[x + (y - 1) * nT];
  }
  add_residual(dst, stride, r, nT, bit_depth);
}

void orc_bypass_add(orc_pixel* dst, ptrdiff_t stride, int nT, const int16_t* coeffs, int bit_depth, int rdpcm)
{
  /* transform.cc:408-448, fallback-dct.cc:161-225 */
  int32_t r[32 * 32];
  for (int i = 0; i < nT * nT; i++) r[i] = coeffs[i];
  if (rdpcm == 1) {
    for (int y = 0; y < nT; y++) for (int x = 1; x < nT; x++) r[x + y * nT] += r[x - 1 + y * nT];
  } else if (rdpcm == 2) {
    for (int x = 0; x < nT; x++) for (int y = 1; y < nT; y++) r[x + y * nT] += r[x + (y - 1) * nT];
  }
  add_residual(dst, stride, r, nT, bit_depth);
}

/* ------------------------------------------------------------------------------------------
 * Motion compensation
 * ---------------------------------------------------------------------------------------- */

/* fallback-motion.cc:531-555: luma taps at integer offsets -3..+4 for quarter phases 1..3 */
static const int8_t qpel_taps[4][8] = {
    {0, 0, 0, 64, 0, 0, 0, 0}, {-1, 4, -10, 58, 17, -5, 1, 0}, {-1, 4, -11, 40, 40, -11, 4, -1}, {0, 1, -5, 17, 58, -10, 4, -1}};
/* fallback-motion.cc:357-364: chroma taps at offsets -1..+2 for eighth phases 1..7 */
static const int8_t epel_taps[8][4] = {{0, 64, 0, 0},   {-2, 58, 10, -2}, {-4, 54, 16, -2}, {-6, 46, 28, -4},
                                       {-4, 36, 36, -4}, {-4, 28, 46, -6}, {-2, 16, 54, -4}, {-2, 10, 58, -2}};

static void mc_generic(int16_t* out, int out_stride, const orc_pixel* ref, ptrdiff_t ref_stride, int pw, int ph,
                       int x_int, int y_int, int x_frac, int y_frac, int w, int h, int bit_depth,
                       const int8_t* taps_h, const int8_t* taps_v, int ntaps, int before)
{
  /* motion.cc:66,90,134-159 / :193-260: integer position + coordinate clamping (no padded surface);
   * fallback-motion.cc:492-636 / :305-415: H pass >> (bd-8) into int16, V pass >> 6 (>> (bd-8) when
   * no H filter ran), results stored as int16 with C++ truncation (SURVEY App. A.1). */
  const int shift1 = bit_depth - 8;
  const int shift3 = MAXI(2, 14 - bit_depth);
  if (x_frac == 0 && y_frac == 0) {
    for (int y = 0; y < h; y++)
      for (int x = 0; x < w; x++) {
        int xa = clip3(0, pw - 1, x + x_int), ya = clip3(0, ph - 1, y + y_int);
        out[y * out_stride + x] = (int16_t)(ref[xa + ya * ref_stride] << shift3);
      }
    return;
  }
  const int after = ntaps - 1 - before;
  int16_t tmp[(64 + 7) * 64];
  /* The H pass works on one source row gathered with the clamped coordinates (same samples as clamping per tap,
   * motion.cc:147-153; a straight copy when the window lies inside the picture), which keeps the tap loops free of
   * address arithmetic. Rows the V pass does not need are skipped (the reference filters them too: no effect). */
  const int y_lo = y_frac ? -before : 0, y_hi = y_frac ? h + after : h;
  const int x_lo = x_frac ? -before : 0, x_n = w + (x_frac ? ntaps - 1 : 0);
  const int inside = (x_int + x_lo >= 0) && (x_int + x_lo + x_n <= pw);
  for (int y = y_lo; y < y_hi; y++) {
    const orc_pixel* rowp = ref + (ptrdiff_t)clip3(0, ph - 1, y + y_int) * ref_stride;
    orc_pixel line[64 + 8];
    const orc_pixel* r;
    if (inside) {
      r = rowp + x_int + x_lo;
    } else {
      for (int x = 0; x < x_n; x++) line[x] = rowp[clip3(0, pw - 1, x_int + x_lo + x)];
      r = line;
    }
    int16_t* t = tmp + (y + before) * w;
    if (x_frac == 0) {
      for (int x = 0; x < w; x++) t[x] = (int16_t)r[x];
    } else if (ntaps == 8) {
      for (int x = 0; x < w; x++) {
        int sum = taps_h[0] * r[x] + taps_h[1] * r[x + 1] + taps_h[2] * r[x + 2] + taps_h[3] * r[x + 3] + taps_h[4] * r[x + 4] +
                  taps_h[5] * r[x + 5] + taps_h[6] * r[x + 6] + taps_h[7] * r[x + 7];
        t[x] = (int16_t)(sum >> shift1);
      }
    } else {
      for (int x = 0; x < w; x++) {
        int sum = taps_h[0] * r[x] + taps_h[1] * r[x + 1] + taps_h[2] * r[x + 2] + taps_h[3] * r[x + 3];
        t[x] = (int16_t)(sum >> shift1);
      }
    }
  }
  const int vshift = (x_frac == 0) ? shift1 : 6;
  for (int y = 0; y < h; y++) {
    int16_t* o = out + (ptrdiff_t)y * out_stride;
    if (y_frac == 0) {
      for (int x = 0; x < w; x++) o[x] = tmp[(y + before) * w + x];
    } else {
      const int16_t* t = tmp + y * w;
      for (int x = 0; x < w; x++) {
        int sum = 0;
        for (int k = 0; k < ntaps; k++) sum += taps_v[k] * t[k * w + x];
        o[x] = (int16_t)(sum >> vshift);
      }
    }
  }
}

void orc_mc_luma(int16_t* out, int out_stride, const orc_pixel* ref, ptrdiff_t ref_stride, int pic_w, int pic_h,
                 int xP, int yP, int mvx, int mvy, int w, int h, int bit_depth)
{
  /* motion.cc:54-60 */
  int xf = mvx & 3, yf = mvy & 3;
  mc_generic(out, out_stride, ref, ref_stride, pic_w, pic_h, xP + (mvx >> 2), yP + (mvy >> 2), xf, yf, w, h, bit_depth,
             qpel_taps[xf], qpel_taps[yf], 8, 3);
}

void orc_mc_chroma(int16_t* out, int out_stride, const orc_pixel* ref, ptrdiff_t ref_stride, int pic_w, int pic_h,
                   int sub_w, int sub_h, int xP, int yP, int mvx, int mvy, int wC, int hC, int bit_depth)
{
  /* motion.cc:193-206: chroma picture size by integer division, mv scaled to eighth-sample units */
  int wc = pic_w / sub_w, hc = pic_h / sub_h;
  mvx *= 2 / sub_w;
  mvy *= 2 / sub_h;
  int xf = mvx & 7, yf = mvy & 7;
  mc_generic(out, out_stride, ref, ref_stride, wc, hc, xP / sub_w + (mvx >> 3), yP / sub_h + (mvy >> 3), xf, yf, wC, hC,
             bit_depth, epel_taps[xf], epel_taps[yf], 4, 1);
}

void orc_put_unweighted(orc_pixel* dst, ptrdiff_t stride, const int16_t* src, int ss, int w, int h, int bd)
{
  /* fallback-motion.cc:33-52,164-186 */
  int shift1 = MAXI(2, 14 - bd), off = 1 << (shift1 - 1);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) dst[y * stride + x] = (orc_pixel)clip_bd((src[y * ss + x] + off) >> shift1, bd);
}

void orc_put_avg(orc_pixel* dst, ptrdiff_t stride, const int16_t* s1, const int16_t* s2, int ss, int w, int h, int bd)
{
  /* fallback-motion.cc:97-158,232-256 */
  int shift2 = MAXI(3, 15 - bd), off = 1 << (shift2 - 1);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++)
      dst[y * stride + x] = (orc_pixel)clip_bd((s1[y * ss + x] + s2[y * ss + x] + off) >> shift2, bd);
}

void orc_put_weighted(orc_pixel* dst, ptrdiff_t stride, const int16_t* src, int ss, int w, int h, int wt, int o,
                      int log2wd, int bd)
{
  /* fallback-motion.cc:55-73,190-208: offset added AFTER the shift */
  int rnd = 1 << (log2wd - 1);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) dst[y * stride + x] = (orc_pixel)clip_bd(((src[y * ss + x] * wt + rnd) >> log2wd) + o, bd);
}

void orc_put_weighted_bi(orc_pixel* dst, ptrdiff_t stride, const int16_t* s1, const int16_t* s2, int ss, int w, int h,
                         int w1, int o1, int w2, int o2, int log2wd, int bd)
{
  /* fallback-motion.cc:75-94,210-229 */
  int rnd = (int)((unsigned)(o1 + o2 + 1) << log2wd);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++)
      dst[y * stride + x] = (orc_pixel)clip_bd((s1[y * ss + x] * w1 + s2[y * ss + x] * w2 + rnd) >> (log2wd + 1), bd);
}

/* ------------------------------------------------------------------------------------------
 * Intra prediction
 * ---------------------------------------------------------------------------------------- */

void orc_intra_border(orc_pixel* border, const orc_pixel* plane, ptrdiff_t stride, int xB, int yB, int nT,
                      uint64_t avail, int bit_depth)
{
  /* intrapred.h:529-633 with the metadata tests replaced by the precomputed mask, then the
   * substitution process :637-674 (scan from border[-2nT] upwards, then along the top). */
  uint8_t av_mem[4 * 32 + 1];
  uint8_t* av = av_mem + 2 * nT;
  memset(av_mem, 0, sizeof(av_mem));
  int n_avail = 0;
  for (int k = 0; k < nT / 2; k++)
    if (avail & (1ull << k))
      for (int i = 0; i < 4; i++) {
        int r = 4 * k + i;
        border[-r - 1] = plane[(xB - 1) + (yB + r) * stride];
        av[-r - 1] = 1;
        n_avail++;
      }
  if (avail & (1ull << B200_AVAIL_CORNER_BIT)) {
    border[0] = plane[(xB - 1) + (yB - 1) * stride];
    av[0] = 1;
    n_avail++;
  }
  for (int k = 0; k < nT / 2; k++)
    if (avail & (1ull << (B200_AVAIL_TOP_BIT0 + k)))
      for (int i = 0; i < 4; i++) {
        int c = 4 * k + i;
        border[c + 1] = plane[(xB + c) + (yB - 1) * stride];
        av[c + 1] = 1;
        n_avail++;
      }
  if (n_avail == 4 * nT + 1) return;
  if (n_avail == 0) {
    for (int i = -2 * nT; i <= 2 * nT; i++) border[i] = (orc_pixel)(1 << (bit_depth - 1));
    return;
  }
  if (!av[-2 * nT]) {
    /* firstValue = first available sample in scan order (intrapred.h:572,596,622) */
    int i = -2 * nT;
    while (!av[i]) i++;
    border[-2 * nT] = border[i];
  }
  for (int i = -2 * nT + 1; i <= 2 * nT; i++)
    if (!av[i]) border[i] = border[i - 1];
}

void orc_intra_filter(orc_pixel* p, int nT, int cIdx, int mode, int strong, int bit_depth_luma)
{
  /* intrapred.h:185-258 */
  int filter;
  if (mode == 1 || nT == 4) {
    filter = 0;
  } else {
    int d = MINI(iabs(mode - 26), iabs(mode - 10));
    filter = (nT == 8) ? (d > 7) : (nT == 16) ? (d > 1) : (nT == 32) ? (d > 0) : 0;
  }
  if (!filter) return;
  orc_pixel f_mem[4 * 32 + 1];
  orc_pixel* f = f_mem + 2 * nT;
  int bi = strong && cIdx == 0 && nT == 32 && iabs(p[0] + p[64] - 2 * p[32]) < (1 << (bit_depth_luma - 5)) &&
           iabs(p[0] + p[-64] - 2 * p[-32]) < (1 << (bit_depth_luma - 5));
  f[-2 * nT] = p[-2 * nT];
  f[2 * nT] = p[2 * nT];
  if (bi) {
    f[0] = p[0];
    for (int i = 1; i <= 63; i++) {
      f[-i] = (orc_pixel)(p[0] + ((i * (p[-64] - p[0]) + 32) >> 6));
      f[i] = (orc_pixel)(p[0] + ((i * (p[64] - p[0]) + 32) >> 6));
    }
  } else {
    for (int i = -(2 * nT - 1); i <= 2 * nT - 1; i++) f[i] = (orc_pixel)((p[i + 1] + 2 * p[i] + p[i - 1] + 2) >> 2);
  }
  memcpy(p - 2 * nT, f - 2 * nT, (4 * nT + 1) * sizeof(orc_pixel));
}

/* intrapred.cc:268-274 */
static const int8_t intra_angle[35] = {0,   0,   32,  26,  21,  17, 13, 9,  5,  2,  0,  -2, -5, -9, -13, -17, -21, -26,
                                       -32, -26, -21, -17, -13, -9, -5, -2, 0,  2,  5,  9,  13, 17, 21,  26,  32};
static const int16_t inv_angle[15] = {-4096, -1638, -910, -630, -482, -390, -315, -256, -315, -390, -482, -630, -910, -1638, -4096};

void orc_intra_pred(orc_pixel* dst, ptrdiff_t stride, int nT, int cIdx, int mode, const orc_pixel* border, int bit_depth,
                    int disable_boundary_filter)
{
  const int log2 = ilog2(nT);
  if (mode == 0) { /* planar, intrapred.h:261-285 */
    for (int y = 0; y < nT; y++)
      for (int x = 0; x < nT; x++)
        dst[x + y * stride] = (orc_pixel)(((nT - 1 - x) * border[-1 - y] + (x + 1) * border[1 + nT] + (nT - 1 - y) * border[1 + x] +
                                           (y + 1) * border[-1 - nT] + nT) >> (log2 + 1));
    return;
  }
  if (mode == 1) { /* DC, intrapred.h:288-322 */
    int dc = nT;
    for (int i = 0; i < nT; i++) dc += border[i + 1] + border[-i - 1];
    dc >>= log2 + 1;
    for (int y = 0; y < nT; y++)
      for (int x = 0; x < nT; x++) dst[x + y * stride] = (orc_pixel)dc;
    if (cIdx == 0 && nT < 32) {
      dst[0] = (orc_pixel)((border[-1] + 2 * dc + border[1] + 2) >> 2);
      for (int x = 1; x < nT; x++) dst[x] = (orc_pixel)((border[x + 1] + 3 * dc + 2) >> 2);
      for (int y = 1; y < nT; y++) dst[y * stride] = (orc_pixel)((border[-y - 1] + 3 * dc + 2) >> 2);
    }
    return;
  }
  /* angular, intrapred.h:330-433.  For modes < 18 the roles of x/y and of the top/left border swap. */
  orc_pixel ref_mem[4 * 32 + 1];
  orc_pixel* ref = ref_mem + 2 * 32;
  const int angle = intra_angle[mode];
  const int vert = mode >= 18;
  const int sgn = vert ? 1 : -1; /* ref[x] = border[sgn*x] */
  for (int x = 0; x <= nT; x++) ref[x] = border[sgn * x];
  if (angle < 0) {
    int inv = inv_angle[mode - 11];
    int last = (nT * angle) >> 5;
    if (last < -1)
      for (int x = last; x <= -1; x++) ref[x] = border[-sgn * ((x * inv + 128) >> 8)];
  } else {
    for (int x = nT + 1; x <= 2 * nT; x++) ref[x] = border[sgn * x];
  }
  for (int y = 0; y < nT; y++)
    for (int x = 0; x < nT; x++) {
      int a = vert ? y : x, b = vert ? x : y; /* a: distance from the reference row, b: along it */
      int idx = ((a + 1) * angle) >> 5, fact = ((a + 1) * angle) & 31;
      int v = fact ? ((32 - fact) * ref[b + idx + 1] + fact * ref[b + idx + 2] + 16) >> 5 : ref[b + idx + 1];
      dst[x + y * stride] = (orc_pixel)v;
    }
  if (cIdx == 0 && nT < 32 && !disable_boundary_filter) {
    if (mode == 26)
      for (int y = 0; y < nT; y++) dst[y * stride] = (orc_pixel)clip_bd(border[1] + ((border[-1 - y] - border[0]) >> 1), bit_depth);
    if (mode == 10)
      for (int x = 0; x < nT; x++) dst[x] = (orc_pixel)clip_bd(border[-1] + ((border[1 + x] - border[0]) >> 1), bit_depth);
  }
}

/* ------------------------------------------------------------------------------------------
 * Deblocking
 * ---------------------------------------------------------------------------------------- */

void orc_deblock_luma_seg(orc_pixel* ptr, ptrdiff_t stride, int vertical, int dE, int dEp, int dEq, int tc, int filterP,
                          int filterQ, int bd)
{
  /* fallback-deblk.h:32-98.  a = step across the edge, b = step along it. */
  ptrdiff_t a = vertical ? 1 : stride, b = vertical ? stride : 1;
  for (int k = 0; k < 4; k++) {
    orc_pixel* q = ptr + k * b;
    int p0 = q[-a], p1 = q[-2 * a], p2 = q[-3 * a], p3 = q[-4 * a];
    int q0 = q[0], q1 = q[a], q2 = q[2 * a], q3 = q[3 * a];
    if (dE == 2) {
      if (filterP) {
        q[-a] = (orc_pixel)clip3(p0 - 2 * tc, p0 + 2 * tc, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
        q[-2 * a] = (orc_pixel)clip3(p1 - 2 * tc, p1 + 2 * tc, (p2 + p1 + p0 + q0 + 2) >> 2);
        q[-3 * a] = (orc_pixel)clip3(p2 - 2 * tc, p2 + 2 * tc, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
      }
      if (filterQ) {
        q[0] = (orc_pixel)clip3(q0 - 2 * tc, q0 + 2 * tc, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
        q[a] = (orc_pixel)clip3(q1 - 2 * tc, q1 + 2 * tc, (p0 + q0 + q1 + q2 + 2) >> 2);
        q[2 * a] = (orc_pixel)clip3(q2 - 2 * tc, q2 + 2 * tc, (p0 + q0 + q1 + 3 * q2 + 2 * q3 + 4) >> 3);
      }
    } else {
      int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
      if (iabs(delta) < tc * 10) {
        delta = clip3(-tc, tc, delta);
        if (filterP) q[-a] = (orc_pixel)clip_bd(p0 + delta, bd);
        if (filterQ) q[0] = (orc_pixel)clip_bd(q0 - delta, bd);
        if (dEp == 1 && filterP) {
          int dp = clip3(-(tc >> 1), tc >> 1, (((p2 + p0 + 1) >> 1) - p1 + delta) >> 1);
          q[-2 * a] = (orc_pixel)clip_bd(p1 + dp, bd);
        }
        if (dEq == 1 && filterQ) {
          int dq = clip3(-(tc >> 1), tc >> 1, (((q2 + q0 + 1) >> 1) - q1 - delta) >> 1);
          q[a] = (orc_pixel)clip_bd(q1 + dq, bd);
        }
      }
    }
  }
}

void orc_deblock_chroma_seg(orc_pixel* ptr, ptrdiff_t stride, int vertical, int tc, int filterP, int filterQ, int bd)
{
  /* fallback-deblk.h:102-124 */
  ptrdiff_t a = vertical ? 1 : stride, b = vertical ? stride : 1;
  for (int k = 0; k < 4; k++) {
    orc_pixel* q = ptr + k * b;
    int p0 = q[-a], p1 = q[-2 * a], q0 = q[0], q1 = q[a];
    int delta = clip3(-tc, tc, ((((q0 - p0) * 4) + p1 - q1 + 4) >> 3));
    if (filterP) q[-a] = (orc_pixel)clip_bd(p0 + delta, bd);
    if (filterQ) q[0] = (orc_pixel)clip_bd(q0 - delta, bd);
  }
}

/* deblock.cc:397-407 */
static const uint8_t tab_beta[52] = {0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  6,  7,
                                     8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 22, 24, 26, 28, 30, 32,
                                     34, 36, 38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64};
static const uint8_t tab_tc[54] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,  0,  0,  1,  1,  1,  1,  1,  1,  1,  1,  1,
                                   2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8,  9,  10, 11, 13, 14, 16, 18, 20, 22, 24};
/* transform.cc:27 + transform.h:29-34 */
static int table8_22(int qPi)
{
  static const int t[13] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37};
  if (qPi < 30) return qPi;
  if (qPi >= 43) return qPi - 6;
  return t[qPi - 30];
}

typedef struct pic_geom {
  int w, h, w4, h4, w8, h8, log2ctb, wctb, hctb, sub_w, sub_h;
} pic_geom;

static pic_geom geom_of(const b200_pic_params* p)
{
  pic_geom g;
  g.w = p->width;
  g.h = p->height;
  g.w4 = (g.w + 3) / 4;
  g.h4 = (g.h + 3) / 4;
  g.w8 = (g.w + 7) / 8;
  g.h8 = (g.h + 7) / 8;
  g.log2ctb = p->log2_ctb_size;
  g.wctb = (g.w + (1 << g.log2ctb) - 1) >> g.log2ctb;
  g.hctb = (g.h + (1 << g.log2ctb) - 1) >> g.log2ctb;
  g.sub_w = (p->chroma_format_idc == 1 || p->chroma_format_idc == 2) ? 2 : 1;
  g.sub_h = (p->chroma_format_idc == 1) ? 2 : 1;
  return g;
}

static inline int qpy_at(const b200_picture* pic, const pic_geom* g, int x, int y) { return pic->qp_map[(x >> 3) + (y >> 3) * g->w8]; }
static inline int nofilt_at(const b200_picture* pic, const pic_geom* g, int x, int y) { return pic->nofilt_map[(x >> 3) + (y >> 3) * g->w8] & 1; }
static inline const b200_slice_info* slice_at(const b200_picture* pic, const pic_geom* g, int x, int y)
{
  return &pic->slices[pic->ctbs[(x >> g->log2ctb) + (y >> g->log2ctb) * g->wctb].slice_idx];
}

void orc_deblock_picture(orc_surface* s, const b200_picture* pic, int vertical)
{
  const pic_geom g = geom_of(&pic->params);
  /* luma: deblock.cc:412-605 — every 4-line segment on the 8x8 grid */
  const int x_inc = vertical ? 2 : 1, y_inc = vertical ? 1 : 2;
  const int bd_y = pic->params.bit_depth_luma, bd_c = pic->params.bit_depth_chroma;
  for (int y = 0; y < g.h4; y += y_inc)
    for (int x = 0; x < g.w4; x += x_inc) {
      int xd = x << 2, yd = y << 2;
      int b = pic->bs_map[x + y * g.w4];
      int bS = vertical ? B200_BS_V(b) : B200_BS_H(b);
      if (bS == 0) continue;
      orc_pixel* ptr = s->plane[0] + xd + yd * s->stride[0];
      ptrdiff_t a = vertical ? 1 : s->stride[0], bb = vertical ? s->stride[0] : 1;
      int qp_q = qpy_at(pic, &g, xd, yd);
      int qp_p = vertical ? qpy_at(pic, &g, xd - 1, yd) : qpy_at(pic, &g, xd, yd - 1);
      int qpl = (qp_q + qp_p + 1) >> 1;
      const b200_slice_info* sl = slice_at(pic, &g, xd, yd); /* slice of the Q sample, deblock.cc:521-523 */
      int beta = tab_beta[clip3(0, 51, qpl + sl->beta_offset)] * (1 << (bd_y - 8));
      int tc = tab_tc[clip3(0, 53, qpl + 2 * (bS - 1) + sl->tc_offset)] * (1 << (bd_y - 8));
#define P(k, i) ((int)ptr[(k)*bb - ((i) + 1) * a])
#define Q(k, i) ((int)ptr[(k)*bb + (i)*a])
      int dp0 = iabs(P(0, 2) - 2 * P(0, 1) + P(0, 0)), dp3 = iabs(P(3, 2) - 2 * P(3, 1) + P(3, 0));
      int dq0 = iabs(Q(0, 2) - 2 * Q(0, 1) + Q(0, 0)), dq3 = iabs(Q(3, 2) - 2 * Q(3, 1) + Q(3, 0));
      int dpq0 = dp0 + dq0, dpq3 = dp3 + dq3, dp = dp0 + dp3, dq = dq0 + dq3, d = dpq0 + dpq3;
      int dE = 0, dEp = 0, dEq = 0;
      if (d < beta) {
        int s0 = 2 * dpq0 < (beta >> 2) && iabs(P(0, 3) - P(0, 0)) + iabs(Q(0, 0) - Q(0, 3)) < (beta >> 3) &&
                 iabs(P(0, 0) - Q(0, 0)) < ((5 * tc + 1) >> 1);
        int s3 = 2 * dpq3 < (beta >> 2) && iabs(P(3, 3) - P(3, 0)) + iabs(Q(3, 0) - Q(3, 3)) < (beta >> 3) &&
                 iabs(P(3, 0) - Q(3, 0)) < ((5 * tc + 1) >> 1);
        dE = (s0 && s3) ? 2 : 1;
        if (dp < ((beta + (beta >> 1)) >> 3)) dEp = 1;
        if (dq < ((beta + (beta >> 1)) >> 3)) dEq = 1;
      }
#undef P
#undef Q
      if (dE) {
        int fP = !(vertical ? nofilt_at(pic, &g, xd - 1, yd) : nofilt_at(pic, &g, xd, yd - 1));
        int fQ = !nofilt_at(pic, &g, xd, yd);
        orc_deblock_luma_seg(ptr, s->stride[0], vertical, dE, dEp, dEq, tc, fP, fQ, bd_y);
      }
    }
  if (pic->params.chroma_format_idc == 0) return;
  /* chroma: deblock.cc:635-761 — only bS==2, on the chroma 8x8 grid */
  const int cx_inc = x_inc * g.sub_w, cy_inc = y_inc * g.sub_h;
  for (int y = 0; y < g.h4; y += cy_inc)
    for (int x = 0; x < g.w4; x += cx_inc) {
      int xd = x << (3 - g.sub_w), yd = y << (3 - g.sub_h); /* chroma sample position */
      int xl = xd * g.sub_w, yl = yd * g.sub_h;             /* luma position */
      int b = pic->bs_map[(xl >> 2) + (yl >> 2) * g.w4];
      int bS = vertical ? B200_BS_V(b) : B200_BS_H(b);
      if (bS < 2) continue;
      for (int c = 1; c <= 2; c++) {
        int off = (c == 1) ? pic->params.pps_cb_qp_offset : pic->params.pps_cr_qp_offset;
        int qp_q = qpy_at(pic, &g, xl, yl);
        int qp_p = vertical ? qpy_at(pic, &g, xl - 1, yl) : qpy_at(pic, &g, xl, yl - 1);
        int qpi = ((qp_q + qp_p + 1) >> 1) + off;
        int qpc = (pic->params.chroma_format_idc == 1) ? table8_22(qpi) : MINI(qpi, 51);
        const b200_slice_info* sl = slice_at(pic, &g, xl, yl);
        int tc = tab_tc[clip3(0, 53, qpc + 2 * (bS - 1) + sl->tc_offset)] * (1 << (bd_c - 8));
        int fP = !(vertical ? nofilt_at(pic, &g, xl - 1, yl) : nofilt_at(pic, &g, xl, yl - 1));
        int fQ = !nofilt_at(pic, &g, xl, yl);
        orc_deblock_chroma_seg(s->plane[c] + xd + yd * s->stride[c], s->stride[c], vertical, tc, fP, fQ, bd_c);
      }
    }
}

/* ------------------------------------------------------------------------------------------
 * SAO
 * ---------------------------------------------------------------------------------------- */

static void sao_ctb(const orc_surface* in, orc_surface* out, const b200_picture* pic, const pic_geom* g, int xCtb, int yCtb, int cIdx)
{
  /* sao.cc:28-263 */
  const b200_ctb_info* ci = &pic->ctbs[xCtb + yCtb * g->wctb];
  int type = (ci->sao_type >> (2 * cIdx)) & 3;
  if (type == 0) return;
  const int bd = cIdx ? pic->params.bit_depth_chroma : pic->params.bit_depth_luma;
  const int maxv = (1 << bd) - 1;
  const int sw = cIdx ? g->sub_w : 1, sh = cIdx ? g->sub_h : 1;
  const int shw = sw - 1, shh = sh - 1; /* chroma shifts */
  const int nSW = (1 << g->log2ctb) / sw, nSH = (1 << g->log2ctb) / sh;
  const int xC = xCtb * nSW, yC = yCtb * nSH;
  const int width = cIdx ? in->cw : in->width, height = cIdx ? in->ch : in->height;
  const int ctbW = (xC + nSW > width) ? width - xC : nSW, ctbH = (yC + nSH > height) ? height - yC : nSH;
  const ptrdiff_t is = in->stride[cIdx], os = out->stride[cIdx];
  const orc_pixel* ip = in->plane[cIdx];
  orc_pixel* op = out->plane[cIdx];
  /* sao.cc:49: get_SliceHeader(xC,yC) is evaluated with COMPONENT coordinates (a reference quirk
   * that matters for chroma in multi-slice pictures); restated literally. */
  const int ctb_slice_addr = (int)slice_at(pic, g, MINI(xC, g->w - 1), MINI(yC, g->h - 1))->slice_addr_rs;
  if (type == 2) {
    static const int8_t hpos[4][2] = {{-1, 1}, {0, 0}, {-1, 1}, {1, -1}};
    static const int8_t vpos[4][2] = {{0, 0}, {-1, 1}, {-1, 1}, {-1, 1}};
    int cls = (ci->sao_eo_class >> (2 * cIdx)) & 3;
    int offs[5] = {ci->sao_offset[cIdx][0], ci->sao_offset[cIdx][1], 0, ci->sao_offset[cIdx][2], ci->sao_offset[cIdx][3]};
    for (int j = 0; j < ctbH; j++)
      for (int i = 0; i < ctbW; i++) {
        int xl = (xC + i) << shw, yl = (yC + j) << shh;
        if (nofilt_at(pic, g, xl, yl)) continue;
        int edge = -1;
        if (i == 0 || j == 0 || i == ctbW - 1 || j == ctbH - 1)
          for (int k = 0; k < 2; k++) {
            int xS = xC + i + hpos[cls][k], yS = yC + j + vpos[cls][k];
            if (xS < 0 || yS < 0 || xS >= width || yS >= height) { edge = 0; break; }
            const b200_slice_info* sn = slice_at(pic, g, xS << shw, yS << shh);
            const b200_slice_info* sc = slice_at(pic, g, xl, yl);
            if ((int)sn->slice_addr_rs < ctb_slice_addr && !(sc->flags & B200_SLICE_LF_ACROSS_SLICES)) { edge = 0; break; }
            if ((int)sn->slice_addr_rs > ctb_slice_addr && !(sn->flags & B200_SLICE_LF_ACROSS_SLICES)) { edge = 0; break; }
            if (!(pic->params.flags & B200_PIC_LF_ACROSS_TILES)) {
              int tn = pic->ctbs[((xS << shw) >> g->log2ctb) + ((yS << shh) >> g->log2ctb) * g->wctb].tile_id;
              if (tn != ci->tile_id) { edge = 0; break; }
            }
          }
        if (edge != 0) {
          int c = ip[xC + i + (yC + j) * is];
          int a = ip[xC + i + hpos[cls][0] + (yC + j + vpos[cls][0]) * is];
          int b = ip[xC + i + hpos[cls][1] + (yC + j + vpos[cls][1]) * is];
          int e = ((c > a) - (c < a)) + ((c > b) - (c < b));
          op[xC + i + (yC + j) * os] = (orc_pixel)clip3(0, maxv, c + offs[e + 2]);
        }
      }
  } else {
    int band_shift = bd - 5;
    int table[32];
    memset(table, 0, sizeof(table));
    for (int k = 0; k < 4; k++) table[(k + ci->sao_band_pos[cIdx]) & 31] = k + 1;
    for (int j = 0; j < ctbH; j++)
      for (int i = 0; i < ctbW; i++) {
        if (nofilt_at(pic, g, (xC + i) << shw, (yC + j) << shh)) continue;
        int c = ip[xC + i + (yC + j) * is];
        int idx = table[clip3(0, maxv, c) >> band_shift];
        if (idx > 0) op[xC + i + (yC + j) * os] = (orc_pixel)clip3(0, maxv, c + ci->sao_offset[cIdx][idx - 1]);
      }
  }
}

void orc_sao_picture(const orc_surface* in, orc_surface* out, const b200_picture* pic)
{
  /* sao.cc:327-382: out starts as a copy of the deblocked picture; every CTB reads only `in`. */
  const pic_geom g = geom_of(&pic->params);
  int nc = pic->params.chroma_format_idc ? 3 : 1;
  for (int c = 0; c < nc; c++)
    for (int yCtb = 0; yCtb < g.hctb; yCtb++)
      for (int xCtb = 0; xCtb < g.wctb; xCtb++) {
        const b200_slice_info* sl = &pic->slices[pic->ctbs[xCtb + yCtb * g.wctb].slice_idx];
        if (c == 0 && !(sl->flags & B200_SLICE_SAO_LUMA)) continue;
        if (c != 0 && !(sl->flags & B200_SLICE_SAO_CHROMA)) continue;
        sao_ctb(in, out, pic, &g, xCtb, yCtb, c);
      }
}

/* ------------------------------------------------------------------------------------------
 * Picture replay
 * ---------------------------------------------------------------------------------------- */

struct orc_ctx {
  orc_surface slot[B200_MAX_SLOTS];
  orc_surface scratch;
};

static void surf_free(orc_surface* s)
{
  for (int c = 0; c < 3; c++) { free(s->plane[c]); s->plane[c] = NULL; }
}

static int surf_ensure(orc_surface* s, const b200_pic_params* p)
{
  const pic_geom g = geom_of(p);
  int cw = p->chroma_format_idc ? p->width / g.sub_w : 0, ch = p->chroma_format_idc ? p->height / g.sub_h : 0;
  /* any format difference starts a new zero-filled picture, as the reference's image allocation does (ref_replay.cc ensure_slot) */
  if (s->plane[0] && s->width == p->width && s->height == p->height && s->chroma_format_idc == p->chroma_format_idc &&
      s->bd_y == p->bit_depth_luma && s->bd_c == p->bit_depth_chroma)
    return 0;
  surf_free(s);
  s->width = p->width; s->height = p->height; s->cw = cw; s->ch = ch;
  s->chroma_format_idc = p->chroma_format_idc;
  s->bd_y = p->bit_depth_luma; s->bd_c = p->bit_depth_chroma;
  s->stride[0] = p->width; s->stride[1] = s->stride[2] = cw;
  s->plane[0] = (orc_pixel*)calloc((size_t)p->width * p->height, sizeof(orc_pixel)); /* new pictures are zero-filled, image.cc:164 */
  if (!s->plane[0]) return B200_ERR_NOMEM;
  for (int c = 1; c < 3 && cw; c++) {
    s->plane[c] = (orc_pixel*)calloc((size_t)cw * ch, sizeof(orc_pixel));
    if (!s->plane[c]) return B200_ERR_NOMEM;
  }
  return 0;
}

orc_ctx* orc_create(void) { return (orc_ctx*)calloc(1, sizeof(orc_ctx)); }

void orc_destroy(orc_ctx* c)
{
  if (!c) return;
  for (int i = 0; i < B200_MAX_SLOTS; i++) surf_free(&c->slot[i]);
  surf_free(&c->scratch);
  free(c);
}

const orc_surface* orc_slot(orc_ctx* c, int slot) { return (slot >= 0 && slot < B200_MAX_SLOTS && c->slot[slot].plane[0]) ? &c->slot[slot] : NULL; }

int orc_fill_slot(orc_ctx* c, int slot, const b200_pic_params* p, int vy, int vc)
{
  if (slot < 0 || slot >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  orc_surface* s = &c->slot[slot];
  int e = surf_ensure(s, p);
  if (e) return e;
  for (size_t i = 0; i < (size_t)s->width * s->height; i++) s->plane[0][i] = (orc_pixel)vy;
  for (int k = 1; k < 3 && s->cw; k++)
    for (size_t i = 0; i < (size_t)s->cw * s->ch; i++) s->plane[k][i] = (orc_pixel)vc;
  return 0;
}

int orc_upload_slot(orc_ctx* c, int slot, const b200_pic_params* p, const void* const planes[3], const size_t strides[3])
{
  if (slot < 0 || slot >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  orc_surface* s = &c->slot[slot];
  int e = surf_ensure(s, p);
  if (e) return e;
  for (int k = 0; k < 3; k++) {
    int w = k ? s->cw : s->width, h = k ? s->ch : s->height, bd = k ? s->bd_c : s->bd_y;
    if (!w) continue;
    for (int y = 0; y < h; y++) {
      const uint8_t* row = (const uint8_t*)planes[k] + (size_t)y * strides[k];
      for (int x = 0; x < w; x++) s->plane[k][x + y * s->stride[k]] = bd > 8 ? ((const uint16_t*)row)[x] : row[x];
    }
  }
  return 0;
}

int orc_read_slot(orc_ctx* c, int slot, void* const planes[3], const size_t strides[3])
{
  const orc_surface* s = orc_slot(c, slot);
  if (!s) return B200_ERR_INVALID;
  for (int k = 0; k < 3; k++) {
    int w = k ? s->cw : s->width, h = k ? s->ch : s->height, bd = k ? s->bd_c : s->bd_y;
    if (!w || !planes[k]) continue;
    for (int y = 0; y < h; y++) {
      uint8_t* row = (uint8_t*)planes[k] + (size_t)y * strides[k];
      for (int x = 0; x < w; x++) {
        orc_pixel v = s->plane[k][x + y * s->stride[k]];
        if (bd > 8) ((uint16_t*)row)[x] = v; else row[x] = (uint8_t)v;
      }
    }
  }
  return 0;
}

static void inter_pred_pu(orc_ctx* c, orc_surface* cur, const b200_picture* pic, const pic_geom* g, const b200_pu* pu)
{
  /* motion.cc:288-729 */
  static int16_t pred[2][3][64 * 64];
  const int nc = pic->params.chroma_format_idc ? 3 : 1;
  const int wC = pu->w / g->sub_w, hC = pu->h / g->sub_h;
  int use[2] = {pu->flags & B200_PU_PRED_L0 ? 1 : 0, pu->flags & B200_PU_PRED_L1 ? 1 : 0};
  for (int l = 0; l < 2; l++) {
    if (!use[l]) continue;
    const orc_surface* ref = pu->ref_slot[l] >= 0 ? orc_slot(c, pu->ref_slot[l]) : NULL;
    /* motion.cc:385-405: a reference of another size, chroma format or luma / chroma bit depth counts as missing */
    if (ref && (ref->width != pic->params.width || ref->height != pic->params.height || ref->chroma_format_idc != pic->params.chroma_format_idc ||
                ref->bd_y != pic->params.bit_depth_luma || ref->bd_c != pic->params.bit_depth_chroma))
      ref = NULL;
    if (!ref) { /* motion.cc:362-376: mid-grey in 14-bit intermediate precision */
      for (int k = 0; k < nc; k++)
        for (int i = 0; i < 64 * 64; i++) pred[l][k][i] = 1 << 13;
      continue;
    }
    orc_mc_luma(pred[l][0], 64, ref->plane[0], ref->stride[0], g->w, g->h, pu->x, pu->y, pu->mv[l][0], pu->mv[l][1], pu->w, pu->h,
                pic->params.bit_depth_luma);
    for (int k = 1; k < nc; k++)
      orc_mc_chroma(pred[l][k], 64, ref->plane[k], ref->stride[k], g->w, g->h, g->sub_w, g->sub_h, pu->x, pu->y, pu->mv[l][0],
                    pu->mv[l][1], wC, hC, pic->params.bit_depth_chroma);
  }
  const b200_weight_entry* we = (pu->flags & B200_PU_WEIGHTED) ? &pic->weights[pu->wt_idx] : NULL;
  for (int k = 0; k < nc; k++) {
    int w = k ? wC : pu->w, h = k ? hC : pu->h, bd = k ? pic->params.bit_depth_chroma : pic->params.bit_depth_luma;
    int x = k ? pu->x / g->sub_w : pu->x, y = k ? pu->y / g->sub_h : pu->y;
    orc_pixel* dst = cur->plane[k] + x + y * cur->stride[k];
    int log2wd = we ? (k ? we->log2wd_chroma : we->log2wd_luma) : 0;
    if (use[0] && use[1]) {
      if (we) orc_put_weighted_bi(dst, cur->stride[k], pred[0][k], pred[1][k], 64, w, h, we->w[0][k], we->o[0][k], we->w[1][k], we->o[1][k], log2wd, bd);
      else orc_put_avg(dst, cur->stride[k], pred[0][k], pred[1][k], 64, w, h, bd);
    } else if (use[0] || use[1]) {
      int l = use[0] ? 0 : 1;
      if (we) orc_put_weighted(dst, cur->stride[k], pred[l][k], 64, w, h, we->w[l][k], we->o[l][k], log2wd, bd);
      else orc_put_unweighted(dst, cur->stride[k], pred[l][k], 64, w, h, bd);
    }
  }
}

static const uint8_t* scaling_matrix(const b200_picture* pic, const b200_tu* tu)
{
  /* transform.cc:489-510; the factors are valid only under B200_PIC_SCALING_LIST (sps.scaling_list_enable_flag) */
  if (!(tu->flags & B200_TU_SCALING_LIST) || !(pic->params.flags & B200_PIC_SCALING_LIST) || !pic->scaling_factors) return NULL;
  int nT = 1 << tu->log2_size;
  int m = tu->cidx;
  if (nT == 32) m = 0;
  if (tu->flags & B200_TU_INTER_MATRIX) m += (nT < 32) ? 3 : 1;
  const uint8_t* f = pic->scaling_factors;
  switch (nT) {
    case 4: return f + m * 16;
    case 8: return f + 6 * 16 + m * 64;
    case 16: return f + 6 * 16 + 6 * 64 + m * 256;
    default: return f + 6 * 16 + 6 * 64 + 6 * 256 + m * 1024;
  }
}

static void recon_tu(orc_surface* cur, const b200_picture* pic, const b200_tu* tu)
{
  /* slice.cc:3460-3524 decode_TU */
  const int nT = 1 << tu->log2_size, c = tu->cidx;
  const int bd = c ? pic->params.bit_depth_chroma : pic->params.bit_depth_luma;
  orc_pixel* dst = cur->plane[c] + tu->x + (ptrdiff_t)tu->y * cur->stride[c];
  const ptrdiff_t stride = cur->stride[c];
  const b200_coeff* co = pic->coeffs + tu->coeff_off;
  if (tu->flags & B200_TU_PCM) { /* slice.cc:4211-4255 */
    for (int i = 0; i < tu->n_coeff; i++) dst[(co[i].pos % nT) + (co[i].pos / nT) * stride] = (orc_pixel)(uint16_t)co[i].level;
    return;
  }
  if (tu->flags & B200_TU_INTRA) { /* intrapred.cc:277-319 */
    orc_pixel bmem[4 * 32 + 1];
    orc_pixel* border = bmem + 2 * nT;
    orc_intra_border(border, cur->plane[c], stride, tu->x, tu->y, nT, tu->avail, bd);
    if (!(pic->params.flags & B200_PIC_INTRA_SMOOTHING_OFF) && (c == 0 || pic->params.chroma_format_idc == 3))
      orc_intra_filter(border, nT, c, tu->intra_mode, (pic->params.flags & B200_PIC_STRONG_INTRA_SMOOTHING) != 0, pic->params.bit_depth_luma);
    orc_intra_pred(dst, stride, nT, c, tu->intra_mode, border, bd, (tu->flags & B200_TU_NO_BOUNDARY_FILTER) != 0);
  }
  if (!(tu->flags & B200_TU_CBF)) return;
  /* transform.cc:361-642 scale_coefficients_internal */
  int16_t buf[32 * 32];
  memset(buf, 0, sizeof(int16_t) * nT * nT);
  const int rdpcm = (tu->flags & B200_TU_RDPCM_H) ? 1 : (tu->flags & B200_TU_RDPCM_V) ? 2 : 0;
  if (tu->flags & B200_TU_BYPASS) {
    for (int i = 0; i < tu->n_coeff; i++) buf[co[i].pos] = co[i].level;
  } else {
    int16_t lv[32 * 32];
    uint16_t ps[32 * 32];
    for (int i = 0; i < tu->n_coeff; i++) { lv[i] = co[i].level; ps[i] = co[i].pos; }
    orc_dequant(buf, lv, ps, tu->n_coeff, tu->qp, bd, tu->log2_size, scaling_matrix(pic, tu));
  }
  if ((tu->flags & B200_TU_ROTATE) && (tu->flags & (B200_TU_BYPASS | B200_TU_TSKIP))) { /* fallback-dct.cc:250-256 */
    for (int i = 0; i < nT * nT / 2; i++) { int16_t t = buf[i]; buf[i] = buf[nT * nT - 1 - i]; buf[nT * nT - 1 - i] = t; }
  }
  if (tu->flags & B200_TU_BYPASS) orc_bypass_add(dst, stride, nT, buf, bd, rdpcm);
  else if (tu->flags & B200_TU_TSKIP) orc_tskip_add(dst, stride, nT, buf, bd, rdpcm);
  else if (tu->flags & B200_TU_DST) orc_dst4_add(dst, stride, buf, bd);
  else orc_idct_add(dst, stride, nT, buf, bd);
}

int orc_reconstruct(orc_ctx* c, const b200_picture* pic)
{
  const b200_pic_params* p = &pic->params;
  if (p->dst_slot >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  const pic_geom g = geom_of(p);
  orc_surface* cur = &c->slot[p->dst_slot];
  int e = surf_ensure(cur, p);
  if (e) return e;
  for (uint32_t i = 0; i < pic->n_pu; i++) inter_pred_pu(c, cur, pic, &g, &pic->pus[i]);
  if (p->stop_after_stage == B200_STAGE_INTER_PRED) return 0;
  for (uint32_t i = 0; i < pic->n_tu; i++) recon_tu(cur, pic, &pic->tus[i]);
  if (p->stop_after_stage == B200_STAGE_RECON) return 0;
  if (!(p->flags & B200_PIC_SKIP_DEBLOCK) && pic->bs_map) {
    orc_deblock_picture(cur, pic, 1); /* all vertical edges of the picture first (deblock.cc:908-946) */
    orc_deblock_picture(cur, pic, 0);
  }
  if (p->stop_after_stage == B200_STAGE_DEBLOCK) return 0;
  if ((p->flags & B200_PIC_SAO_ENABLED) && !(p->flags & B200_PIC_SKIP_SAO)) {
    e = surf_ensure(&c->scratch, p);
    if (e) return e;
    int nc = p->chroma_format_idc ? 3 : 1;
    for (int k = 0; k < nc; k++) {
      size_t n = (size_t)(k ? cur->cw * cur->ch : cur->width * cur->height);
      memcpy(c->scratch.plane[k], cur->plane[k], n * sizeof(orc_pixel));
    }
    orc_sao_picture(&c->scratch, cur, pic);
  }
  return 0;
}
