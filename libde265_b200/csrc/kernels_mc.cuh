// kernels_mc.cuh — inter prediction: luma 8-tap / chroma 4-tap separable interpolation fused with
// (un)weighted uni/bi prediction.  Replaces mc_luma / mc_chroma (motion.cc:48-282), every
// put_hevc_qpel/epel table entry (fallback-motion.cc:262-636) and the four put_*_pred functions
// (fallback-motion.cc:33-256) for one picture's worth of PUs in ONE launch.
//
// Work split: the host cuts every PU into tiles of at most 16x16 luma samples (+ the co-located
// 8x8 Cb/Cr samples); one warp owns one tile, four warps per CTA.  Per list the warp runs the
// horizontal pass straight from the (border-padded) reference plane into a
// per-warp shared-memory int16 strip, then the vertical pass + weighting from shared memory, and
// writes the predicted samples with 4-sample (luma) / 2-sample (chroma) vector stores.
#pragma once
#include "dev_common.cuh"

#define MC_TILE 16
#define MC_LUMA_ROWS (MC_TILE + 7)
#define MC_CH_ROWS (MC_TILE / 2 + 3)
// per warp, per list: luma strip 23x16 + two chroma strips 11x8
#define MC_STRIP (MC_LUMA_ROWS * MC_TILE + 2 * MC_CH_ROWS * (MC_TILE / 2))

struct WeightParams {
  int mode;  // 0 uni unweighted, 1 bi average, 2 uni explicit, 3 bi explicit
  int w0, o0, w1, o1, log2wd;
};

// fallback-motion.cc:33-256 for one sample; a/b are the 14-bit intermediates of list 0/1 (or the used list in `a`)
__device__ __forceinline__ int weight_sample(int a, int b, const WeightParams& wp, int bd)
{
  int v;
  switch (wp.mode) {
    case 0: { int s = max(2, 14 - bd); v = (a + (1 << (s - 1))) >> s; break; }
    case 1: { int s = max(3, 15 - bd); v = (a + b + (1 << (s - 1))) >> s; break; }
    case 2: v = ((a * wp.w0 + (1 << (wp.log2wd - 1))) >> wp.log2wd) + wp.o0; break;
    default: v = (a * wp.w0 + b * wp.w1 + (int)((unsigned)(wp.o0 + wp.o1 + 1) << wp.log2wd)) >> (wp.log2wd + 1); break;
  }
  return clip_bd(v, bd);
}

template <typename P, int NT, bool PADDED = false>
__device__ __forceinline__ void mc_hpass(int16_t* strip, const uint8_t* ref, int pitch, int pw, int ph, int x_int, int y_int,
                                         int x_frac, int y_frac, int tw, int th, int bd, int lane, const int8_t* taps_h)
{
  if (!PADDED) {  // plain buffers (the per-block DSP table, dsp_table.cuh): every coordinate clamped as motion.cc:147-153 does
    constexpr int TWMAX = (NT == 8) ? MC_TILE : MC_TILE / 2;
    constexpr int BEFORE = (NT == 8) ? 3 : 1;
    const int before = y_frac ? BEFORE : 0;
    const int nrows = th + (y_frac ? NT - 1 : 0);
    const int shift1 = bd - 8;
    for (int idx = lane; idx < nrows * TWMAX; idx += B200_WARP) {
      const int r = idx / TWMAX, c = idx % TWMAX;
      if (c >= tw) continue;
      const int ya = clip3i(0, ph - 1, y_int + r - before);
      const P* row = row_ptr<P>(ref, pitch, ya);
      int v;
      if (x_frac == 0) {
        v = row[clip3i(0, pw - 1, x_int + c)];
      } else {
        int sum = 0;
#pragma unroll
        for (int k = 0; k < NT; k++) sum += taps_h[k] * (int)row[clip3i(0, pw - 1, x_int + c + k - BEFORE)];
        v = sum >> shift1;
      }
      strip[r * TWMAX + c] = (int16_t)v;
    }
    return;
  }
  // Rows [-before, th+after) when a vertical filter follows, else th rows.  Strip row stride = TWMAX.
  // The reference surfaces carry a replicated border (dpb.cuh), so the coordinate clamping of motion.cc:147-153 is done ONCE per
  // tile: the window of (tw + NT - 1) x (th + NT - 1) samples is moved to the border's rim when the motion vector points further
  // out (same samples), and the taps read it without any per-sample clamp.
  constexpr int TWMAX = (NT == 8) ? MC_TILE : MC_TILE / 2;
  constexpr int BEFORE = (NT == 8) ? 3 : 1;
  constexpr int PADX = (NT == 8) ? B200_PAD_X : B200_PAD_CX, PADY = (NT == 8) ? B200_PAD_Y : B200_PAD_CY;
  constexpr int WIN = TWMAX + NT - 1;
  const int wx = clip3i(-PADX, pw + PADX - WIN, x_int - BEFORE), wy = clip3i(-PADY, ph + PADY - WIN, y_int - BEFORE);
  const int r0 = y_frac ? 0 : BEFORE;  // first window row the strip needs
  const int nrows = th + (y_frac ? NT - 1 : 0);
  const int shift1 = bd - 8;
  for (int idx = lane; idx < nrows * TWMAX; idx += B200_WARP) {
    const int r = idx / TWMAX, c = idx % TWMAX;
    if (c >= tw) continue;
    const P* row = row_ptr<P>(ref, pitch, wy + r0 + r) + wx + c;
    int v;
    if (x_frac == 0) {
      v = row[BEFORE];
    } else {
      int sum = 0;
#pragma unroll
      for (int k = 0; k < NT; k++) sum += taps_h[k] * (int)row[k];
      v = sum >> shift1;
    }
    strip[r * TWMAX + c] = (int16_t)v;
  }
}

template <int NT>
__device__ __forceinline__ int mc_vsample(const int16_t* strip, int r, int c, int x_frac, int y_frac, int bd, const int8_t* taps_v)
{
  constexpr int TWMAX = (NT == 8) ? MC_TILE : MC_TILE / 2;
  int v;
  if (y_frac == 0) {
    v = strip[r * TWMAX + c];
    if (x_frac == 0) v = v << max(2, 14 - bd);  // full-sample position (fallback-motion.cc:262-302,431-485)
  } else {
    int sum = 0;
#pragma unroll
    for (int k = 0; k < NT; k++) sum += taps_v[k] * (int)strip[(r + k) * TWMAX + c];
    v = sum >> (x_frac == 0 ? bd - 8 : 6);
  }
  return (int)(int16_t)v;  // int16 storage with wrap-around (SURVEY App. A.1)
}

template <typename P>
__global__ void __launch_bounds__(128) k_inter_pred(DevPic pic, RefTable refs, const b200_pu* __restrict__ pus,
                                                    const b200_weight_entry* __restrict__ wts, const uint32_t* __restrict__ tiles,
                                                    int n_tiles)
{
  __shared__ int16_t s_strip[4][2][MC_STRIP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x * 4 + warp;
  if (tile >= n_tiles) return;
  const uint32_t t = tiles[tile];
  const b200_pu pu = pus[t & 0xFFFFF];
  const int tx = (t >> 20) & 3, ty = (t >> 22) & 3;
  const int x0 = pu.x + tx * MC_TILE, y0 = pu.y + ty * MC_TILE;
  const int tw = min(MC_TILE, pu.w - tx * MC_TILE), th = min(MC_TILE, pu.h - ty * MC_TILE);
  const bool use0 = pu.flags & B200_PU_PRED_L0, use1 = pu.flags & B200_PU_PRED_L1;
  const bool has_chroma = pic.chroma != 0;
  const int cwd = tw >> 1, chh = th >> 1;

  int xf[2], yf[2], xfc[2], yfc[2];
  bool missing[2] = {false, false};
#pragma unroll
  for (int l = 0; l < 2; l++) {
    if (!(l ? use1 : use0)) continue;
    const int slot = pu.ref_slot[l];
    const uint8_t* ry = (slot >= 0) ? refs.plane[slot][0] : nullptr;
    if (!ry) { missing[l] = true; continue; }
    const int mvx = pu.mv[l][0], mvy = pu.mv[l][1];
    xf[l] = mvx & 3; yf[l] = mvy & 3;
    int16_t* strip = s_strip[warp][l];
    mc_hpass<P, 8, true>(strip, ry, pic.pitch[0], pic.w, pic.h, x0 + (mvx >> 2), y0 + (mvy >> 2), xf[l], yf[l], tw, th, pic.bd_y, lane, k_qpel[xf[l]]);
    if (has_chroma) {
      // 4:2:0: chroma mv in eighth samples = luma mv (motion.cc:196-206)
      xfc[l] = mvx & 7; yfc[l] = mvy & 7;
      const int xi = (x0 >> 1) + (mvx >> 3), yi = (y0 >> 1) + (mvy >> 3);
      mc_hpass<P, 4, true>(strip + MC_LUMA_ROWS * MC_TILE, refs.plane[slot][1], pic.pitch[1], pic.cw, pic.ch, xi, yi, xfc[l], yfc[l], cwd, chh,
                     pic.bd_c, lane, k_epel[xfc[l]]);
      mc_hpass<P, 4, true>(strip + MC_LUMA_ROWS * MC_TILE + MC_CH_ROWS * (MC_TILE / 2), refs.plane[slot][2], pic.pitch[2], pic.cw, pic.ch, xi, yi,
                     xfc[l], yfc[l], cwd, chh, pic.bd_c, lane, k_epel[xfc[l]]);
    }
  }
  __syncwarp();

  // weighting parameters per plane (motion.cc:493-688)
  const bool bi = use0 && use1;
  const int lu = use0 ? 0 : 1;  // the list used for uni-prediction
  WeightParams wp[3];
  {
    const bool wgt = pu.flags & B200_PU_WEIGHTED;
    b200_weight_entry we;
    if (wgt) we = wts[pu.wt_idx];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      wp[c].mode = (bi ? 1 : 0) + (wgt ? 2 : 0);
      if (wgt) {
        wp[c].log2wd = c ? we.log2wd_chroma : we.log2wd_luma;
        if (bi) { wp[c].w0 = we.w[0][c]; wp[c].o0 = we.o[0][c]; wp[c].w1 = we.w[1][c]; wp[c].o1 = we.o[1][c]; }
        else { wp[c].w0 = we.w[lu][c]; wp[c].o0 = we.o[lu][c]; wp[c].w1 = 0; wp[c].o1 = 0; }
      }
    }
  }

  // ---- luma: lane -> 4 consecutive samples of one row; 8 rows per iteration ----
  {
    const int c0 = (lane & 3) * 4;
    for (int r = lane >> 2; r < th; r += 8) {
      if (c0 >= tw) continue;
      int res[4];
#pragma unroll
      for (int i = 0; i < 4; i++) {
        int a, b = 0;
        if (bi) {
          a = missing[0] ? (1 << 13) : mc_vsample<8>(s_strip[warp][0], r, c0 + i, xf[0], yf[0], pic.bd_y, k_qpel[yf[0]]);
          b = missing[1] ? (1 << 13) : mc_vsample<8>(s_strip[warp][1], r, c0 + i, xf[1], yf[1], pic.bd_y, k_qpel[yf[1]]);
        } else {
          a = missing[lu] ? (1 << 13) : mc_vsample<8>(s_strip[warp][lu], r, c0 + i, xf[lu], yf[lu], pic.bd_y, k_qpel[yf[lu]]);
        }
        res[i] = weight_sample(a, b, wp[0], pic.bd_y);
      }
      P* dst = row_ptr<P>(pic.cur[0], pic.pitch[0], y0 + r) + x0 + c0;
      if (sizeof(P) == 1) {
        *reinterpret_cast<uint32_t*>(dst) = (uint32_t)res[0] | ((uint32_t)res[1] << 8) | ((uint32_t)res[2] << 16) | ((uint32_t)res[3] << 24);
      } else {
        *reinterpret_cast<uint2*>(dst) = make_uint2((uint32_t)res[0] | ((uint32_t)res[1] << 16), (uint32_t)res[2] | ((uint32_t)res[3] << 16));
      }
    }
  }
  // ---- chroma: lane -> 2 consecutive samples of one row of Cb and of Cr ----
  if (has_chroma) {
    const int c0 = (lane & 3) * 2, r = lane >> 2;
    if (r < chh && c0 < cwd) {
#pragma unroll
      for (int pl = 0; pl < 2; pl++) {
        const int off = MC_LUMA_ROWS * MC_TILE + pl * MC_CH_ROWS * (MC_TILE / 2);
        int res[2];
#pragma unroll
        for (int i = 0; i < 2; i++) {
          int a, b = 0;
          if (bi) {
            a = missing[0] ? (1 << 13) : mc_vsample<4>(s_strip[warp][0] + off, r, c0 + i, xfc[0], yfc[0], pic.bd_c, k_epel[yfc[0]]);
            b = missing[1] ? (1 << 13) : mc_vsample<4>(s_strip[warp][1] + off, r, c0 + i, xfc[1], yfc[1], pic.bd_c, k_epel[yfc[1]]);
          } else {
            a = missing[lu] ? (1 << 13) : mc_vsample<4>(s_strip[warp][lu] + off, r, c0 + i, xfc[lu], yfc[lu], pic.bd_c, k_epel[yfc[lu]]);
          }
          res[i] = weight_sample(a, b, wp[1 + pl], pic.bd_c);
        }
        P* dst = row_ptr<P>(pic.cur[1 + pl], pic.pitch[1 + pl], (y0 >> 1) + r) + (x0 >> 1) + c0;
        if (sizeof(P) == 1) *reinterpret_cast<uint16_t*>(dst) = (uint16_t)(res[0] | (res[1] << 8));
        else *reinterpret_cast<uint32_t*>(dst) = (uint32_t)res[0] | ((uint32_t)res[1] << 16);
      }
    }
  }
}
