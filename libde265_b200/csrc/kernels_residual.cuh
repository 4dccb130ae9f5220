// kernels_residual.cuh — residual of SMALL transform units with sub-warp work splits and packed dot products.
//
// 72 % of the TUs of a typical picture are 4x4 and 22 % are 8x8 (a handful of coefficients each); a warp per TU
// wastes nearly every lane on them.  Here:
//   res4_lane     one LANE per 4x4 TU (32 TUs per warp): coefficients scattered into a lane-private, bank-conflict
//                 free shared-memory scratch (8 words), both transform passes in registers.
//   res8_quarter  8 lanes per 8x8 TU (4 TUs per warp): pass 1 lane = column, pass 2 lane = row (so a lane adds and
//                 stores one 8-sample row with a single vector read-modify-write).
// Both use dp2a: two vertically (pass 1) / horizontally (pass 2) adjacent int16 operands share a register, the
// int8 transform matrix is packed 4 rows per word (ResTables, built on the host from the core transform), so one
// instruction performs two MACs and the operand loads halve.
//
// Arithmetic follows scale_coefficients (transform.cc:361-642) and fallback-dct.cc exactly as tu_residual
// (kernels_recon.cuh) does: dequant with the 64-bit intermediate, its low 32 bits clipped to int16 (transform.cc:452-525), first-stage
// (sum + 64) >> 7 clipped to int16, second stage (sum + rnd) >> (20 - bd) (DST: clipped to int16 again),
// transform-skip / bypass / RDPCM / rotation (transform.cc:402-448, 548-596; fallback-dct.cc:81-91,161-225).
#pragma once
#include "dev_common.cuh"

struct __align__(16) ResTables {
  uint32_t m4[4];       // [i]      bytes (M4[0][i], M4[1][i], M4[2][i], M4[3][i]),  M_nT[j][i] = core[(32/nT) j][i]
  uint32_t m8[2][8];    // [jq][i]  bytes M8[4jq .. 4jq+3][i]
  uint32_t m16[4][16];
  uint32_t m32[8][32];
  uint32_t dst4[4];     // DST-VII 4x4 (fallback-dct.cc:260-265), same packing as m4
};
__constant__ ResTables c_res;

__device__ __forceinline__ int dp2a_lo(uint32_t a, uint32_t b, int c)
{
  int d;
  asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int dp2a_hi(uint32_t a, uint32_t b, int c)
{
  int d;
  asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int clip16(int v) { return min(max(v, -32768), 32767); }
// Residual scratch of the intra kernel: int16 with saturation.  Exact: the residual is only ever added to a prediction sample in
// [0, 2^bd) and clipped to that range (fallback-dct.h:65-73), and a residual beyond +-32767 saturates the sum either way.
typedef int16_t res_t;
__device__ __forceinline__ void res_store4(res_t* p, int a, int b, int c, int d)  // p 8-byte aligned
{
  *reinterpret_cast<uint2*>(p) = make_uint2(((uint32_t)clip16(a) & 0xffffu) | ((uint32_t)clip16(b) << 16), ((uint32_t)clip16(c) & 0xffffu) | ((uint32_t)clip16(d) << 16));
}
__device__ __forceinline__ uint32_t pack16(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }
__device__ __forceinline__ int lo16(uint32_t w) { return (int)(int16_t)(w & 0xffffu); }
__device__ __forceinline__ int hi16(uint32_t w) { return (int)w >> 16; }

// ---- dequantisation (transform.cc:452-525) ----
struct Dequant {
  const uint8_t* scl;  // scaling factors of this TU's matrix or null (flat 16, folded into bd_shift)
  int ls, qd, bd_shift;
  bool bypass, rotate;
};
__device__ __forceinline__ Dequant dequant_setup(const b200_tu& tu, const uint8_t* __restrict__ scaling, int bd)
{
  Dequant d;
  const int flags = tu.flags, log2 = tu.log2_size, nT = 1 << log2;
  d.bypass = flags & B200_TU_BYPASS;
  d.rotate = (flags & B200_TU_ROTATE) && (flags & (B200_TU_BYPASS | B200_TU_TSKIP));
  d.scl = nullptr;
  if ((flags & B200_TU_SCALING_LIST) && scaling) {
    int m = (nT == 32) ? 0 : tu.cidx;
    if (flags & B200_TU_INTER_MATRIX) m += (nT < 32) ? 3 : 1;
    const int base = (nT == 4) ? 0 : (nT == 8) ? 6 * 16 : (nT == 16) ? 6 * 16 + 6 * 64 : 6 * 16 + 6 * 64 + 6 * 256;
    d.scl = scaling + base + m * nT * nT;
  }
  d.bd_shift = bd + log2 - 5 - (d.scl ? 0 : 4);
  const int qp = tu.qp, qm = qp % 6;
  d.qd = qp / 6;
  d.ls = (qm == 0) ? 40 : (qm == 1) ? 45 : (qm == 2) ? 51 : (qm == 3) ? 57 : (qm == 4) ? 64 : 72;
  return d;
}
__device__ __forceinline__ int dequant_level(const Dequant& d, const b200_coeff c)
{
  if (d.bypass) return c.level;
  const long long fact = (long long)((d.scl ? d.scl[c.pos] : 1) * d.ls) << d.qd;
  const long long q = ((long long)c.level * fact + (1ll << (d.bd_shift - 1))) >> d.bd_shift;
  return clip16((int)(unsigned)q);  // the low 32 bits, clipped: the reference's Clip3(int, int, int) (transform.cc:522-523)
}

// dst[0..N) = Clip(dst + r) with one vector load and one vector store (N = 4 or 8 samples, naturally aligned)
template <typename P, int N>
__device__ __forceinline__ void add_row(P* p, const int (&r)[N], int bd)
{
  if (sizeof(P) == 1) {
    uint32_t w[N / 4];
    if (N == 4) w[0] = *reinterpret_cast<const uint32_t*>(p);
    else { const uint2 t = *reinterpret_cast<const uint2*>(p); w[0] = t.x; w[N / 4 - 1] = t.y; }
#pragma unroll
    for (int k = 0; k < N / 4; k++) {
      uint32_t o = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) o |= (uint32_t)clip_bd((int)((w[k] >> (8 * b)) & 0xff) + r[4 * k + b], bd) << (8 * b);
      w[k] = o;
    }
    if (N == 4) *reinterpret_cast<uint32_t*>(p) = w[0];
    else *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[N / 4 - 1]);
  } else {
    uint32_t w[N / 2];
    if (N == 4) { const uint2 t = *reinterpret_cast<const uint2*>(p); w[0] = t.x; w[1] = t.y; }
    else { const uint4 t = *reinterpret_cast<const uint4*>(p); w[0] = t.x; w[1] = t.y; w[N / 2 - 2] = t.z; w[N / 2 - 1] = t.w; }
#pragma unroll
    for (int k = 0; k < N / 2; k++)
      w[k] = (uint32_t)clip_bd((int)(w[k] & 0xffff) + r[2 * k], bd) | ((uint32_t)clip_bd((int)(w[k] >> 16) + r[2 * k + 1], bd) << 16);
    if (N == 4) *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1]);
    else *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[N / 2 - 2], w[N / 2 - 1]);
  }
}

// -------------------------------------------------------------------------------------------------
// One 4x4 TU per lane.  sc = this warp's scratch, 8 x 32 words, word k of lane l at sc[k*32 + l].
// TO_RES: res[x + 4y] (res_t, 8-byte aligned) receives the residual; else it is added onto dst (global memory).
// No warp-level synchronisation inside: lanes are independent, inactive lanes simply do not call.
// -------------------------------------------------------------------------------------------------
template <typename P, bool TO_RES>
__device__ __forceinline__ void res4_lane(const b200_tu& tu, const b200_coeff* __restrict__ co, const uint8_t* __restrict__ scaling, P* dst, int dstride,
                                          res_t* res, int bd, uint32_t* sc, int lane, const ResTables& tb)
{
#pragma unroll
  for (int k = 0; k < 8; k++) sc[k * 32 + lane] = 0;
  const int flags = tu.flags, n = tu.n_coeff;
  const Dequant dq = dequant_setup(tu, scaling, bd);
  {
    int16_t* sc16 = reinterpret_cast<int16_t*>(sc);
    for (int i = 0; i < n; i++) {
      const b200_coeff c = co[i];
      const int v = dequant_level(dq, c);
      const int pos = (dq.rotate ? 15 - c.pos : c.pos) & 15;
      const int j = pos >> 2, cc = pos & 3;  // row, column; words hold vertical pairs: word(cc, j>>1)
      sc16[((cc * 2 + (j >> 1)) * 32 + lane) * 2 + (j & 1)] = (int16_t)v;
    }
  }
  uint32_t w[8];
#pragma unroll
  for (int k = 0; k < 8; k++) w[k] = sc[k * 32 + lane];
  int r[16];  // r[x + 4y]
  if (flags & (B200_TU_BYPASS | B200_TU_TSKIP)) {
    const bool ts = !(flags & B200_TU_BYPASS);
    const int bd_shift = 20 - bd, rnd = 1 << (bd_shift - 1);
#pragma unroll
    for (int y = 0; y < 4; y++)
#pragma unroll
      for (int x = 0; x < 4; x++) {
        const uint32_t wd = w[x * 2 + (y >> 1)];
        int c = (y & 1) ? hi16(wd) : lo16(wd);
        if (ts) c = ((int)((unsigned)c << 7) + rnd) >> bd_shift;  // tsShift = 5 + log2(nT)
        r[x + 4 * y] = c;
      }
    if (flags & B200_TU_RDPCM_H) {
#pragma unroll
      for (int y = 0; y < 4; y++)
#pragma unroll
        for (int x = 1; x < 4; x++) r[x + 4 * y] += r[x - 1 + 4 * y];
    } else if (flags & B200_TU_RDPCM_V) {
#pragma unroll
      for (int x = 0; x < 4; x++)
#pragma unroll
        for (int y = 1; y < 4; y++) r[x + 4 * y] += r[x + 4 * (y - 1)];
    }
  } else {
    const bool dst7 = flags & B200_TU_DST;
    uint32_t m[4];
#pragma unroll
    for (int i = 0; i < 4; i++) m[i] = dst7 ? tb.dst4[i] : tb.m4[i];
    const int post_shift = 20 - bd, rnd2 = 1 << (post_shift - 1);
    uint32_t gp[4][2];  // first-stage rows, horizontally paired
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int g[4];
#pragma unroll
      for (int c = 0; c < 4; c++) g[c] = clip16(dp2a_hi(w[2 * c + 1], m[i], dp2a_lo(w[2 * c], m[i], 64)) >> 7);
      gp[i][0] = pack16(g[0], g[1]);
      gp[i][1] = pack16(g[2], g[3]);
    }
#pragma unroll
    for (int y = 0; y < 4; y++)
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int v = dp2a_hi(gp[y][1], m[i], dp2a_lo(gp[y][0], m[i], rnd2)) >> post_shift;
        r[i + 4 * y] = dst7 ? clip16(v) : v;
      }
  }
  if (TO_RES) {
#pragma unroll
    for (int y = 0; y < 4; y++) res_store4(res + 4 * y, r[4 * y], r[4 * y + 1], r[4 * y + 2], r[4 * y + 3]);
  } else {
#pragma unroll
    for (int y = 0; y < 4; y++) {
      const int rr[4] = {r[4 * y], r[4 * y + 1], r[4 * y + 2], r[4 * y + 3]};
      add_row<P, 4>(dst + (size_t)y * dstride, rr, bd);
    }
  }
}

// -------------------------------------------------------------------------------------------------
// One 8x8 TU per quarter-warp.  qs = this quarter's scratch, 64 words: [0,32) coefficients, column-major int16
// (column c = 4 words = vertical pairs), [32,64) first-stage rows.  ALL 32 lanes must call (two __syncwarp inside);
// quarters without a TU pass active = false.  TO_RES: res[x + 8y] (res_t, 8-byte aligned).
// -------------------------------------------------------------------------------------------------
template <typename P, bool TO_RES>
__device__ __forceinline__ void res8_quarter(bool active, const b200_tu& tu, const b200_coeff* __restrict__ co, const uint8_t* __restrict__ scaling, P* dst,
                                             int dstride, res_t* res, int bd, uint32_t* qs, int sub, const ResTables& tb)
{
  *reinterpret_cast<uint4*>(qs + sub * 4) = make_uint4(0, 0, 0, 0);
  __syncwarp();
  const int flags = active ? tu.flags : 0;
  int16_t* c16 = reinterpret_cast<int16_t*>(qs);
  int16_t* g16 = reinterpret_cast<int16_t*>(qs + 32);
  if (active) {
    const Dequant dq = dequant_setup(tu, scaling, bd);
    const int n = tu.n_coeff;
    for (int i = sub; i < n; i += 8) {
      const b200_coeff c = co[i];
      const int v = dequant_level(dq, c);
      const int pos = (dq.rotate ? 63 - c.pos : c.pos) & 63;
      c16[(pos & 7) * 8 + (pos >> 3)] = (int16_t)v;
    }
  }
  __syncwarp();
  const bool special = flags & (B200_TU_BYPASS | B200_TU_TSKIP);
  const int post_shift = 20 - bd, rnd2 = 1 << (post_shift - 1);
  if (active && special) {
    // lane = row (or column for vertical RDPCM): coefficient (x, y) = c16[x*8 + y]
    const bool ts = !(flags & B200_TU_BYPASS);
    const bool vert = flags & B200_TU_RDPCM_V, acc = flags & (B200_TU_RDPCM_H | B200_TU_RDPCM_V);
    int sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int x = vert ? sub : k, y = vert ? k : sub;
      int c = c16[x * 8 + y];
      if (ts) c = ((int)((unsigned)c << 8) + rnd2) >> post_shift;  // tsShift = 5 + log2(nT)
      sum = acc ? sum + c : c;
      if (TO_RES) res[x + 8 * y] = (res_t)clip16(sum);
      else dst[x + (size_t)y * dstride] = (P)clip_bd((int)dst[x + (size_t)y * dstride] + sum, bd);
    }
  } else if (active) {
    // pass 1: lane = column
    const uint4 w = *reinterpret_cast<const uint4*>(qs + sub * 4);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const uint32_t m0 = tb.m8[0][i], m1 = tb.m8[1][i];
      int s = dp2a_lo(w.x, m0, 64);
      s = dp2a_hi(w.y, m0, s);
      s = dp2a_lo(w.z, m1, s);
      s = dp2a_hi(w.w, m1, s);
      g16[i * 8 + sub] = (int16_t)clip16(s >> 7);
    }
  }
  __syncwarp();
  if (active && !special) {
    // pass 2: lane = row
    const uint4 g = *reinterpret_cast<const uint4*>(qs + 32 + sub * 4);
    int r[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const uint32_t m0 = tb.m8[0][i], m1 = tb.m8[1][i];
      int s = dp2a_lo(g.x, m0, rnd2);
      s = dp2a_hi(g.y, m0, s);
      s = dp2a_lo(g.z, m1, s);
      s = dp2a_hi(g.w, m1, s);
      r[i] = s >> post_shift;
    }
    if (TO_RES) {
      res_store4(res + 8 * sub, r[0], r[1], r[2], r[3]);
      res_store4(res + 8 * sub + 4, r[4], r[5], r[6], r[7]);
    } else {
      add_row<P, 8>(dst + (size_t)sub * dstride, r, bd);
    }
  }
  __syncwarp();
}
