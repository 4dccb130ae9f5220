// kernels_mct.cuh — 8-bit inter prediction, tiled and TMA-staged (the roofline-graded kernel, second generation).
//
// Replaces mc_luma / mc_chroma (motion.cc:48-282), every put_hevc_qpel/epel table entry (fallback-motion.cc:262-636) and the
// four put_*_pred functions (fallback-motion.cc:33-256) for one picture's worth of PUs in ONE launch.
//
// Work split.  The host cuts every PU into TILES of at most 16x16 luma samples (+ the co-located 8x8 Cb/Cr samples) and sorts
// them into 8 classes (wide: more than 8 columns | bi-predicted | tall: more than 8 rows); a BATCH is 8 tiles of one class.
// Persistent CTAs of MCT_THREADS compute threads (+ one producer warp) take batches; inside a batch all threads run over FLAT task lists, so lanes stay busy for
// every PU size and nothing in a task body depends on the PU shape except two uniform loop bounds:
//   stage   16 producer threads (one per tile and list) decode the PU records and issue one 2-D TMA box (48 bytes x 26 rows,
//           luma) and one 3-D TMA box (32 bytes x 14 rows x {Cb, Cr}) per used reference list into shared memory, completion
//           on an mbarrier.  TMA box origins must be 16-byte aligned in the innermost dimension (measured: an unaligned origin
//           raises "illegal instruction", tools/tma_probe2.cu), so the box starts at the 16-byte boundary left of the window and
//           pass 1 picks the window up at its byte offset.  Reference surfaces carry a replicated border (dpb.cuh), so
//           there is no coordinate clamping here: a window further out than the border is moved to the border's rim.
//           The next batch's boxes are issued as soon as pass 1 has consumed the current windows (they land during pass 2).
//   pass 1  horizontal filter on bytes, as the reference orders it (fallback-motion.cc:492-560): a task = 2 window rows x 8
//           columns of one tile and list: 4 aligned words + funnel shifts give 16 source bytes per row, output j is
//           dp4a(b0,T[j][0]) + dp4a(b1,T[j][1]) + dp4a(b2,T[j][2]) with the 8 taps pre-shifted by j bytes (11 dp4a per 4
//           outputs).  The two rows' results (|v| < 2^15: no shift at 8 bit) are interleaved into VERTICAL int16 pairs and
//           stored as one "pair row" with two 16-byte stores.
//   pass 2  vertical filter on the pair rows with dp2a (4 per even output row, 5 per odd one: taps pre-packed for both
//           parities), >> 6 with the reference's int16 wrap (one bit-field extract), weighting (all four modes through one
//           branch-free multiply-add-shift-offset form), saturation, and 32 outputs per lane leave as whole row segments:
//           16 columns x 2 rows (one 128-bit store per row) in the wide classes, 8 columns x 4 rows (64-bit stores) otherwise.
// Integer phases use identity taps, so there is one code path.  Missing references predict mid-grey (motion.cc:362).
//
// The task bodies are __host__ __device__ so that tests/mct_emul.cu can run the very same code on the CPU against the oracle
// (TMA replaced by a window copy); only the staging / synchronisation below is device-only.
#pragma once
#include "dev_common.cuh"
#include "kernels_mc8.cuh"  // Mc8Tables, Mc8Weight, mc8_weight

#define MCT_HD __host__ __device__ __forceinline__

#ifndef MCT_THREADS
#define MCT_THREADS 192                  // compute threads per CTA (warps 0..MCT_THREADS/32-1); one more warp is the producer. 576 pass-1 and 192 pass-2 tasks per big batch: 3 + 1 full rounds
#endif
#ifndef MCT_TLS
#define MCT_TLS 32                       // tile-list items per batch with the small boxes (a power of two); half as many with the big ones
#endif
#define MCT_L2TLS (MCT_TLS == 32 ? 5 : MCT_TLS == 16 ? 4 : 3)
#define MCT_MAX_TL MCT_TLS
#define MCT_MAX_TILES MCT_TLS            // tiles per batch (small, uni-predicted)
#define MCT_WIN_BYTES (MCT_TLS * 1280)   // window region: TLS/2 x (1280 + 896) big  |  TLS x (640 + 640) small
#define MCT_INT_WORDS (MCT_TLS * 200)    // intermediate region: TLS/2 x (244 + 148) big  |  TLS x (100 + 100) small
// big boxes (tiles wider or taller than 8): luma 48 bytes x 26 rows (16-byte aligned origin + up to 15 + 23 columns; 23 rows + up
// to 3 rows of bank skew), chroma 32 bytes x 14 rows x {Cb, Cr}
#define MCT_LWB_PITCH 48
#define MCT_LWB_ROWS 26
#define MCT_LWB_SLOT 1280
#define MCT_CWB_PITCH 32
#define MCT_CWB_ROWS 14
#define MCT_CWB_SLOT 896
// small boxes (tiles of at most 8x8): luma 32 bytes x 18 rows (up to 15 + 15 columns, 15 rows + skew), chroma 32 x 10 x 2
#define MCT_LWS_PITCH 32
#define MCT_LWS_ROWS 18
#define MCT_LWS_SLOT 640
#define MCT_CWS_PITCH 32
#define MCT_CWS_ROWS 10
#define MCT_CWS_SLOT 640

// tile word: bits 0-19 PU index, 20-21 x offset / 16, 22-23 y offset / 16, 24-26 class; 0xFFFFFFFF = padding
#define MCT_CLASS_WIDE 1
#define MCT_CLASS_BI 2
#define MCT_CLASS_TALL 4
#define MCT_TILE_WORD(pu, tx, ty, cls) ((uint32_t)(pu) | ((uint32_t)(tx) << 20) | ((uint32_t)(ty) << 22) | ((uint32_t)(cls) << 24))
#define MCT_INVALID 0xFFFFFFFFu
// tiles per batch of a class: 32 tile-list items with the small boxes (narrow and short), 16 otherwise
#define MCT_CLASS_TILES(cls) ((((cls) & (MCT_CLASS_WIDE | MCT_CLASS_TALL)) ? MCT_TLS / 2 : MCT_TLS) >> (((cls) & MCT_CLASS_BI) ? 1 : 0))
// batch word (host planner -> kernel): bits 0-27 index of the batch's first tile word, 28-30 class
#define MCT_BATCH_WORD(first, cls) ((uint32_t)(first) | ((uint32_t)(cls) << 28))

struct MctTile {
  int dst_y, dst_c;       // byte offsets of the tile's first luma / chroma sample in the destination planes
  uint32_t shape;         // tw | th << 8 | nl << 16 | valid << 24 | plain << 25 (plain: no explicit weights, fallback-motion.cc:33-62)
  uint32_t l[2];          // per list slot, luma: window byte offset | pass-1 tap table index << 8 | vertical phase << 16 | final shift << 24 | missing << 31
  uint32_t c[2];          // the same for chroma
  Mc8Weight w[3];
};
#define MCT_TW(sh) ((int)((sh) & 0xff))
#define MCT_TH(sh) ((int)(((sh) >> 8) & 0xff))
#define MCT_NL(sh) ((int)(((sh) >> 16) & 0xff))
#define MCT_VALID(sh) (((sh) >> 24) & 1)
#define MCT_PLAIN(sh) (((sh) >> 25) & 1)
#define MCT_XO(w) ((int)((w) & 0xff))
#define MCT_HIDX(w) ((int)(((w) >> 8) & 0xff))
#define MCT_YF(w) ((int)(((w) >> 16) & 0xff))
#define MCT_SH6(w) ((int)(((w) >> 24) & 0x7f))
#define MCT_MISSING(w) ((w) >> 31)

// ---- task-space and shared-memory geometry of a batch class ----
struct MctGeom {
  int small;            // small boxes
  int nl, ntl, ntiles;  // list slots per tile (1 | 2), tile-list items and tiles per batch
  int nco;              // luma column octets per tile (1 | 2)
  int nrp, nrpc;        // pair rows of the luma / chroma intermediate that pass 1 produces
  int nu, nuc;          // output row pairs per tile in pass 2 (luma, chroma)
  int l2ntl, l2nu, l2nuc;  // log2 of ntl / nu / nuc (task decode by shifts)
  int n1l, n1c;         // pass-1 task counts (luma, chroma)
  int n2l, n2c;         // pass-2 task counts
  int lw_pitch, lw_slot, cw_off, cw_pitch, cw_plane, cw_slot;        // window region (bytes)
  int li_pitch, li_words, ci_off, ci_pitch, ci_plane, ci_words;      // intermediate region (words)
};
MCT_HD MctGeom mct_geom(int cls)
{
  MctGeom g;
  const bool wide = cls & MCT_CLASS_WIDE, tall = cls & MCT_CLASS_TALL;
  g.small = !wide && !tall;
  g.nl = (cls & MCT_CLASS_BI) ? 2 : 1;
  g.ntl = g.small ? MCT_TLS : MCT_TLS / 2;
  g.ntiles = g.ntl / g.nl;
  g.nco = wide ? 2 : 1;
  g.nrp = tall ? 12 : 8;
  g.nrpc = tall ? 6 : 4;
  g.nu = tall ? 8 : 4;
  g.nuc = tall ? 4 : 2;
  g.l2ntl = g.small ? MCT_L2TLS : MCT_L2TLS - 1; g.l2nu = tall ? 3 : 2; g.l2nuc = tall ? 2 : 1;
  g.n1l = g.nrp * g.ntl * g.nco;
  g.n1c = g.nrpc * g.ntl * 2;
  g.n2l = g.ntiles * g.nco * g.nu;   // 8 columns x 2 rows per task
  g.n2c = g.ntiles * 2 * g.nuc;
  if (g.small) {
    g.lw_pitch = MCT_LWS_PITCH; g.lw_slot = MCT_LWS_SLOT; g.cw_off = MCT_TLS * MCT_LWS_SLOT; g.cw_pitch = MCT_CWS_PITCH;
    g.cw_plane = MCT_CWS_PITCH * MCT_CWS_ROWS; g.cw_slot = MCT_CWS_SLOT;
    g.li_pitch = 12; g.li_words = 100; g.ci_off = MCT_TLS * 100; g.ci_pitch = 12; g.ci_plane = 48; g.ci_words = 100;
  } else {
    g.lw_pitch = MCT_LWB_PITCH; g.lw_slot = MCT_LWB_SLOT; g.cw_off = MCT_TLS / 2 * MCT_LWB_SLOT; g.cw_pitch = MCT_CWB_PITCH;
    g.cw_plane = MCT_CWB_PITCH * MCT_CWB_ROWS; g.cw_slot = MCT_CWB_SLOT;
    // slot strides of 244 / 148 words (= 20 mod 32): the 8 lanes of a 16-byte store phase, one slot each, hit 8 different bank groups
    // (240 / 144 = 16 mod 32 put them on two)
    g.li_pitch = 20; g.li_words = 244; g.ci_off = MCT_TLS / 2 * 244; g.ci_pitch = 12; g.ci_plane = 72; g.ci_words = 148;
  }
  return g;
}

#ifndef MCT_DB
#define MCT_DB 1  // window buffers: 2 = the producer fetches a whole batch ahead (the boxes of batch n+1 land while batch n is computed).
                  // The second buffer costs shared memory and with it resident CTAs per SM: 1 is the default.
#endif
struct MctShared {
  alignas(128) uint8_t win[MCT_DB][MCT_WIN_BYTES];
  alignas(16) uint32_t interm[MCT_INT_WORDS];
  MctTile info[2][MCT_MAX_TILES];
  MctGeom geom[2];
  alignas(16) Mc8Tables tab;
  alignas(8) unsigned long long bar[2], bar_empty[2];
};

// ---- portable forms of the packed-integer instructions (host emulation) ----
MCT_HD int mct_dp4a(uint32_t a, uint32_t b, int c)  // unsigned bytes of a x signed bytes of b
{
#ifdef __CUDA_ARCH__
  return dp4a_us(a, b, c);
#else
  for (int i = 0; i < 4; i++) c += (int)((a >> (8 * i)) & 0xff) * (int)(int8_t)((b >> (8 * i)) & 0xff);
  return c;
#endif
}
MCT_HD int mct_dp2a_lo(uint32_t a, uint32_t b, int c)  // int16 halves of a x signed bytes 0,1 of b
{
#ifdef __CUDA_ARCH__
  return dp2a_lo_ss(a, b, c);
#else
  return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)(b & 0xff) + (int)(int16_t)(a >> 16) * (int)(int8_t)((b >> 8) & 0xff);
#endif
}
MCT_HD int mct_dp2a_hi(uint32_t a, uint32_t b, int c)  // int16 halves of a x signed bytes 2,3 of b
{
#ifdef __CUDA_ARCH__
  return dp2a_hi_ss(a, b, c);
#else
  return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)((b >> 16) & 0xff) + (int)(int16_t)(a >> 16) * (int)(int8_t)((b >> 24) & 0xff);
#endif
}
MCT_HD uint32_t mct_funnel(uint32_t lo, uint32_t hi, int sh)  // bytes of hi:lo starting at bit sh (sh in 0, 8, 16, 24)
{
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, sh);
#else
  return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}
MCT_HD uint32_t mct_pack16(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }
MCT_HD int mct_wrap16(int v, int shift)  // (v >> shift) as int16 with wrap-around (SURVEY App. A.1)
{
#ifdef __CUDA_ARCH__
  return shr_wrap16(v, shift);
#else
  return (int)(int16_t)(uint16_t)((uint32_t)v >> shift);
#endif
}
MCT_HD int mct_clip3(int lo, int hi, int v) { return v < lo ? lo : v > hi ? hi : v; }
MCT_HD int mct_sat_u8(int v)
{
#ifdef __CUDA_ARCH__
  return sat_u8(v);
#else
  return v < 0 ? 0 : v > 255 ? 255 : v;
#endif
}

// ---- pass 1, luma: task -> (pair row rp, tile-list item, column octet) ----
MCT_HD void mct_pass1_luma(int t, const MctGeom& g, const MctTile* info, const uint8_t* win, uint32_t* interm, const Mc8Tables& tab)
{
  const int co = g.nco == 2 ? (t & 1) : 0;
  const int u = g.nco == 2 ? (t >> 1) : t;
  const int tli = u & (g.ntl - 1), rp = u >> g.l2ntl;
  const int tile = g.nl == 2 ? (tli >> 1) : tli, s = g.nl == 2 ? (tli & 1) : 0;
  const MctTile& ti = info[tile];
  const uint32_t shape = ti.shape, lw = ti.l[s];
  if (!MCT_VALID(shape) || MCT_MISSING(lw) || 2 * rp >= MCT_TH(shape) + 7 || 8 * co >= MCT_TW(shape)) return;
  uint32_t T[4][3];
  {  // 12 words = three 16-byte loads (qh[f] is 48 bytes, the table 16-byte aligned)
    const uint4* tp = reinterpret_cast<const uint4*>(&tab.qh[MCT_HIDX(lw)][0][0]);
    const uint4 t0 = tp[0], t1 = tp[1], t2 = tp[2];
    T[0][0] = t0.x; T[0][1] = t0.y; T[0][2] = t0.z; T[1][0] = t0.w; T[1][1] = t1.x; T[1][2] = t1.y;
    T[2][0] = t1.z; T[2][1] = t1.w; T[2][2] = t2.x; T[3][0] = t2.y; T[3][1] = t2.z; T[3][2] = t2.w;
  }
  const int b = MCT_XO(lw) + 8 * co, sh = (b & 3) * 8;
  const uint8_t* base = win + tli * g.lw_slot + (2 * rp + (tli & 3)) * g.lw_pitch + (b & ~3);
  int o[2][8];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const uint32_t* wp_ = reinterpret_cast<const uint32_t*>(base + i * g.lw_pitch);
    const uint32_t w0 = wp_[0], w1 = wp_[1], w2 = wp_[2], w3 = wp_[3], w4 = wp_[4];
    uint32_t sb[4];
    sb[0] = mct_funnel(w0, w1, sh); sb[1] = mct_funnel(w1, w2, sh); sb[2] = mct_funnel(w2, w3, sh); sb[3] = mct_funnel(w3, w4, sh);
#pragma unroll
    for (int q = 0; q < 2; q++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        int v = mct_dp4a(sb[q], T[j][0], 0);
        v = mct_dp4a(sb[q + 1], T[j][1], v);
        if (j > 0) v = mct_dp4a(sb[q + 2], T[j][2], v);
        o[i][4 * q + j] = v;
      }
  }
  uint32_t* dst = interm + tli * g.li_words + rp * g.li_pitch + 8 * co;
  uint4 a, c;
  a.x = mct_pack16(o[0][0], o[1][0]); a.y = mct_pack16(o[0][1], o[1][1]); a.z = mct_pack16(o[0][2], o[1][2]); a.w = mct_pack16(o[0][3], o[1][3]);
  c.x = mct_pack16(o[0][4], o[1][4]); c.y = mct_pack16(o[0][5], o[1][5]); c.z = mct_pack16(o[0][6], o[1][6]); c.w = mct_pack16(o[0][7], o[1][7]);
  *reinterpret_cast<uint4*>(dst) = a;
  *reinterpret_cast<uint4*>(dst + 4) = c;
}

// ---- pass 1, chroma: task -> (pair row, tile-list item, plane); 8 columns x 2 rows ----
MCT_HD void mct_pass1_chroma(int t, const MctGeom& g, const MctTile* info, const uint8_t* win, uint32_t* interm, const Mc8Tables& tab)
{
  const int pl = t & 1, u = t >> 1;
  const int tli = u & (g.ntl - 1), rp = u >> g.l2ntl;
  const int tile = g.nl == 2 ? (tli >> 1) : tli, s = g.nl == 2 ? (tli & 1) : 0;
  const MctTile& ti = info[tile];
  const uint32_t shape = ti.shape, cw_ = ti.c[s];
  if (!MCT_VALID(shape) || MCT_MISSING(cw_) || 2 * rp >= (MCT_TH(shape) >> 1) + 3) return;
  uint32_t T[4][2];
  {  // 8 words = two 16-byte loads (eh starts 320 bytes into the table, eh[f] is 32 bytes)
    const uint4* tp = reinterpret_cast<const uint4*>(&tab.eh[MCT_HIDX(cw_)][0][0]);
    const uint4 t0 = tp[0], t1 = tp[1];
    T[0][0] = t0.x; T[0][1] = t0.y; T[1][0] = t0.z; T[1][1] = t0.w; T[2][0] = t1.x; T[2][1] = t1.y; T[3][0] = t1.z; T[3][1] = t1.w;
  }
  const int b = MCT_XO(cw_), sh = (b & 3) * 8;
  const uint8_t* base = win + g.cw_off + tli * g.cw_slot + pl * g.cw_plane + (2 * rp + (tli & 3)) * g.cw_pitch + (b & ~3);
  int o[2][8];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const uint32_t* wp_ = reinterpret_cast<const uint32_t*>(base + i * g.cw_pitch);
    const uint32_t w0 = wp_[0], w1 = wp_[1], w2 = wp_[2], w3 = wp_[3];
    uint32_t sb[3];
    sb[0] = mct_funnel(w0, w1, sh); sb[1] = mct_funnel(w1, w2, sh); sb[2] = mct_funnel(w2, w3, sh);
#pragma unroll
    for (int q = 0; q < 2; q++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        int v = mct_dp4a(sb[q], T[j][0], 0);
        if (j > 0) v = mct_dp4a(sb[q + 1], T[j][1], v);
        o[i][4 * q + j] = v;
      }
  }
  uint32_t* dst = interm + g.ci_off + tli * g.ci_words + pl * g.ci_plane + rp * g.ci_pitch;
  uint4 a, c;
  a.x = mct_pack16(o[0][0], o[1][0]); a.y = mct_pack16(o[0][1], o[1][1]); a.z = mct_pack16(o[0][2], o[1][2]); a.w = mct_pack16(o[0][3], o[1][3]);
  c.x = mct_pack16(o[0][4], o[1][4]); c.y = mct_pack16(o[0][5], o[1][5]); c.z = mct_pack16(o[0][6], o[1][6]); c.w = mct_pack16(o[0][7], o[1][7]);
  *reinterpret_cast<uint4*>(dst) = a;
  *reinterpret_cast<uint4*>(dst + 4) = c;
}

// Vertical 8-tap filter of 8 columns x 2 rows (an even row and the next) from the 5 pair rows at `src`:
// out[i][c], already shifted / wrapped to the reference's int16 intermediate.
MCT_HD void mct_vpair8(const uint32_t* src, int pitch, const uint32_t (&tv)[5], int sh6, int (&out)[2][8])
{
#pragma unroll
  for (int c4 = 0; c4 < 2; c4++) {
    uint32_t V[5][4];
#pragma unroll
    for (int p = 0; p < 5; p++) {
      const uint4 q = *reinterpret_cast<const uint4*>(src + p * pitch + 4 * c4);
      V[p][0] = q.x; V[p][1] = q.y; V[p][2] = q.z; V[p][3] = q.w;
    }
#pragma unroll
    for (int c = 0; c < 4; c++) {
      int e = mct_dp2a_lo(V[0][c], tv[0], 0);
      e = mct_dp2a_hi(V[1][c], tv[0], e);
      e = mct_dp2a_lo(V[2][c], tv[1], e);
      e = mct_dp2a_hi(V[3][c], tv[1], e);
      int o = mct_dp2a_lo(V[0][c], tv[2], 0);
      o = mct_dp2a_hi(V[1][c], tv[2], o);
      o = mct_dp2a_lo(V[2][c], tv[3], o);
      o = mct_dp2a_hi(V[3][c], tv[3], o);
      o = mct_dp2a_lo(V[4][c], tv[4], o);
      out[0][4 * c4 + c] = mct_wrap16(e, sh6);
      out[1][4 * c4 + c] = mct_wrap16(o, sh6);
    }
  }
}

// Vertical 4-tap filter (chroma): 8 columns x 2 rows from 3 pair rows.
MCT_HD void mct_vpair4(const uint32_t* src, int pitch, const uint32_t (&tv)[3], int sh6, int (&out)[2][8])
{
#pragma unroll
  for (int c4 = 0; c4 < 2; c4++) {
    uint32_t V[3][4];
#pragma unroll
    for (int p = 0; p < 3; p++) {
      const uint4 q = *reinterpret_cast<const uint4*>(src + p * pitch + 4 * c4);
      V[p][0] = q.x; V[p][1] = q.y; V[p][2] = q.z; V[p][3] = q.w;
    }
#pragma unroll
    for (int c = 0; c < 4; c++) {
      int e = mct_dp2a_lo(V[0][c], tv[0], 0);
      e = mct_dp2a_hi(V[1][c], tv[0], e);
      int o = mct_dp2a_lo(V[0][c], tv[1], 0);
      o = mct_dp2a_hi(V[1][c], tv[1], o);
      o = mct_dp2a_lo(V[2][c], tv[2], o);
      out[0][4 * c4 + c] = mct_wrap16(e, sh6);
      out[1][4 * c4 + c] = mct_wrap16(o, sh6);
    }
  }
}

// four values saturated to bytes, v0 in the lowest byte: two cvt.pack.sat (I2IP) instead of four saturating converts + merges
MCT_HD uint32_t mct_pack_sat4(int v0, int v1, int v2, int v3)
{
#ifdef __CUDA_ARCH__
  uint32_t hi, d;
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(v3), "r"(v2), "r"(0));
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(v1), "r"(v0), "r"(hi));
  return d;
#else
  return (uint32_t)mct_sat_u8(v0) | ((uint32_t)mct_sat_u8(v1) << 8) | ((uint32_t)mct_sat_u8(v2) << 16) | ((uint32_t)mct_sat_u8(v3) << 24);
#endif
}
MCT_HD uint32_t mct_weight4(const int* a, const int* b, const Mc8Weight& w)
{
  int v[4];
#pragma unroll
  for (int k = 0; k < 4; k++) v[k] = ((a[k] * w.w0 + b[k] * w.w1 + w.rnd) >> w.shift) + w.off;
  return mct_pack_sat4(v[0], v[1], v[2], v[3]);
}
MCT_HD uint32_t mct_plain4(const int* a, const int* b, int rnd, int shift)  // (a + 32) >> 6 resp. (a + b + 64) >> 7 (fallback-motion.cc:33-62); b = 0 for uni
{
  return mct_pack_sat4((a[0] + b[0] + rnd) >> shift, (a[1] + b[1] + rnd) >> shift, (a[2] + b[2] + rnd) >> shift, (a[3] + b[3] + rnd) >> shift);
}

// Row segment store: nbytes (<= 8; multiple of 4 for luma, of 2 for chroma) of the two words to dst, widest aligned form available.
MCT_HD void mct_store_row(uint8_t* dst, uint32_t w0, uint32_t w1, int nbytes)
{
  if (nbytes == 8 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
    *reinterpret_cast<uint2*>(dst) = make_uint2(w0, w1);
  } else if ((nbytes & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(dst) = w0;
    if (nbytes == 8) *reinterpret_cast<uint32_t*>(dst + 4) = w1;
  } else {
    for (int k = 0; k < nbytes / 2; k++) *reinterpret_cast<uint16_t*>(dst + 2 * k) = (uint16_t)((k < 2 ? w0 : w1) >> (16 * (k & 1)));
  }
}

// ---- pass 2, luma: task -> (tile, column octet, output row pair); 8 columns x 2 rows ----
MCT_HD void mct_pass2_luma(int t, const MctGeom& g, const MctTile* info, const uint32_t* interm, const Mc8Tables& tab, uint8_t* plane, int pitch)
{
  const int u = t & (g.nu - 1), tc = t >> g.l2nu;
  const int co = g.nco == 2 ? (tc & 1) : 0, tile = g.nco == 2 ? (tc >> 1) : tc;
  const MctTile& ti = info[tile];
  const uint32_t shape = ti.shape;
  const int y0 = 2 * u, tw = MCT_TW(shape), th = MCT_TH(shape), nl = MCT_NL(shape);
  if (!MCT_VALID(shape) || y0 >= th || 8 * co >= tw) return;
  int v[2][2][8];
#pragma unroll
  for (int s = 0; s < 2; s++) {
    const uint32_t lw = s < nl ? ti.l[s] : 0x80000000u;
    if (!MCT_MISSING(lw)) {
      uint32_t tv[5];
#pragma unroll
      for (int k = 0; k < 5; k++) tv[k] = tab.qv[MCT_YF(lw)][k];
      mct_vpair8(interm + (tile * g.nl + s) * g.li_words + u * g.li_pitch + 8 * co, g.li_pitch, tv, MCT_SH6(lw), v[s]);
    } else {
      const int fill = s < nl ? (1 << 13) : 0;  // missing reference: mid-grey intermediate (motion.cc:362)
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int c = 0; c < 8; c++) v[s][i][c] = fill;
    }
  }
  const Mc8Weight w = ti.w[0];
  const int nbytes = tw - 8 * co < 8 ? tw - 8 * co : 8;
  uint8_t* dst = plane + ti.dst_y + (size_t)y0 * pitch + 8 * co;
  const int nr = th - y0 < 2 ? 1 : 2;
  if (MCT_PLAIN(shape)) {
#pragma unroll
    for (int i = 0; i < 2; i++)
      if (i < nr) mct_store_row(dst + (size_t)i * pitch, mct_plain4(&v[0][i][0], &v[1][i][0], w.rnd, w.shift), mct_plain4(&v[0][i][4], &v[1][i][4], w.rnd, w.shift), nbytes);
  } else {
#pragma unroll
    for (int i = 0; i < 2; i++)
      if (i < nr) mct_store_row(dst + (size_t)i * pitch, mct_weight4(&v[0][i][0], &v[1][i][0], w), mct_weight4(&v[0][i][4], &v[1][i][4], w), nbytes);
  }
}

// ---- pass 2, chroma: task -> (tile, plane, output row pair); 8 columns x 2 rows ----
MCT_HD void mct_pass2_chroma(int t, const MctGeom& g, const MctTile* info, const uint32_t* interm, const Mc8Tables& tab, uint8_t* cb, uint8_t* cr, int pitch)
{
  const int u = t & (g.nuc - 1), tp_ = t >> g.l2nuc;
  const int pl = tp_ & 1, tile = tp_ >> 1;
  const MctTile& ti = info[tile];
  const uint32_t shape = ti.shape;
  const int y0 = 2 * u, ch = MCT_TH(shape) >> 1, cwd = MCT_TW(shape) >> 1, nl = MCT_NL(shape);
  if (!MCT_VALID(shape) || y0 >= ch) return;
  int v[2][2][8];
#pragma unroll
  for (int s = 0; s < 2; s++) {
    const uint32_t cw_ = s < nl ? ti.c[s] : 0x80000000u;
    if (!MCT_MISSING(cw_)) {
      uint32_t tv[3];
#pragma unroll
      for (int k = 0; k < 3; k++) tv[k] = tab.ev[MCT_YF(cw_)][k];
      mct_vpair4(interm + g.ci_off + (tile * g.nl + s) * g.ci_words + pl * g.ci_plane + u * g.ci_pitch, g.ci_pitch, tv, MCT_SH6(cw_), v[s]);
    } else {
      const int fill = s < nl ? (1 << 13) : 0;
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int c = 0; c < 8; c++) v[s][i][c] = fill;
    }
  }
  const Mc8Weight w = ti.w[1 + pl];
  uint8_t* dst = (pl ? cr : cb) + ti.dst_c + (size_t)y0 * pitch;
  const int nr = ch - y0 < 2 ? 1 : 2;
  if (MCT_PLAIN(shape)) {
#pragma unroll
    for (int i = 0; i < 2; i++)
      if (i < nr) mct_store_row(dst + (size_t)i * pitch, mct_plain4(&v[0][i][0], &v[1][i][0], w.rnd, w.shift), mct_plain4(&v[0][i][4], &v[1][i][4], w.rnd, w.shift), cwd);
  } else {
#pragma unroll
    for (int i = 0; i < 2; i++)
      if (i < nr) mct_store_row(dst + (size_t)i * pitch, mct_weight4(&v[0][i][0], &v[1][i][0], w), mct_weight4(&v[0][i][4], &v[1][i][4], w), cwd);
  }
}

// ---- tile decode (producer side): fills the tile's info and returns the window geometry of list slot s ----
struct MctBox {
  int active;      // this (tile, slot) fetches windows
  int slot;        // DPB slot of the reference
  int lx, ly;      // luma box origin in picture coordinates (16-byte aligned x)
  int cx, cy;      // chroma box origin
};
MCT_HD MctBox mct_decode_tile(uint32_t word, int s, const b200_pu* pus, const b200_weight_entry* wts, uint32_t valid_slots, const DevPic& pic, MctTile* ti)
{
  MctBox bx;
  bx.active = 0; bx.slot = -1; bx.lx = bx.ly = bx.cx = bx.cy = 0;
  if (word == MCT_INVALID) {
    if (s == 0) ti->shape = 0;
    return bx;
  }
  const b200_pu pu = pus[word & 0xFFFFF];
  const int tx = (word >> 20) & 3, ty = (word >> 22) & 3;
  const int x0 = pu.x + 16 * tx, y0 = pu.y + 16 * ty;
  const int tw = pu.w - 16 * tx < 16 ? pu.w - 16 * tx : 16, th = pu.h - 16 * ty < 16 ? pu.h - 16 * ty : 16;
  const bool use0 = pu.flags & B200_PU_PRED_L0, use1 = pu.flags & B200_PU_PRED_L1;
  const int nl = (use0 && use1) ? 2 : 1;
  const int first = use0 ? 0 : 1;
  if (s == 0) {
    const bool wgt_ = pu.flags & B200_PU_WEIGHTED;
    ti->shape = (uint32_t)tw | ((uint32_t)th << 8) | ((uint32_t)nl << 16) | ((use0 || use1) ? 1u << 24 : 0u) | (wgt_ ? 0u : 1u << 25);
    ti->dst_y = y0 * pic.pitch[0] + x0;
    ti->dst_c = (y0 >> 1) * pic.pitch[1] + (x0 >> 1);
    const bool wgt = pu.flags & B200_PU_WEIGHTED;
    const b200_weight_entry* we = wts + (wgt ? pu.wt_idx : 0);
#pragma unroll
    for (int c = 0; c < 3; c++) ti->w[c] = mc8_weight(nl == 2, wgt, first, we, c);
  }
  if (s >= nl || !(use0 || use1)) return bx;
  const int l = s == 0 ? first : 1;
  const int slot = pu.ref_slot[l];
  const bool missing = slot < 0 || !((valid_slots >> slot) & 1);
  const int mvx = pu.mv[l][0], mvy = pu.mv[l][1];
  const int xf = mvx & 3, yf = mvy & 3, cxf = mvx & 7, cyf = mvy & 7;
  const uint32_t hidx = (xf == 0 && yf == 0) ? 4 : xf;      // full-sample position: gain 64 (<< 6) in pass 1, identity in pass 2
  const uint32_t chidx = (cxf == 0 && cyf == 0) ? 8 : cxf;
  // window origin = first sample the 8-tap (4-tap) filters touch, moved to the border's rim when further out (see dpb.cuh)
  const int wx = mct_clip3(-B200_PAD_X, pic.w + B200_PAD_X - 23, x0 + (mvx >> 2) - 3);
  const int wy = mct_clip3(-B200_PAD_Y, pic.h + B200_PAD_Y - 23, y0 + (mvy >> 2) - 3);
  const int cwx = mct_clip3(-B200_PAD_CX, pic.cw + B200_PAD_CX - 11, (x0 >> 1) + (mvx >> 3) - 1);
  const int cwy = mct_clip3(-B200_PAD_CY, pic.ch + B200_PAD_CY - 11, (y0 >> 1) + (mvy >> 3) - 1);
  ti->l[s] = (uint32_t)(wx & 15) | (hidx << 8) | ((uint32_t)yf << 16) | ((xf && yf) ? 6u << 24 : 0u) | (missing ? 0x80000000u : 0u);
  ti->c[s] = (uint32_t)(cwx & 15) | (chidx << 8) | ((uint32_t)cyf << 16) | ((cxf && cyf) ? 6u << 24 : 0u) | (missing ? 0x80000000u : 0u);
  bx.active = !missing;
  bx.slot = slot;
  bx.lx = wx & ~15; bx.ly = wy;
  bx.cx = cwx & ~15; bx.cy = cwy;
  return bx;
}

#ifdef __CUDACC__
// ---- device-only part: tensor maps, mbarrier, the kernel ----
#include <cuda.h>

#define MCT_MAX_REFS 16
struct MctMaps {
  CUtensorMap luma[2][MCT_MAX_REFS];    // [0] big box 48 x 26, [1] small box 32 x 18; 2-D tensor {pitch bytes, padded rows}
  CUtensorMap chroma[2][MCT_MAX_REFS];  // [0] 32 x 14 x 2, [1] 32 x 10 x 2; 3-D tensor {pitch bytes, padded rows, 2 planes}
  int8_t index_of_slot[B200_MAX_SLOTS];
  uint32_t valid_slots;
};

__device__ __forceinline__ uint32_t mct_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Warp roles: the first MCT_THREADS / 32 warps compute; the last warp is the PRODUCER: it decodes the next batch's tiles (two dependent
// global loads per tile: tile word -> PU record) while the compute warps work, waits until pass 1 has consumed the current windows
// (`empty` mbarrier), publishes the tile info and issues the TMA boxes (`full` mbarrier: 32 arrivals + the boxes' bytes).
#define MCT_CTA_THREADS (MCT_THREADS + 32)
__device__ __forceinline__ void mct_mbar_wait(uint32_t bar, uint32_t parity)
{
  uint32_t done;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}

__global__ void __launch_bounds__(MCT_CTA_THREADS) k_inter_pred_tma(DevPic pic, const __grid_constant__ MctMaps maps, const b200_pu* __restrict__ pus,
                                                                    const b200_weight_entry* __restrict__ wts, const uint32_t* __restrict__ tiles,
                                                                    const uint32_t* __restrict__ batches, int n_batches)
{
  extern __shared__ __align__(128) uint8_t mct_smem_raw[];
  MctShared& sm = *reinterpret_cast<MctShared*>(mct_smem_raw);
  const int tid = threadIdx.x;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&c_mc8);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.tab);
    for (int i = tid; i < (int)(sizeof(Mc8Tables) / 4); i += MCT_CTA_THREADS) dst[i] = src[i];
  }
  // full[b]: the windows + tile info of the batches with (it & 1) == b; empty: one arrival per batch when its windows (MCT_DB == 1:
  // after pass 1) resp. its windows AND tile info (MCT_DB == 2: after pass 2) are free
  // (one barrier per batch parity: a parity wait must never see its barrier two phases ahead)
  const uint32_t full0 = mct_smem(&sm.bar[0]), full1 = mct_smem(&sm.bar[1]), empty0 = mct_smem(&sm.bar_empty[0]), empty1 = mct_smem(&sm.bar_empty[1]);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(full0), "r"(MCT_MAX_TL));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(full1), "r"(MCT_MAX_TL));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(empty0), "r"(1));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(empty1), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const bool has_chroma = pic.chroma != 0;

  if (tid >= MCT_THREADS) {
    // ================= producer warp: lane = tile-list item =================
    const int lane = tid - MCT_THREADS;
    int it = 0;
    for (int batch = blockIdx.x; batch < n_batches; batch += gridDim.x, it++) {
      const uint32_t bw = batches[batch];
      const MctGeom g = mct_geom((bw >> 28) & 7);
      MctTile mine;  // decoded into registers / local memory first: the shared buffers may still be in use
      MctBox bx;
      bx.active = 0;
      const int tile = g.nl == 2 ? (lane >> 1) : lane, s = g.nl == 2 ? (lane & 1) : 0;
      if (lane < g.ntl) bx = mct_decode_tile(tiles[(bw & 0x0FFFFFFF) + tile], s, pus, wts, maps.valid_slots, pic, &mine);
      const int mi = bx.active ? maps.index_of_slot[bx.slot] : -1;
      const uint32_t full = (it & 1) ? full1 : full0;
      uint8_t* win = sm.win[MCT_DB == 2 ? (it & 1) : 0];
      // MCT_DB == 1: the windows (and info[it & 1], last read in pass 2 of batch it-2) are free once pass 1 of batch it-1 is done;
      // MCT_DB == 2: window buffer and info of parity it & 1 are free once pass 2 of batch it-2 is done — a whole batch of lookahead
      if (MCT_DB == 2) { if (it > 1) mct_mbar_wait((it & 1) ? empty1 : empty0, ((it >> 1) - 1) & 1); }  // batch it-2 = previous use of this parity
      else if (it > 0) mct_mbar_wait(((it - 1) & 1) ? empty1 : empty0, ((it - 1) >> 1) & 1);
      MctTile* dst = &sm.info[it & 1][tile];
      if (lane < g.ntl) {
        if (s == 0) {  // slot-0 lane owns the common fields; with two lists the slot-1 lane adds its own
          dst->dst_y = mine.dst_y; dst->dst_c = mine.dst_c; dst->shape = mine.shape;
#pragma unroll
          for (int c = 0; c < 3; c++) dst->w[c] = mine.w[c];
        }
        dst->l[s] = mine.l[s];
        dst->c[s] = mine.c[s];
      }
      if (lane == 0) sm.geom[it & 1] = g;
      if (mi >= 0) {
        const int skew = lane & 3, k = g.small;
        const uint32_t bytes = (k ? MCT_LWS_PITCH * MCT_LWS_ROWS : MCT_LWB_PITCH * MCT_LWB_ROWS) +
                               (has_chroma ? (k ? 2 * MCT_CWS_PITCH * MCT_CWS_ROWS : 2 * MCT_CWB_PITCH * MCT_CWB_ROWS) : 0);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the windows were read through the generic proxy in pass 1
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                         mct_smem(win + lane * g.lw_slot)),
                     "l"(&maps.luma[k][mi]), "r"(bx.lx + B200_PAD_X), "r"(bx.ly + B200_PAD_Y - skew), "r"(full)
                     : "memory");
        if (has_chroma)
          asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                           mct_smem(win + g.cw_off + lane * g.cw_slot)),
                       "l"(&maps.chroma[k][mi]), "r"(bx.cx + B200_PAD_CX), "r"(bx.cy + B200_PAD_CY - skew), "r"(0), "r"(full)
                       : "memory");
      } else if (lane < MCT_MAX_TL) {
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(full) : "memory");
      }
    }
    return;
  }

  // ================= compute warps =================
  int it = 0;
  for (int batch = blockIdx.x; batch < n_batches; batch += gridDim.x, it++) {
    mct_mbar_wait((it & 1) ? full1 : full0, (it >> 1) & 1);  // this batch's windows and tile info
    const uint8_t* win = sm.win[MCT_DB == 2 ? (it & 1) : 0];
    const MctTile* info = sm.info[it & 1];
    const MctGeom g = sm.geom[it & 1];
    const int n1 = g.n1l + (has_chroma ? g.n1c : 0), n2 = g.n2l + (has_chroma ? g.n2c : 0);
    for (int t = tid; t < n1; t += MCT_THREADS) {  // one flat list: luma tasks, then chroma tasks
      if (t < g.n1l) mct_pass1_luma(t, g, info, win, sm.interm, sm.tab);
      else mct_pass1_chroma(t - g.n1l, g, info, win, sm.interm, sm.tab);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(MCT_THREADS) : "memory");
    if (MCT_DB == 1 && tid == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((it & 1) ? empty1 : empty0) : "memory");  // the windows are free: the producer fetches ahead
    for (int t = tid; t < n2; t += MCT_THREADS) {
      if (t < g.n2l) mct_pass2_luma(t, g, info, sm.interm, sm.tab, pic.cur[0], pic.pitch[0]);
      else mct_pass2_chroma(t - g.n2l, g, info, sm.interm, sm.tab, pic.cur[1], pic.cur[2], pic.pitch[1]);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(MCT_THREADS) : "memory");
    if (MCT_DB == 2 && tid == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((it & 1) ? empty1 : empty0) : "memory");  // buffer + info of this parity are free
  }
}
#endif  // __CUDACC__
