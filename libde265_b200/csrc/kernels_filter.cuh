// kernels_filter.cuh — in-loop filters for one picture.
//
// k_deblock<P, VERT>: one thread per 4-line edge segment (luma on the 8x8 grid, Cb and Cr on the
//   chroma 8x8 grid), decisions + filtering fused.  Replaces edge_filtering_luma_internal
//   (deblock.cc:412-605), edge_filtering_chroma_internal (:635-761) and the deblock_luma/chroma
//   kernels (fallback-deblk.h:32-124).  Launched twice per picture: all vertical edges, then all
//   horizontal edges (deblock.cc:908-946).  Edge flags / boundary strengths arrive in bs_map.
// k_sao<P>: one thread per sample, reads the deblocked surface, writes the DPB surface (out-of-place
//   exactly like sao.cc:327-382), copying samples that SAO leaves untouched.  Replaces apply_sao_internal
//   (sao.cc:28-263).
#pragma once
#include <type_traits>

#include "dev_common.cuh"

struct FilterArgs {
  const uint8_t* bs_map;
  const int8_t* qp_map;
  const uint8_t* nofilt_map;
  const b200_slice_info* slices;
  const b200_ctb_info* ctbs;
  const uint16_t* sao_avail;  // k_sao_prep output: [luma CTBs | chroma CTBs]
};

__constant__ uint8_t k_tab_beta[52] = {0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  6,  7,
                                       8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 22, 24, 26, 28, 30, 32,
                                       34, 36, 38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64};
__constant__ uint8_t k_tab_tc[54] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,  0,  0,  1,  1,  1,  1,  1,  1,  1,  1,  1,
                                     2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8,  9,  10, 11, 13, 14, 16, 18, 20, 22, 24};
__constant__ uint8_t k_tab_qpc[13] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37};

__device__ __forceinline__ int qpy_at(const DevPic& pic, const FilterArgs& a, int x, int y) { return a.qp_map[(x >> 3) + (y >> 3) * pic.w8]; }
__device__ __forceinline__ int nofilt_at(const DevPic& pic, const FilterArgs& a, int x, int y) { return a.nofilt_map[(x >> 3) + (y >> 3) * pic.w8] & 1; }
__device__ __forceinline__ const b200_slice_info& slice_at(const DevPic& pic, const FilterArgs& a, int x, int y)
{
  return a.slices[a.ctbs[(x >> pic.log2ctb) + (y >> pic.log2ctb) * pic.wctb].slice_idx];
}

template <typename P, bool VERT>
__global__ void __launch_bounds__(128) k_deblock(DevPic pic, FilterArgs a)
{
  // blockIdx.y: 0 luma, 1 chroma (both Cb and Cr per thread)
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {
    // luma segments: VERT: x even (8-px grid), every y;  HORZ: every x, y even   [units of 4 samples]
    const int nx = VERT ? (pic.w4 + 1) / 2 : pic.w4;
    const int ny = VERT ? pic.h4 : (pic.h4 + 1) / 2;
    if (id >= nx * ny) return;
    const int ux = VERT ? (id % nx) * 2 : id % nx, uy = VERT ? id / nx : (id / nx) * 2;
    const int b = a.bs_map[ux + uy * pic.w4];
    const int bS = VERT ? B200_BS_V(b) : B200_BS_H(b);
    if (bS == 0) return;
    const int xd = ux << 2, yd = uy << 2;
    const int pitch = pic.pitch[0];
    const ptrdiff_t sa = VERT ? 1 : pitch / (int)sizeof(P), sb = VERT ? pitch / (int)sizeof(P) : 1;  // across / along the edge, in samples
    P* ptr = row_ptr<P>(pic.cur[0], pitch, yd) + xd;
    const int bd = pic.bd_y;
    int p[4][4], q[4][4];
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
      for (int i = 0; i < 4; i++) {
        q[k][i] = ptr[k * sb + i * sa];
        p[k][i] = ptr[k * sb - (i + 1) * sa];
      }
    const int qp_q = qpy_at(pic, a, xd, yd);
    const int qp_p = VERT ? qpy_at(pic, a, xd - 1, yd) : qpy_at(pic, a, xd, yd - 1);
    const int qpl = (qp_q + qp_p + 1) >> 1;
    const b200_slice_info sl = slice_at(pic, a, xd, yd);
    const int beta = k_tab_beta[clip3i(0, 51, qpl + sl.beta_offset)] * (1 << (bd - 8));
    const int tc = k_tab_tc[clip3i(0, 53, qpl + 2 * (bS - 1) + sl.tc_offset)] * (1 << (bd - 8));
    const int dp0 = abs(p[0][2] - 2 * p[0][1] + p[0][0]), dp3 = abs(p[3][2] - 2 * p[3][1] + p[3][0]);
    const int dq0 = abs(q[0][2] - 2 * q[0][1] + q[0][0]), dq3 = abs(q[3][2] - 2 * q[3][1] + q[3][0]);
    const int dpq0 = dp0 + dq0, dpq3 = dp3 + dq3, dp = dp0 + dp3, dq = dq0 + dq3, d = dpq0 + dpq3;
    if (d >= beta) return;
    const bool s0 = 2 * dpq0 < (beta >> 2) && abs(p[0][3] - p[0][0]) + abs(q[0][0] - q[0][3]) < (beta >> 3) && abs(p[0][0] - q[0][0]) < ((5 * tc + 1) >> 1);
    const bool s3 = 2 * dpq3 < (beta >> 2) && abs(p[3][3] - p[3][0]) + abs(q[3][0] - q[3][3]) < (beta >> 3) && abs(p[3][0] - q[3][0]) < ((5 * tc + 1) >> 1);
    const bool strong = s0 && s3;
    const bool dEp = dp < ((beta + (beta >> 1)) >> 3), dEq = dq < ((beta + (beta >> 1)) >> 3);
    const bool fP = !(VERT ? nofilt_at(pic, a, xd - 1, yd) : nofilt_at(pic, a, xd, yd - 1));
    const bool fQ = !nofilt_at(pic, a, xd, yd);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int p0 = p[k][0], p1 = p[k][1], p2 = p[k][2], p3 = p[k][3], q0 = q[k][0], q1 = q[k][1], q2 = q[k][2], q3 = q[k][3];
      P* c = ptr + k * sb;
      if (strong) {
        if (fP) {
          c[-sa] = (P)clip3i(p0 - 2 * tc, p0 + 2 * tc, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
          c[-2 * sa] = (P)clip3i(p1 - 2 * tc, p1 + 2 * tc, (p2 + p1 + p0 + q0 + 2) >> 2);
          c[-3 * sa] = (P)clip3i(p2 - 2 * tc, p2 + 2 * tc, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
        }
        if (fQ) {
          c[0] = (P)clip3i(q0 - 2 * tc, q0 + 2 * tc, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
          c[sa] = (P)clip3i(q1 - 2 * tc, q1 + 2 * tc, (p0 + q0 + q1 + q2 + 2) >> 2);
          c[2 * sa] = (P)clip3i(q2 - 2 * tc, q2 + 2 * tc, (p0 + q0 + q1 + 3 * q2 + 2 * q3 + 4) >> 3);
        }
      } else {
        int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
        if (abs(delta) < tc * 10) {
          delta = clip3i(-tc, tc, delta);
          if (fP) c[-sa] = (P)clip_bd(p0 + delta, bd);
          if (fQ) c[0] = (P)clip_bd(q0 - delta, bd);
          if (dEp && fP) c[-2 * sa] = (P)clip_bd(p1 + clip3i(-(tc >> 1), tc >> 1, (((p2 + p0 + 1) >> 1) - p1 + delta) >> 1), bd);
          if (dEq && fQ) c[sa] = (P)clip_bd(q1 + clip3i(-(tc >> 1), tc >> 1, (((q2 + q0 + 1) >> 1) - q1 - delta) >> 1), bd);
        }
      }
    }
  } else {
    if (!pic.chroma) return;
    // chroma (4:2:0): edges on the chroma 8x8 grid = every 16 luma samples across, 4 chroma lines = 8 luma lines along
    // [units of 4 luma samples]: VERT: x step 4, y step 2;  HORZ: x step 2, y step 4   (deblock.cc:650-663)
    const int xs = VERT ? 4 : 2, ys = VERT ? 2 : 4;
    const int nx = (pic.w4 + xs - 1) / xs, ny = (pic.h4 + ys - 1) / ys;
    if (id >= nx * ny) return;
    const int ux = (id % nx) * xs, uy = (id / nx) * ys;
    const int b = a.bs_map[ux + uy * pic.w4];
    const int bS = VERT ? B200_BS_V(b) : B200_BS_H(b);
    if (bS < 2) return;
    const int xl = ux << 2, yl = uy << 2, xd = xl >> 1, yd = yl >> 1;
    const int qp_q = qpy_at(pic, a, xl, yl);
    const int qp_p = VERT ? qpy_at(pic, a, xl - 1, yl) : qpy_at(pic, a, xl, yl - 1);
    const b200_slice_info sl = slice_at(pic, a, xl, yl);
    const bool fP = !(VERT ? nofilt_at(pic, a, xl - 1, yl) : nofilt_at(pic, a, xl, yl - 1));
    const bool fQ = !nofilt_at(pic, a, xl, yl);
    const int bd = pic.bd_c;
#pragma unroll
    for (int c = 1; c <= 2; c++) {
      const int qpi = ((qp_q + qp_p + 1) >> 1) + (c == 1 ? pic.cb_qp_off : pic.cr_qp_off);
      const int qpc = (qpi < 30) ? qpi : (qpi >= 43) ? qpi - 6 : k_tab_qpc[qpi - 30];  // table8_22, transform.h:29-34
      const int tc = k_tab_tc[clip3i(0, 53, qpc + 2 * (bS - 1) + sl.tc_offset)] * (1 << (bd - 8));
      const int pitch = pic.pitch[c];
      const ptrdiff_t sa = VERT ? 1 : pitch / (int)sizeof(P), sb = VERT ? pitch / (int)sizeof(P) : 1;
      P* ptr = row_ptr<P>(pic.cur[c], pitch, yd) + xd;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        P* e = ptr + k * sb;
        const int p0 = e[-sa], p1 = e[-2 * sa], q0 = e[0], q1 = e[sa];
        const int delta = clip3i(-tc, tc, ((((q0 - p0) * 4) + p1 - q1 + 4) >> 3));
        if (fP) e[-sa] = (P)clip_bd(p0 + delta, bd);
        if (fQ) e[0] = (P)clip_bd(q0 - delta, bd);
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------
// One SAO sample (sao.cc:103-262).  xC/yC = CTB origin in this plane, i/j = position inside the CTB.
template <typename P>
__device__ __forceinline__ int sao_sample(const DevPic& pic, const FilterArgs& a, const b200_ctb_info& ci, int c, int sh, int x, int y, int v,
                                          int width, int height, int type, int ctbshift)
{
  const int bd = c ? pic.bd_c : pic.bd_y, maxv = (1 << bd) - 1;
  if (nofilt_at(pic, a, x << sh, y << sh)) return v;
  if (type == 2) {
    const int cls = (ci.sao_eo_class >> (2 * c)) & 3;
    const int hx0 = (cls == 1) ? 0 : (cls == 3) ? 1 : -1, hx1 = -hx0;
    const int vy0 = (cls == 0) ? 0 : -1, vy1 = -vy0;
    const int S = 1 << ctbshift;
    const int xC = (x >> ctbshift) << ctbshift, yC = (y >> ctbshift) << ctbshift;
    const int ctbW = min(S, width - xC), ctbH = min(S, height - yC);
    const int i = x - xC, j = y - yC;
    if (i == 0 || j == 0 || i == ctbW - 1 || j == ctbH - 1) {
      // sao.cc:49: slice address of the CTB looked up with COMPONENT coordinates (reference quirk, kept)
      const int ctb_addr = (int)slice_at(pic, a, min(xC, pic.w - 1), min(yC, pic.h - 1)).slice_addr_rs;
      const b200_slice_info& sc = slice_at(pic, a, x << sh, y << sh);
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int xS = x + (k ? hx1 : hx0), yS = y + (k ? vy1 : vy0);
        if (xS < 0 || yS < 0 || xS >= width || yS >= height) return v;
        const b200_ctb_info& cn = a.ctbs[((xS << sh) >> pic.log2ctb) + ((yS << sh) >> pic.log2ctb) * pic.wctb];
        const b200_slice_info& sn = a.slices[cn.slice_idx];
        if ((int)sn.slice_addr_rs < ctb_addr && !(sc.flags & B200_SLICE_LF_ACROSS_SLICES)) return v;
        if ((int)sn.slice_addr_rs > ctb_addr && !(sn.flags & B200_SLICE_LF_ACROSS_SLICES)) return v;
        if (!(pic.flags & B200_PIC_LF_ACROSS_TILES) && cn.tile_id != ci.tile_id) return v;
      }
    }
    const int na = row_ptr<P>(pic.cur[c], pic.pitch[c], y + vy0)[x + hx0];
    const int nb = row_ptr<P>(pic.cur[c], pic.pitch[c], y + vy1)[x + hx1];
    const int e = ((v > na) - (v < na)) + ((v > nb) - (v < nb));
    const int off = (e == 0) ? 0 : ci.sao_offset[c][e < 0 ? e + 2 : e + 1];  // [-2,-1,1,2] -> offsets 0,1,2,3 (sao.cc:95-100)
    return clip3i(0, maxv, v + off);
  }
  const int band = clip3i(0, maxv, v) >> (bd - 5);
  const int k = (band - ci.sao_band_pos[c]) & 31;
  return (k < 4) ? clip3i(0, maxv, v + ci.sao_offset[c][k]) : v;
}

// Per CTB and plane kind (0 luma, 1 chroma): which of the 8 neighbouring CTBs SAO edge classification may read
// (sao.cc:125-190: picture bounds, slice order + slice_loop_filter_across_slices, tiles).  Bit (dy+1)*3 + (dx+1).
// The "current" slice address is looked up with the CTB origin in COMPONENT coordinates (sao.cc:49, kept).
__global__ void k_sao_prep(DevPic pic, FilterArgs a, uint16_t* __restrict__ avail)
{
  const int n_ctb = pic.wctb * pic.hctb;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n_ctb) return;
  const int kind = t / n_ctb, ctb = t - kind * n_ctb;
  const int cx = ctb % pic.wctb, cy = ctb / pic.wctb;
  const b200_ctb_info& ci = a.ctbs[ctb];
  const b200_slice_info& sc = a.slices[ci.slice_idx];
  const int xC = (cx << pic.log2ctb) >> kind, yC = (cy << pic.log2ctb) >> kind;  // component coordinates
  const int ctb_addr = (int)slice_at(pic, a, min(xC, pic.w - 1), min(yC, pic.h - 1)).slice_addr_rs;
  // the centre bit follows the same rule: with the component-coordinate lookup the "current" slice address may differ from
  // the CTB's own, and the reference applies the test to both neighbours of every sample on the CTB border
  unsigned m = 0;
  for (int dy = -1; dy <= 1; dy++)
    for (int dx = -1; dx <= 1; dx++) {
      const int nx = cx + dx, ny = cy + dy;
      if (nx < 0 || ny < 0 || nx >= pic.wctb || ny >= pic.hctb) continue;
      const b200_ctb_info& cn = a.ctbs[nx + ny * pic.wctb];
      const b200_slice_info& sn = a.slices[cn.slice_idx];
      if ((int)sn.slice_addr_rs < ctb_addr && !(sc.flags & B200_SLICE_LF_ACROSS_SLICES)) continue;
      if ((int)sn.slice_addr_rs > ctb_addr && !(sn.flags & B200_SLICE_LF_ACROSS_SLICES)) continue;
      if (!(pic.flags & B200_PIC_LF_ACROSS_TILES) && cn.tile_id != ci.tile_id) continue;
      m |= 1u << ((dy + 1) * 3 + dx + 1);
    }
  avail[t] = (uint16_t)m;
}

// One thread per 8 horizontally adjacent samples (8 never straddles a CTB: CTB widths are multiples of 8 in
// every plane).  SAO-off groups move as one 8/16-byte vector.  Edge-offset groups read their two neighbour rows as
// one vector + one scalar each and classify all 8 samples in registers, using the CTB's neighbour-availability
// mask from k_sao_prep for samples whose neighbours lie in another CTB; only groups touching a no-filter block
// (pcm / transquant bypass) take the per-sample path.
template <typename P>
__global__ void __launch_bounds__(128) k_sao(DevPic pic, FilterArgs a)
{
  const int c = blockIdx.z;  // colour plane
  const int sh = c ? 1 : 0;
  const int width = c ? pic.cw : pic.w, height = c ? pic.ch : pic.h;
  const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 8, y = blockIdx.y;
  if (x >= width || y >= height) return;
  const int pitch = pic.pitch[c];
  const P* in = row_ptr<P>(pic.cur[c], pitch, y) + x;
  P* out = row_ptr<P>(pic.out[c], pitch, y) + x;
  const int ctbshift = pic.log2ctb - sh;
  const int ctb = (x >> ctbshift) + (y >> ctbshift) * pic.wctb;
  // the 24-byte CTB record as three 64-bit words (fields extracted with shifts: no dynamically indexed local copy)
  const unsigned long long* cw = reinterpret_cast<const unsigned long long*>(a.ctbs + ctb);
  const unsigned long long w0 = cw[0], w1 = cw[1], w2 = cw[2];
  const b200_slice_info& sl = a.slices[w0 & 0xFFFF];
  const bool on = c ? (sl.flags & B200_SLICE_SAO_CHROMA) : (sl.flags & B200_SLICE_SAO_LUMA);
  const int type = on ? (int)(w0 >> (32 + 2 * c)) & 3 : 0;
  const int n = min(8, width - x);  // picture widths are multiples of 4 in every plane (8 luma)
  typedef typename std::conditional<sizeof(P) == 1, uint2, uint4>::type V8;  // 8 samples
  union Vec { V8 q; P s[8]; };
  Vec v, r;
  v.q = *reinterpret_cast<const V8*>(in);  // the row pitch leaves >= 16 bytes after the last sample
  auto store = [&](const Vec& t) {  // n is 8, or 4 at the right edge of a plane whose width is 4 mod 8
    if (n == 8) *reinterpret_cast<V8*>(out) = t.q;
    else if (sizeof(P) == 1) *reinterpret_cast<uint32_t*>(out) = *reinterpret_cast<const uint32_t*>(&t.q);
    else *reinterpret_cast<uint2*>(out) = *reinterpret_cast<const uint2*>(&t.q);
  };
  if (type == 0) {
    store(v);
    return;
  }
  const int bd = c ? pic.bd_c : pic.bd_y, maxv = (1 << bd) - 1;
  // no-filter flags of the 8x8 luma blocks under this group (1 block for luma, 2 for chroma)
  const uint8_t* nfp = a.nofilt_map + ((x << sh) >> 3) + ((y << sh) >> 3) * pic.w8;
  const bool nf = (nfp[0] & 1) || (sh && ((x << sh) >> 3) + 1 < pic.w8 && (nfp[1] & 1));
  const unsigned o4 = (c == 0) ? (unsigned)(w1 >> 8) : (c == 1) ? ((unsigned)(w1 >> 40) | ((unsigned)w2 << 24)) : (unsigned)(w2 >> 8);
  if (nf) {
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k < n) out[k] = (P)sao_sample<P>(pic, a, a.ctbs[ctb], c, sh, x + k, y, v.s[k], width, height, type, ctbshift);
    return;
  }
  // Offsets as bytes [o0, o1, 0, o2, o3]: an edge sample indexes it with e + 2 (sao.cc:95-100), a band sample with its
  // band number mapped 0,1,2,3 -> 0,1,3,4; index 2 = no offset.  One byte permute with sign replication does the lookup,
  // so edge and band CTBs (and all four edge classes) share one instruction stream: no divergence inside a warp.
  const unsigned tlo = (o4 & 0xFFFFu) | ((o4 & 0xFF0000u) << 8), thi = o4 >> 24;
  const bool edge = type == 2;
  unsigned bad = 0;  // edge: samples whose neighbours are not available
  int na_[8], nb_[8];
  if (edge) {
    const int S = 1 << ctbshift;
    const int xC = (x >> ctbshift) << ctbshift, yC = (y >> ctbshift) << ctbshift;
    const int ctbW = min(S, width - xC), ctbH = min(S, height - yC);
    const int i = x - xC, j = y - yC;
    const int cls = (int)(w0 >> (40 + 2 * c)) & 3;
    const int hx0 = (cls == 1) ? 0 : (cls == 3) ? 1 : -1;
    const int vy0 = (cls == 0) ? 0 : -1;
    // neighbour a = (x+hx0, y+vy0), neighbour b = (x-hx0, y-vy0)
    const unsigned m = a.sao_avail[(c ? pic.wctb * pic.hctb : 0) + ctb];
    const int dya = (j + vy0 < 0) ? -1 : 0, dyb = (j - vy0 >= ctbH) ? 1 : 0;  // vy0 <= 0
    // availability of a / b in the CTB column of the sample itself, and in the column one step in a's / b's x direction
    const unsigned a_mid = (m >> ((dya + 1) * 3 + 1)) & 1, b_mid = (m >> ((dyb + 1) * 3 + 1)) & 1;
    const unsigned a_side = (m >> ((dya + 1) * 3 + 1 + hx0)) & 1, b_side = (m >> ((dyb + 1) * 3 + 1 - hx0)) & 1;
    const unsigned first = (i == 0) ? 1u : 0u, last = (i + 8 >= ctbW) ? 1u << (ctbW - 1 - i) : 0u;  // CTB border columns in this group
    unsigned ma = a_mid ? 0xFFu : 0u, mb = b_mid ? 0xFFu : 0u;
    const unsigned sa = (hx0 < 0) ? first : (hx0 > 0) ? last : 0u, sb = (hx0 > 0) ? first : (hx0 < 0) ? last : 0u;  // sample whose a / b is in the side CTB
    ma = (ma & ~sa) | (a_side ? sa : 0u);
    mb = (mb & ~sb) | (b_side ? sb : 0u);
    const unsigned border = (j == 0 || j == ctbH - 1) ? 0xFFu : (first | last);  // sao.cc:125: tests only on the CTB border
    bad = border & ~(ma & mb);
    const int ya = max(y + vy0, 0), yb = min(y - vy0, height - 1);  // clamped rows are only read when unavailable
    const P* ra = row_ptr<P>(pic.cur[c], pitch, ya) + x;
    const P* rb = row_ptr<P>(pic.cur[c], pitch, yb) + x;
    Vec va, vb;
    va.q = *reinterpret_cast<const V8*>(ra);
    vb.q = *reinterpret_cast<const V8*>(rb);
    // samples x-1 and x+8 of both rows (never read before the first sample of a row)
    const int la = x ? ra[-1] : 0, lb = x ? rb[-1] : 0, ha = ra[8], hb = rb[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int am = k ? va.s[k - 1] : la, ap = (k < 7) ? va.s[k + 1] : ha;
      const int bm = k ? vb.s[k - 1] : lb, bp = (k < 7) ? vb.s[k + 1] : hb;
      na_[k] = (hx0 < 0) ? am : (hx0 > 0) ? ap : (int)va.s[k];
      nb_[k] = (hx0 < 0) ? bp : (hx0 > 0) ? bm : (int)vb.s[k];
    }
  }
  const int pos = (c == 0) ? (int)(w0 >> 48) & 0xFF : (c == 1) ? (int)(w0 >> 56) : (int)(w1 & 0xFF);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int s = v.s[k];
    int idx;
    if (edge) {
      const int e = clip3i(-1, 1, s - na_[k]) + clip3i(-1, 1, s - nb_[k]);
      idx = ((bad >> k) & 1) ? 2 : e + 2;
    } else {
      const int b = ((s >> (bd - 5)) - pos) & 31;
      idx = (b > 3) ? 2 : b + (b >> 1);
    }
    int off;  // byte idx of {thi:tlo}, sign-extended (selector nibble bit 3 = replicate the byte's sign)
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(off) : "r"(tlo), "r"(thi), "r"((unsigned)idx * 0x1111u + 0x8880u));
    r.s[k] = (P)clip3i(0, maxv, s + off);
  }
  store(r);
}

// -------------------------------------------------------------------------------------------------
// k_sao8: SAO for 8-bit samples with byte-parallel arithmetic (CTB sizes 32 and 64; other cases run k_sao).
// k_sao spends ~70 instructions per sample (one sample per step of an unrolled loop: classification, table look-up, clip) and is
// bound by instruction issue, not by its 25 MB of traffic per 4K picture.  Here a lane owns 16 samples x
// SAO8_R rows as 32-bit words and classifies / offsets four samples per instruction:
//   * unsigned byte compare  x < y  =  bit 7 of  (~x & y) | (~(x ^ y) & ~((x | 0x80..) - (y & 0x7f..)))  (no carries between
//     bytes), widened to a byte mask by one PRMT with sign replication;
//   * the five edge categories are mask algebra on (s<a, s>a, s<b, s>b): e = -2 both less, -1 one less + one equal, ... ;
//     offsets are selected as replicated positive / negative parts and applied with byte-wise saturating add / subtract;
//   * band offsets: (s >> 3) - band_position per byte, compared with 0..3 by a zero-byte test.
// A WARP covers one CTB of one plane (64 bytes x 8 rows x SAO8_R for a 64x64 luma CTB): type, class, offsets and the neighbour
// availability mask are warp-uniform — no divergence between edge / band / off CTBs, the CTB record is one broadcast load.
// The sample left / right of a lane's 16 bytes comes from the neighbour lane (shuffle) or, at the CTB's side, one byte load.
// Same results as k_sao (tests compare both against the oracle).
// -------------------------------------------------------------------------------------------------
#define SAO8_R 2
#define SAO8_WARPS 8

#include "sao8_swar.cuh"

struct Sao8Layout {
  int n_ctb, ipl, ipc;  // items (warps) per luma / chroma CTB
};

__global__ void __launch_bounds__(SAO8_WARPS * 32, 4) k_sao8(DevPic pic, FilterArgs a, Sao8Layout lay)
{
  const int lane = threadIdx.x & 31;
  int item = blockIdx.x * SAO8_WARPS + (threadIdx.x >> 5);
  int c, ctb, sub;
  if (item < lay.n_ctb * lay.ipl) {
    c = 0;
    ctb = item / lay.ipl;
    sub = item - ctb * lay.ipl;
  } else {
    item -= lay.n_ctb * lay.ipl;
    if (item >= 2 * lay.n_ctb * lay.ipc) return;
    c = 1 + item / (lay.n_ctb * lay.ipc);
    item -= (c - 1) * lay.n_ctb * lay.ipc;
    ctb = item / lay.ipc;
    sub = item - ctb * lay.ipc;
  }
  const int sh = c ? 1 : 0;
  const int width = c ? pic.cw : pic.w, height = c ? pic.ch : pic.h;
  const int ctbshift = pic.log2ctb - sh, S = 1 << ctbshift;
  const int segs = S >> 4, l2segs = ctbshift - 4;  // 16-byte segments per CTB row: 4, 2 or 1
  const int cx = ctb % pic.wctb, cy = ctb / pic.wctb;
  const int xC = cx << ctbshift, yC = cy << ctbshift;
  const int ctbW = min(S, width - xC), ctbH = min(S, height - yC);
  const int seg = lane & (segs - 1), i0 = seg << 4;
  const int j0 = (sub * (32 >> l2segs) + (lane >> l2segs)) * SAO8_R;  // first of this lane's rows inside the CTB
  const bool active = i0 < ctbW && j0 < ctbH;
  const int x = xC + i0;
  const int pitch = pic.pitch[c];
  // the CTB record: warp-uniform
  const unsigned long long* cw = reinterpret_cast<const unsigned long long*>(a.ctbs + ctb);
  const unsigned long long w0 = cw[0], w1 = cw[1], w2 = cw[2];
  const b200_slice_info& sl = a.slices[w0 & 0xFFFF];
  const bool on = c ? (sl.flags & B200_SLICE_SAO_CHROMA) : (sl.flags & B200_SLICE_SAO_LUMA);
  const int type = on ? (int)(w0 >> (32 + 2 * c)) & 3 : 0;
  const int n_valid = min(16, ctbW - i0);  // samples of this segment inside the picture (multiple of 4)
  auto store_row = [&](int y, const uint4& v) {
    uint8_t* out = pic.out[c] + (size_t)y * pitch + x;
    if (n_valid == 16) *reinterpret_cast<uint4*>(out) = v;
    else {
      uint32_t* o = reinterpret_cast<uint32_t*>(out);
      o[0] = v.x;  // n_valid >= 4
      if (n_valid > 4) o[1] = v.y;
      if (n_valid > 8) o[2] = v.z;
    }
  };
  if (type == 0) {
    if (active)
      for (int r = 0; r < SAO8_R; r++)
        if (j0 + r < ctbH) store_row(yC + j0 + r, *reinterpret_cast<const uint4*>(pic.cur[c] + (size_t)(yC + j0 + r) * pitch + x));
    return;
  }
  const unsigned o4 = (c == 0) ? (unsigned)(w1 >> 8) : (c == 1) ? ((unsigned)(w1 >> 40) | ((unsigned)w2 << 24)) : (unsigned)(w2 >> 8);
  uint32_t opos[4], oneg[4];  // the four offsets, positive / negative parts replicated into every byte
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int o = (int)(int8_t)(o4 >> (8 * k));
    opos[k] = (uint32_t)max(o, 0) * 0x01010101u;
    oneg[k] = (uint32_t)max(-o, 0) * 0x01010101u;
  }
  // no-filter (pcm / transquant-bypass) 8x8 luma blocks keep their samples: byte masks per word of every row
  // (luma: word k lies in block k >> 1 of the segment; chroma: word k is block k)
  const bool edge = type == 2;
  const int cls = (int)(w0 >> (40 + 2 * c)) & 3;
  const int hx0 = (cls == 1) ? 0 : (cls == 3) ? 1 : -1;  // neighbour a = (x + hx0, y + vy0), b = (x - hx0, y - vy0)
  const int vy0 = (cls == 0) ? 0 : -1;
  // which of the 8 neighbouring CTBs edge classification may read (k_sao_prep's rule, sao.cc:125-190): lane l < 9 tests the
  // neighbour (l % 3 - 1, l / 3 - 1), one ballot gives the mask — no separate launch in front of this kernel
  unsigned m = 0;
  if (edge) {
    bool ok = false;
    if (lane < 9) {
      const int nx = cx + lane % 3 - 1, ny = cy + lane / 3 - 1;
      if (nx >= 0 && ny >= 0 && nx < pic.wctb && ny < pic.hctb) {
        const int ctb_addr = (int)slice_at(pic, a, min(xC, pic.w - 1), min(yC, pic.h - 1)).slice_addr_rs;  // component coordinates (sao.cc:49)
        const b200_ctb_info& cn = a.ctbs[nx + ny * pic.wctb];
        const b200_slice_info& sn = a.slices[cn.slice_idx];
        ok = !((int)sn.slice_addr_rs < ctb_addr && !(sl.flags & B200_SLICE_LF_ACROSS_SLICES)) &&
             !((int)sn.slice_addr_rs > ctb_addr && !(sn.flags & B200_SLICE_LF_ACROSS_SLICES)) &&
             !(!(pic.flags & B200_PIC_LF_ACROSS_TILES) && cn.tile_id != (uint16_t)(w0 >> 16));
      }
    }
    m = __ballot_sync(0xffffffffu, ok) & 0x1FFu;
  }
  const int pos = (c == 0) ? (int)(w0 >> 48) & 0xFF : (c == 1) ? (int)(w0 >> 56) : (int)(w1 & 0xFF);
  const uint32_t pos4 = (uint32_t)(pos & 31) * 0x01010101u;

  // rows j0-1 .. j0+SAO8_R of the (deblocked) input with the bytes left and right of the segment
  uint32_t row[SAO8_R + 2][4];
  uint32_t lft[SAO8_R + 2], rgt[SAO8_R + 2];
  const bool need_v = edge && vy0 != 0, need_h = edge && hx0 != 0;
#pragma unroll
  for (int r = 0; r < SAO8_R + 2; r++) {
    const bool use = (r >= 1 && r <= SAO8_R) || need_v;
    if (use && active) {
      // rows above / below the picture lie in the surface's border (their samples only reach results that `bad` discards)
      const uint8_t* p = pic.cur[c] + (size_t)(yC + j0 + r - 1) * pitch + x;
      const uint4 v = *reinterpret_cast<const uint4*>(p);
      row[r][0] = v.x; row[r][1] = v.y; row[r][2] = v.z; row[r][3] = v.w;
    } else {
      row[r][0] = row[r][1] = row[r][2] = row[r][3] = 0;
    }
    lft[r] = rgt[r] = 0;
    if (need_h && use) {  // warp-uniform condition: every lane takes part in the shuffles
      const uint32_t from_l = __shfl_up_sync(0xffffffffu, row[r][3], 1), from_r = __shfl_down_sync(0xffffffffu, row[r][0], 1);
      if (active) {
        const uint8_t* p = pic.cur[c] + (size_t)(yC + j0 + r - 1) * pitch + x;
        lft[r] = (seg == 0) ? (uint32_t)p[-1] : from_l >> 24;         // byte x-1 (the border column for x == 0)
        rgt[r] = (seg == segs - 1) ? (uint32_t)p[16] : from_r & 0xFF;  // byte x+16
      }
    }
  }
  if (!active) return;

#pragma unroll
  for (int r = 0; r < SAO8_R; r++) {
    const int j = j0 + r, y = yC + j;
    if (j >= ctbH) break;
    const uint32_t* s = row[r + 1];
    uint32_t nfm[4];
    {
      const int bx = (x << sh) >> 3;
      const uint8_t* nfp = a.nofilt_map + bx + ((y << sh) >> 3) * pic.w8;
      uint32_t f[4];
#pragma unroll
      for (int b = 0; b < 4; b++) f[b] = ((b < 2 || sh) && bx + b < pic.w8 && (nfp[b] & 1)) ? 0xFFFFFFFFu : 0u;
      nfm[0] = f[0];
      nfm[1] = sh ? f[1] : f[0];
      nfm[2] = sh ? f[2] : f[1];
      nfm[3] = sh ? f[3] : f[1];
    }
    uint32_t out[4];
    if (edge) {
      // neighbour words: a = row (r + 1 + vy0) shifted by hx0 samples, b = row (r + 1 - vy0) shifted by -hx0
      // (rows picked with selects: r is a compile-time index, vy0 is not)
      uint32_t Ra[4], Rb[4], A[4], B[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        Ra[k] = vy0 ? row[r][k] : row[r + 1][k];
        Rb[k] = vy0 ? row[r + 2][k] : row[r + 1][k];
      }
      const uint32_t la = vy0 ? lft[r] : lft[r + 1], ga = vy0 ? rgt[r] : rgt[r + 1];
      const uint32_t lb = vy0 ? lft[r + 2] : lft[r + 1], gb = vy0 ? rgt[r + 2] : rgt[r + 1];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint32_t am = k ? Ra[k ? k - 1 : 0] : la << 24, ap = (k < 3) ? Ra[k < 3 ? k + 1 : 3] : ga;
        const uint32_t bm = k ? Rb[k ? k - 1 : 0] : lb << 24, bp = (k < 3) ? Rb[k < 3 ? k + 1 : 3] : gb;
        // sample x-1 of word k: (w << 8) | (prev >> 24); sample x+1: (w >> 8) | (next << 24)
        A[k] = (hx0 < 0) ? __funnelshift_l(am, Ra[k], 8) : (hx0 > 0) ? __funnelshift_r(Ra[k], ap, 8) : Ra[k];
        B[k] = (hx0 < 0) ? __funnelshift_r(Rb[k], bp, 8) : (hx0 > 0) ? __funnelshift_l(bm, Rb[k], 8) : Rb[k];
      }
      // samples whose neighbours must not be used (sao.cc:125-190), as in k_sao but for 16 samples
      unsigned bad = 0;
      {
        const int i = i0;
        const unsigned first = (i == 0) ? 1u : 0u, last = (i + 16 >= ctbW) ? 1u << (ctbW - 1 - i) : 0u;
        const bool hrow = (j == 0 || j == ctbH - 1);
        if (hrow || first || last) {
          const int dya = (j + vy0 < 0) ? -1 : 0, dyb = (j - vy0 >= ctbH) ? 1 : 0;  // vy0 <= 0
          const unsigned a_mid = (m >> ((dya + 1) * 3 + 1)) & 1, b_mid = (m >> ((dyb + 1) * 3 + 1)) & 1;
          const unsigned a_side = (m >> ((dya + 1) * 3 + 1 + hx0)) & 1, b_side = (m >> ((dyb + 1) * 3 + 1 - hx0)) & 1;
          unsigned ma = a_mid ? 0xFFFFu : 0u, mb = b_mid ? 0xFFFFu : 0u;
          const unsigned sa = (hx0 < 0) ? first : (hx0 > 0) ? last : 0u, sb = (hx0 > 0) ? first : (hx0 < 0) ? last : 0u;
          ma = (ma & ~sa) | (a_side ? sa : 0u);
          mb = (mb & ~sb) | (b_side ? sb : 0u);
          const unsigned border = hrow ? 0xFFFFu : (first | last);  // sao.cc:125: tests only on the CTB border
          bad = border & ~(ma & mb);
        }
      }
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint32_t ltA = sao8_lt(s[k], A[k]), gtA = sao8_lt(A[k], s[k]), ltB = sao8_lt(s[k], B[k]), gtB = sao8_lt(B[k], s[k]);
        const uint32_t m2n = ltA & ltB, m2p = gtA & gtB;
        const uint32_t m1n = (ltA ^ ltB) & ~(gtA | gtB), m1p = (gtA ^ gtB) & ~(ltA | ltB);
        uint32_t keep = nfm[k];
        if (bad) keep |= sao8_mask4(bad >> (4 * k));
        const uint32_t p = ((m2n & opos[0]) | (m1n & opos[1]) | (m1p & opos[2]) | (m2p & opos[3])) & ~keep;
        const uint32_t n = ((m2n & oneg[0]) | (m1n & oneg[1]) | (m1p & oneg[2]) | (m2p & oneg[3])) & ~keep;
        out[k] = sao8_apply(s[k], p, n);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint32_t band = (s[k] >> 3) & 0x1F1F1F1Fu;
        const uint32_t kk = ((band | 0x20202020u) - pos4) & 0x1F1F1F1Fu;  // (band - position) & 31 per byte
        const uint32_t e0 = sao8_eq_small(kk, 0u), e1 = sao8_eq_small(kk, 0x01010101u), e2 = sao8_eq_small(kk, 0x02020202u),
                       e3 = sao8_eq_small(kk, 0x03030303u);
        const uint32_t p = ((e0 & opos[0]) | (e1 & opos[1]) | (e2 & opos[2]) | (e3 & opos[3])) & ~nfm[k];
        const uint32_t n = ((e0 & oneg[0]) | (e1 & oneg[1]) | (e2 & oneg[2]) | (e3 & oneg[3])) & ~nfm[k];
        out[k] = sao8_apply(s[k], p, n);
      }
    }
    store_row(y, make_uint4(out[0], out[1], out[2], out[3]));
  }
}
