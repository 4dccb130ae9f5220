// export.cuh — b200_engine_export_slot's RGB conversion: planar 8-bit R, G, B from a 4:2:0 or 4:0:0 picture of any luma / chroma
// depth (8..12 bit each), nearest chroma.  The YUV export is a plain 2-D copy (engine.cu).  The coefficient derivation and the
// per-pixel function are __host__ __device__ so that tests/export_emul.cu runs them on the CPU (tests/test_cpu_export.py).
//
// For each output channel o, integer only:
//   o = clamp(0, 255, (a_o·(Y − oY) + b_o·(Cb − oC) + c_o·(Cr − oC) + 2^15) >> 16)
//   limited range: oY = 16 << (BdY − 8), rangeY = 219 << (BdY − 8), rangeC = 224 << (BdC − 8)
//   full range:    oY = 0, rangeY = 2^BdY − 1, rangeC = 2^BdC − 1;   both: oC = 1 << (BdC − 1)
//   coefficient = floor(2^16 · 255 · k / range + 0.5): k = 1 for Y; R: 2(1 − Kr) for Cr; G: −2Kb(1 − Kb)/Kg for Cb and
//   −2Kr(1 − Kr)/Kg for Cr; B: 2(1 − Kb) for Cb; Kg = 1 − Kr − Kb.
// Every term fits in int32: |coefficient · (sample − offset)| < 2^25 at any depth up to 12 bit.
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define EXPORT_HD __host__ __device__ __forceinline__
#else
#define EXPORT_HD inline
#endif

struct ExportCoefs {
  int y;         // Y -> R, G, B
  int r_cr;      // Cr -> R
  int g_cb, g_cr;
  int b_cb;      // Cb -> B
  int oy, oc;    // luma offset, chroma mid-point
};

// matrix: 1 BT.601, 2 BT.709, 3 BT.2020 (B200_EXPORT_RGB_*).  Host only in practice (double arithmetic).
EXPORT_HD ExportCoefs export_coefs(int matrix, bool full_range, int bd_y, int bd_c)
{
  const double kr = matrix == 1 ? 0.299 : matrix == 2 ? 0.2126 : 0.2627;
  const double kb = matrix == 1 ? 0.114 : matrix == 2 ? 0.0722 : 0.0593;
  const double kg = 1.0 - kr - kb;
  const double range_y = full_range ? (double)((1 << bd_y) - 1) : (double)(219 << (bd_y - 8));
  const double range_c = full_range ? (double)((1 << bd_c) - 1) : (double)(224 << (bd_c - 8));
  auto q = [](double k, double range) { return (int)floor(65536.0 * 255.0 * k / range + 0.5); };
  ExportCoefs c;
  c.y = q(1.0, range_y);
  c.r_cr = q(2.0 * (1.0 - kr), range_c);
  c.g_cb = q(-2.0 * kb * (1.0 - kb) / kg, range_c);
  c.g_cr = q(-2.0 * kr * (1.0 - kr) / kg, range_c);
  c.b_cb = q(2.0 * (1.0 - kb), range_c);
  c.oy = full_range ? 0 : 16 << (bd_y - 8);
  c.oc = 1 << (bd_c - 1);
  return c;
}

EXPORT_HD uint8_t export_clamp8(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

EXPORT_HD void export_rgb_pixel(const ExportCoefs& c, int y, int cb, int cr, uint8_t& r, uint8_t& g, uint8_t& b)
{
  const int ty = c.y * (y - c.oy) + (1 << 15), u = cb - c.oc, v = cr - c.oc;
  r = export_clamp8((ty + c.r_cr * v) >> 16);
  g = export_clamp8((ty + c.g_cb * u + c.g_cr * v) >> 16);
  b = export_clamp8((ty + c.b_cb * u) >> 16);
}

#ifdef __CUDACC__
// One thread: EXPORT_V consecutive pixels of one output row.  Loads and stores are vectors where the addresses allow it (the
// aligned interior); a crop at any even offset, any output pitch and the window's last partial group take the per-sample path.
#define EXPORT_V 8
struct ExportArgs {
  const uint8_t* src[3];  // sample (x, y) of the window in Y, sample (x / 2, y / 2) in Cb / Cr
  int src_pitch[3];
  uint8_t* dst[3];        // R, G, B
  size_t dst_pitch[3];
  int w, h;
  ExportCoefs c;
};

template <typename T, int N>
struct alignas(sizeof(T) * N) Vec { T v[N]; };

template <typename PY, typename PC, bool MONO>
__global__ void __launch_bounds__(256) k_export_rgb(ExportArgs a)
{
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * EXPORT_V, row = blockIdx.y * blockDim.y + threadIdx.y;
  if (x0 >= a.w || row >= a.h) return;
  const PY* ys = reinterpret_cast<const PY*>(a.src[0] + (size_t)row * a.src_pitch[0]) + x0;
  const PC *us = nullptr, *vs = nullptr;
  if (!MONO) {
    us = reinterpret_cast<const PC*>(a.src[1] + (size_t)(row >> 1) * a.src_pitch[1]) + (x0 >> 1);
    vs = reinterpret_cast<const PC*>(a.src[2] + (size_t)(row >> 1) * a.src_pitch[2]) + (x0 >> 1);
  }
  uint8_t* rd = a.dst[0] + (size_t)row * a.dst_pitch[0] + x0;
  uint8_t* gd = a.dst[1] + (size_t)row * a.dst_pitch[1] + x0;
  uint8_t* bd = a.dst[2] + (size_t)row * a.dst_pitch[2] + x0;
  const int n = min(EXPORT_V, a.w - x0);
  int yv[EXPORT_V], uv[EXPORT_V / 2], vv[EXPORT_V / 2];
  if (n == EXPORT_V && (reinterpret_cast<uintptr_t>(ys) % sizeof(Vec<PY, EXPORT_V>)) == 0) {
    const Vec<PY, EXPORT_V> t = *reinterpret_cast<const Vec<PY, EXPORT_V>*>(ys);
#pragma unroll
    for (int i = 0; i < EXPORT_V; i++) yv[i] = t.v[i];
  } else {
#pragma unroll
    for (int i = 0; i < EXPORT_V; i++) yv[i] = i < n ? (int)ys[i] : 0;
  }
  if (MONO) {
#pragma unroll
    for (int i = 0; i < EXPORT_V / 2; i++) uv[i] = vv[i] = a.c.oc;
  } else if (n == EXPORT_V && (reinterpret_cast<uintptr_t>(us) % sizeof(Vec<PC, EXPORT_V / 2>)) == 0 &&
             (reinterpret_cast<uintptr_t>(vs) % sizeof(Vec<PC, EXPORT_V / 2>)) == 0) {
    const Vec<PC, EXPORT_V / 2> tu = *reinterpret_cast<const Vec<PC, EXPORT_V / 2>*>(us), tv = *reinterpret_cast<const Vec<PC, EXPORT_V / 2>*>(vs);
#pragma unroll
    for (int i = 0; i < EXPORT_V / 2; i++) { uv[i] = tu.v[i]; vv[i] = tv.v[i]; }
  } else {
#pragma unroll
    for (int i = 0; i < EXPORT_V / 2; i++) {
      uv[i] = 2 * i < n ? (int)us[i] : 0;
      vv[i] = 2 * i < n ? (int)vs[i] : 0;
    }
  }
  Vec<uint8_t, EXPORT_V> r, g, b;
#pragma unroll
  for (int i = 0; i < EXPORT_V; i++) export_rgb_pixel(a.c, yv[i], uv[i >> 1], vv[i >> 1], r.v[i], g.v[i], b.v[i]);
  if (n == EXPORT_V && ((reinterpret_cast<uintptr_t>(rd) | reinterpret_cast<uintptr_t>(gd) | reinterpret_cast<uintptr_t>(bd)) % EXPORT_V) == 0) {
    *reinterpret_cast<Vec<uint8_t, EXPORT_V>*>(rd) = r;
    *reinterpret_cast<Vec<uint8_t, EXPORT_V>*>(gd) = g;
    *reinterpret_cast<Vec<uint8_t, EXPORT_V>*>(bd) = b;
  } else {
    for (int i = 0; i < n; i++) { rd[i] = r.v[i]; gd[i] = g.v[i]; bd[i] = b.v[i]; }
  }
}

// bytes per luma / chroma sample pick the instantiation; 4:0:0 has no chroma planes.
static void launch_export_rgb(const ExportArgs& a, int bytes_y, int bytes_c, bool mono, cudaStream_t st)
{
  const dim3 block(32, 8), grid((a.w + EXPORT_V * 32 - 1) / (EXPORT_V * 32), (a.h + 7) / 8);
  if (mono) {
    if (bytes_y == 1) k_export_rgb<uint8_t, uint8_t, true><<<grid, block, 0, st>>>(a);
    else k_export_rgb<uint16_t, uint16_t, true><<<grid, block, 0, st>>>(a);
  } else if (bytes_y == 1) {
    if (bytes_c == 1) k_export_rgb<uint8_t, uint8_t, false><<<grid, block, 0, st>>>(a);
    else k_export_rgb<uint8_t, uint16_t, false><<<grid, block, 0, st>>>(a);
  } else {
    if (bytes_c == 1) k_export_rgb<uint16_t, uint8_t, false><<<grid, block, 0, st>>>(a);
    else k_export_rgb<uint16_t, uint16_t, false><<<grid, block, 0, st>>>(a);
  }
}
#endif
