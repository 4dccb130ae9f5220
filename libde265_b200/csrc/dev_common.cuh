// dev_common.cuh — shared device-side definitions for the B200 HEVC reconstruction kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200hevc.h"

#define B200_WARP 32

// Replicated border of every surface plane, in samples (dpb.cuh surface_ensure; the MC kernels rely on it)
#define B200_PAD_X 128   // luma columns, >= widest MC window - 1
#define B200_PAD_Y 80    // luma rows
#define B200_PAD_CX 64   // chroma columns
#define B200_PAD_CY 40

// Geometry + per-picture constants passed by value to every kernel.
struct DevPic {
  int w, h;            // luma size
  int cw, ch;          // chroma size (0 when monochrome)
  int bd_y, bd_c;
  int log2ctb, wctb, hctb;
  int w4, h4, w8, h8;
  int chroma;          // chroma_format_idc (0 or 1 supported on the device)
  int cb_qp_off, cr_qp_off;
  uint32_t flags;      // B200_PIC_*
  uint8_t* cur[3];     // working surface (pre-SAO)
  uint8_t* out[3];     // final surface (DPB slot)
  int pitch[3];        // bytes, identical for cur/out/refs
};

struct RefTable {
  const uint8_t* plane[B200_MAX_SLOTS][3];  // null when the slot holds no picture
};

// ---- tables (filled once per process by engine.cu) ----
__constant__ int8_t c_dct[32][32];  // HEVC core transform (fallback-dct.cc:512-545); single translation unit

__device__ __forceinline__ int clip3i(int lo, int hi, int v) { return min(max(v, lo), hi); }
__device__ __forceinline__ int clip_bd(int v, int bd) { return min(max(v, 0), (1 << bd) - 1); }

template <typename P>
__device__ __forceinline__ P* row_ptr(uint8_t* base, int pitch, int y) { return reinterpret_cast<P*>(base + (size_t)y * pitch); }
template <typename P>
__device__ __forceinline__ const P* row_ptr(const uint8_t* base, int pitch, int y) { return reinterpret_cast<const P*>(base + (size_t)y * pitch); }

// luma taps at integer offsets -3..+4 (fallback-motion.cc:531-555), chroma taps at -1..+2 (:357-364)
__constant__ int8_t k_qpel[4][8] = {
    {0, 0, 0, 64, 0, 0, 0, 0}, {-1, 4, -10, 58, 17, -5, 1, 0}, {-1, 4, -11, 40, 40, -11, 4, -1}, {0, 1, -5, 17, 58, -10, 4, -1}};
__constant__ int8_t k_epel[8][4] = {{0, 64, 0, 0},   {-2, 58, 10, -2}, {-4, 54, 16, -2}, {-6, 46, 28, -4},
                                                      {-4, 36, 36, -4}, {-4, 28, 46, -6}, {-2, 16, 54, -4}, {-2, 10, 58, -2}};
