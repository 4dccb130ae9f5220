// tma_probe.cu — microbenchmark behind the MC kernel's staging design (DESIGN.md §4): how many small 2-D / 3-D TMA boxes
// (reference windows of one MC unit: 23 rows of 32..80 bytes) can one SM fetch per microsecond from an L2/HBM-resident
// padded 4K surface, against the same windows fetched with per-lane 16-byte loads + shared-memory stores?
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_probe tools/tma_probe.cu && ./tma_probe
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CK(x)                                                                         \
  do {                                                                                \
    cudaError_t e_ = (x);                                                             \
    if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } \
  } while (0)

typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, int n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t phase)
{
  asm volatile(
      "{\n.reg .pred p;\nW: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D;\nbra W;\nD:\n}" ::"r"(smem_u32(b)), "r"(phase)
      : "memory");
}
__device__ __forceinline__ void tma2d(void* dst, const CUtensorMap* m, int x, int y, uint64_t* b)
{
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)), "l"(m),
               "r"(x), "r"(y), "r"(smem_u32(b))
               : "memory");
}
__device__ __forceinline__ void tma3d(void* dst, const CUtensorMap* m, int x, int y, int z, uint64_t* b)
{
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(dst)),
               "l"(m), "r"(x), "r"(y), "r"(z), "r"(smem_u32(b))
               : "memory");
}

#define WARPS 4
#define DEPTH 4
#define BUF_BYTES 2304  // >= 96 * 23 (the ldg variant stages 16 extra bytes per row), 128-byte aligned slots

__device__ __forceinline__ uint32_t hash32(uint32_t v)
{
  v ^= v >> 16; v *= 0x7feb352du; v ^= v >> 15; v *= 0x846ca68bu; v ^= v >> 16;
  return v;
}

// mode 0: 2-D TMA of one box per op; mode 1: 3-D TMA (bw x bh x 2 planes); mode 2: per-lane 16-byte loads + STS.128
__constant__ CUtensorMap c_maps[4];

template <int MODE, int SRC>  // SRC: where the tensor map lives: 0 global memory, 1 __grid_constant__ kernel parameter, 2 __constant__ array
__global__ void __launch_bounds__(WARPS * 32) k_probe(const CUtensorMap* gmap, const __grid_constant__ CUtensorMap pmap, const uint8_t* __restrict__ base,
                                                       int pitch, int W, int H, int bw, int bh, int iters, unsigned* sink)
{
  const CUtensorMap* map = SRC == 0 ? gmap : SRC == 1 ? &pmap : &c_maps[1];
  __shared__ __align__(128) uint8_t buf[WARPS][DEPTH][BUF_BYTES];
  __shared__ uint64_t bar[WARPS][DEPTH];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bytes = (uint32_t)bw * bh * (MODE == 1 ? 2 : 1);
  if (lane == 0)
    for (int d = 0; d < DEPTH; d++) mbar_init(&bar[warp][d], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const uint32_t wid = (blockIdx.x * WARPS + warp) * 7919u;
  unsigned acc = 0;
  auto coords = [&](int i, int& x, int& y) {
    const uint32_t h = hash32(wid + i);
    x = (int)(h % (uint32_t)(W - bw)) & ~15;  // TMA box origins must be 16-byte aligned in the innermost dimension (tools/tma_probe2.cu)
    y = (int)((h >> 12) % (uint32_t)(H - bh));
  };
  if (MODE < 2) {
    if (lane == 0)
      for (int d = 0; d < DEPTH && d < iters; d++) {
        int x, y;
        coords(d, x, y);
        mbar_expect(&bar[warp][d], bytes);
        if (MODE == 0) tma2d(buf[warp][d], map, x, y, &bar[warp][d]);
        else tma3d(buf[warp][d], map, x, y, 0, &bar[warp][d]);
      }
    for (int i = 0; i < iters; i++) {
      const int d = i % DEPTH;
      mbar_wait(&bar[warp][d], (i / DEPTH) & 1);
      acc += reinterpret_cast<const uint32_t*>(buf[warp][d])[lane];
      __syncwarp();
      if (lane == 0 && i + DEPTH < iters) {
        int x, y;
        coords(i + DEPTH, x, y);
        mbar_expect(&bar[warp][d], bytes);
        if (MODE == 0) tma2d(buf[warp][d], map, x, y, &bar[warp][d]);
        else tma3d(buf[warp][d], map, x, y, 0, &bar[warp][d]);
      }
    }
  } else {
    // window rows of bw bytes starting at arbitrary x: aligned 16-byte chunks covering [x & ~15, x + bw) -> smem row pitch bw + 16
    const int cpr = bw / 16 + 1;  // chunks per row
    for (int i = 0; i < iters; i++) {
      const int d = i % DEPTH;
      int x, y;
      coords(i, x, y);
      const uint8_t* src = base + (size_t)y * pitch + (x & ~15);
      for (int t = lane; t < bh * cpr; t += 32) {
        const int r = t / cpr, c = t - r * cpr;
        const uint4 v = *reinterpret_cast<const uint4*>(src + (size_t)r * pitch + 16 * c);
        *reinterpret_cast<uint4*>(&buf[warp][d][(r * cpr + c) * 16]) = v;
      }
      __syncwarp();
      acc += reinterpret_cast<const uint32_t*>(buf[warp][d])[lane];
      __syncwarp();
    }
  }
  if (acc == 0x12345678u) *sink = acc;
}

template <int SRC>
static void launch(int mode, int grid, const CUtensorMap* dmap, const CUtensorMap& m, const uint8_t* d, int W, int H, int bw, int bh, int iters, unsigned* sink)
{
  if (mode == 0) k_probe<0, SRC><<<grid, WARPS * 32>>>(dmap, m, d, W, W, H, bw, bh, iters, sink);
  else if (mode == 1) k_probe<1, SRC><<<grid, WARPS * 32>>>(dmap, m, d, W, W, H, bw, bh, iters, sink);
  else k_probe<2, SRC><<<grid, WARPS * 32>>>(dmap, m, d, W, W, H, bw, bh, iters, sink);
}

int main(int argc, char** argv)
{
  const int src = argc > 1 ? atoi(argv[1]) : 1, only = argc > 2 ? atoi(argv[2]) : -1;
  const int W = 4096, H = 2320;  // padded 4K luma surface
  uint8_t* d;
  CK(cudaMalloc(&d, (size_t)W * H * 2));
  CK(cudaMemset(d, 1, (size_t)W * H * 2));
  EncodeTiled enc = nullptr;
  cudaDriverEntryPointQueryResult qr;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &qr));
  if (!enc) { printf("no cuTensorMapEncodeTiled\n"); return 1; }
  unsigned* sink;
  CK(cudaMalloc(&sink, 4));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  int clk = 0;
  CK(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0));
  printf("SMs %d, clock %d kHz, tensor map source %d (0 global, 1 grid_constant param, 2 __constant__)\n", sms, clk, src);
  struct Case { int mode, bw, bh; const char* name; };
  const Case cases[] = {{0, 32, 23, "tma2d 32x23"}, {0, 48, 23, "tma2d 48x23"}, {0, 80, 23, "tma2d 80x23"}, {0, 32, 15, "tma2d 32x15"}, {0, 16, 11, "tma2d 16x11"},
                        {1, 16, 11, "tma3d 16x11x2"}, {1, 48, 11, "tma3d 48x11x2"}, {0, 80, 71, "tma2d 80x71 (5.7 KB: needs BUF 8 KB: skipped)"},
                        {2, 32, 23, "ldg128 32(+16)x23"}, {2, 48, 23, "ldg128 48(+16)x23"}, {2, 80, 23, "ldg128 80(+16)x23"}, {2, 16, 11, "ldg128 16(+16)x11"}};
  CUtensorMap* dmap;
  CK(cudaMalloc(&dmap, sizeof(CUtensorMap)));
  int ci = -1;
  for (const Case& c : cases) {
    ci++;
    if (only >= 0 && ci != only) continue;
    if (c.bw * c.bh * (c.mode == 1 ? 2 : 1) > BUF_BYTES) continue;
    CUtensorMap m;
    memset(&m, 0, sizeof(m));
    if (c.mode == 0) {
      cuuint64_t dims[2] = {(cuuint64_t)W, (cuuint64_t)H}, strides[1] = {(cuuint64_t)W};
      cuuint32_t box[2] = {(cuuint32_t)c.bw, (cuuint32_t)c.bh}, es[2] = {1, 1};
      CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r) { printf("%s: encode failed %d\n", c.name, (int)r); continue; }
    } else if (c.mode == 1) {
      cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, 2}, strides[2] = {(cuuint64_t)W, (cuuint64_t)W * H};
      cuuint32_t box[3] = {(cuuint32_t)c.bw, (cuuint32_t)c.bh, 2}, es[3] = {1, 1, 1};
      CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r) { printf("%s: encode failed %d\n", c.name, (int)r); continue; }
    }
    CK(cudaMemcpy(dmap, &m, sizeof(m), cudaMemcpyHostToDevice));
    CK(cudaMemcpyToSymbol(c_maps, &m, sizeof(m), sizeof(m)));  // slot 1
    for (int ctas_per_sm = 1; ctas_per_sm <= 4; ctas_per_sm *= 2) {
      const int iters = 2000, grid = sms * ctas_per_sm;
      cudaEvent_t e0, e1;
      CK(cudaEventCreate(&e0));
      CK(cudaEventCreate(&e1));
      for (int rep = 0; rep < 2; rep++) {
        CK(cudaEventRecord(e0));
        if (src == 0) launch<0>(c.mode, grid, dmap, m, d, W, H, c.bw, c.bh, iters, sink);
        else if (src == 1) launch<1>(c.mode, grid, dmap, m, d, W, H, c.bw, c.bh, iters, sink);
        else launch<2>(c.mode, grid, dmap, m, d, W, H, c.bw, c.bh, iters, sink);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
      }
      CK(cudaGetLastError());
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      const double ops = (double)grid * WARPS * iters, per_sm_us = ops / sms / (ms * 1e3);
      const double bytes = ops * c.bw * c.bh * (c.mode == 1 ? 2 : 1);
      printf("%-28s ctas/SM %d: %8.3f ms  %7.2f boxes/us/SM  (%6.1f cycles/box/SM @1.965 GHz)  %7.1f GB/s useful\n", c.name, ctas_per_sm, ms, per_sm_us,
             1965.0 / per_sm_us, bytes / (ms * 1e6));
    }
  }
  return 0;
}
