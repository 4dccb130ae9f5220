// dpb.cuh — the picture store: device surfaces with replicated borders, the DPB names mapped onto them, and the per-surface
// events that order pictures across the engine's streams.  It owns no stream: the caller passes the one an access is issued on.
// Host code plus the border kernel.  Included by engine.cu (one translation unit), which defines B200_MAX_CTX (streams).
#pragma once

// ---- surfaces ------------------------------------------------------------------------------------
// A surface keeps a replicated BORDER around every plane (B200_PAD_* samples on each side) so that the motion-compensation
// kernel never clamps a coordinate: mc_luma / mc_chroma clamp every reference sample position to the picture
// (motion.cc:147-153, 251-254), which is the same as reading a picture whose edge samples are replicated outwards; a window
// that lies further out than the border is moved to the border's rim, where every sample already is the edge sample.
// plane[c] points at sample (0, 0); the two chroma planes share one allocation (fixed plane stride) so that one 3-D TMA box
// fetches the Cb and the Cr window of a prediction unit.
// (B200_PAD_X / _Y / _CX / _CY: dev_common.cuh)

struct Surface {
  uint8_t* plane[3] = {nullptr, nullptr, nullptr};  // sample (0,0) of each plane
  uint8_t* alloc[2] = {nullptr, nullptr};           // luma allocation, chroma allocation (Cb then Cr)
  size_t alloc_bytes[2] = {0, 0};
  int pitch[3] = {0, 0, 0};
  int w = 0, h = 0, cw = 0, ch = 0, chroma = 0, bd_y = 0, bd_c = 0;
  bool valid = false;  // holds a picture
  bool has_tm = false; // tensor maps of the padded planes for the TMA-staged MC kernel (8-bit surfaces)
  CUtensorMap tm_luma[2], tm_chroma[2];  // [0] big boxes, [1] small boxes (kernels_mct.cuh)
};

// cuTensorMapEncodeTiled through the runtime (no link-time dependency on libcuda)
typedef CUresult (*b200_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                         const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static b200_encode_tiled_fn encode_tiled()
{
  static b200_encode_tiled_fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) p = nullptr;
    return (b200_encode_tiled_fn)p;
  }();
  return fn;
}

static void surface_free(Surface& s)
{
  for (int i = 0; i < 2; i++) {
    if (s.alloc[i]) cudaFree(s.alloc[i]);
    s.alloc[i] = nullptr;
  }
  for (int c = 0; c < 3; c++) s.plane[c] = nullptr;
  s.w = s.h = 0;
  s.valid = false;
}

static int bytes_per_sample(int bd) { return bd > 8 ? 2 : 1; }

// What a surface's allocation depends on.  A bit-depth change that keeps the bytes per sample (9 <-> 10 <-> 12) only relabels it.
struct SurfaceFormat {
  int w, h, chroma, bytes_y, bytes_c;  // all 0: no allocation
  bool operator==(const SurfaceFormat& o) const { return w == o.w && h == o.h && chroma == o.chroma && bytes_y == o.bytes_y && bytes_c == o.bytes_c; }
};
static SurfaceFormat format_of(const b200_pic_params& p) { return {p.width, p.height, p.chroma_format_idc, bytes_per_sample(p.bit_depth_luma), bytes_per_sample(p.bit_depth_chroma)}; }
static SurfaceFormat format_of(const Surface& s) { return s.plane[0] ? SurfaceFormat{s.w, s.h, s.chroma, bytes_per_sample(s.bd_y), bytes_per_sample(s.bd_c)} : SurfaceFormat{}; }

// A reference whose picture differs from the current one in size, chroma format or the EXACT luma / chroma bit depth is a
// missing reference and predicts mid-grey, as in the reference (motion.cc:385-405, DESIGN §3).  Not the allocation format: a
// 10-bit picture does not reference a 12-bit one, although the two could share a surface.  The CTB size does not matter.
static bool usable_reference(const Surface& s, const b200_pic_params& p)
{
  return s.valid && s.w == p.width && s.h == p.height && s.chroma == p.chroma_format_idc && s.bd_y == p.bit_depth_luma && s.bd_c == p.bit_depth_chroma;
}

// New surfaces are zero-filled ON THE ENGINE'S STREAM (it is non-blocking: a memset on the legacy stream could land after
// kernels launched later on the engine's stream).
static int surface_ensure(Surface& s, const b200_pic_params& p, cudaStream_t st)
{
  const int cw = p.chroma_format_idc ? p.width / 2 : 0, ch = p.chroma_format_idc ? p.height / 2 : 0;
  if (format_of(s) == format_of(p)) {
    s.bd_y = p.bit_depth_luma;
    s.bd_c = p.bit_depth_chroma;
    return B200_OK;
  }
  surface_free(s);
  s.w = p.width; s.h = p.height; s.cw = cw; s.ch = ch; s.chroma = p.chroma_format_idc;
  s.bd_y = p.bit_depth_luma; s.bd_c = p.bit_depth_chroma;
  const int bl = bytes_per_sample(p.bit_depth_luma), bc = bytes_per_sample(p.bit_depth_chroma);
  // rows padded to 256 bytes: sample (0, y) is 128-byte aligned, every CTB row segment 16-byte aligned, and vector accesses may
  // overshoot the picture width inside the border
  s.pitch[0] = (int)align_up((size_t)(p.width + 2 * B200_PAD_X) * bl, 256);
  s.pitch[1] = s.pitch[2] = cw ? (int)align_up((size_t)(cw + 2 * B200_PAD_CX) * bc, 256) : 0;
  s.alloc_bytes[0] = (size_t)s.pitch[0] * (p.height + 2 * B200_PAD_Y);
  CU(cudaMalloc(&s.alloc[0], s.alloc_bytes[0]));
  CU(cudaMemsetAsync(s.alloc[0], 0, s.alloc_bytes[0], st));
  s.plane[0] = s.alloc[0] + (size_t)B200_PAD_Y * s.pitch[0] + (size_t)B200_PAD_X * bl;
  if (cw) {
    const size_t plane_bytes = (size_t)s.pitch[1] * (ch + 2 * B200_PAD_CY);
    s.alloc_bytes[1] = 2 * plane_bytes;
    CU(cudaMalloc(&s.alloc[1], s.alloc_bytes[1]));
    CU(cudaMemsetAsync(s.alloc[1], 0, s.alloc_bytes[1], st));
    for (int c = 1; c < 3; c++) s.plane[c] = s.alloc[1] + (c - 1) * plane_bytes + (size_t)B200_PAD_CY * s.pitch[1] + (size_t)B200_PAD_CX * bc;
  }
  s.has_tm = false;
  if (bl == 1 && bc == 1) {
    // Tensor maps over the PADDED planes (coordinate = picture coordinate + border): rows of `pitch` bytes; boxes of one MC
    // tile's reference window (kernels_mct.cuh).  Out-of-range box parts (skew rows above the surface) are zero-filled and unused.
    b200_encode_tiled_fn enc = encode_tiled();
    if (!enc) return set_err(B200_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
    for (int k = 0; k < 2; k++) {
      cuuint64_t dims[2] = {(cuuint64_t)s.pitch[0], (cuuint64_t)(p.height + 2 * B200_PAD_Y)}, strides[1] = {(cuuint64_t)s.pitch[0]};
      cuuint32_t box[2] = {(cuuint32_t)(k ? MCT_LWS_PITCH : MCT_LWB_PITCH), (cuuint32_t)(k ? MCT_LWS_ROWS : MCT_LWB_ROWS)}, es[2] = {1, 1};
      if (enc(&s.tm_luma[k], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, s.alloc[0], dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return set_err(B200_ERR_CUDA, "cuTensorMapEncodeTiled (luma) failed");
      if (cw) {
        cuuint64_t cdims[3] = {(cuuint64_t)s.pitch[1], (cuuint64_t)(ch + 2 * B200_PAD_CY), 2};
        cuuint64_t cstrides[2] = {(cuuint64_t)s.pitch[1], (cuuint64_t)s.pitch[1] * (ch + 2 * B200_PAD_CY)};
        cuuint32_t cbox[3] = {(cuuint32_t)(k ? MCT_CWS_PITCH : MCT_CWB_PITCH), (cuuint32_t)(k ? MCT_CWS_ROWS : MCT_CWB_ROWS), 2}, ces[3] = {1, 1, 1};
        if (enc(&s.tm_chroma[k], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, s.alloc[1], cdims, cstrides, cbox, ces, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
          return set_err(B200_ERR_CUDA, "cuTensorMapEncodeTiled (chroma) failed");
      } else {
        s.tm_chroma[k] = s.tm_luma[k];
      }
    }
    s.has_tm = true;
  }
  return B200_OK;
}

// Replicates the edge samples of a finished picture into its border (one launch for all planes).  blockIdx.y = plane.
//   part 1 (rows 0..h-1): the pad_x samples left of column 0 and right of column w-1;
//   part 2 (pad_y rows above row 0 and below row h-1): the whole padded row, copied from row 0 / h-1 with the column clamped.
template <typename P>
__global__ void k_extend_borders(uint8_t* p0, uint8_t* p1, uint8_t* p2, int pitch0, int pitch1, int w, int h, int cw, int ch)
{
  const int c = blockIdx.y;
  uint8_t* base = c == 0 ? p0 : c == 1 ? p1 : p2;
  const int pitch = c ? pitch1 : pitch0, pw = c ? cw : w, ph = c ? ch : h;
  const int padx = c ? B200_PAD_CX : B200_PAD_X, pady = c ? B200_PAD_CY : B200_PAD_Y;
  constexpr int V = 16 / sizeof(P);       // samples per 16-byte store
  const int side_chunks = padx / V;       // per side and row
  const int n1 = ph * 2 * side_chunks;
  const int row_chunks = (pw + 2 * padx + V - 1) / V;  // the last chunk may overshoot into the row's alignment padding (pitch is a multiple of 256)
  const int n2 = 2 * pady * row_chunks;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += gridDim.x * blockDim.x) {
    if (i < n1) {
      const int y = i / (2 * side_chunks), k = i - y * 2 * side_chunks;
      const bool right = k >= side_chunks;
      P* row = row_ptr<P>(base, pitch, y);
      const P v = right ? row[pw - 1] : row[0];
      P* dst = right ? row + pw + (k - side_chunks) * V : row - padx + k * V;
      P tmp[V];
#pragma unroll
      for (int j = 0; j < V; j++) tmp[j] = v;
      if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(tmp);
      else
        for (int j = 0; j < V; j++) dst[j] = v;  // chroma widths that are not a multiple of 16 bytes
    } else {
      const int j2 = i - n1;
      const int r = j2 / row_chunks, k = j2 - r * row_chunks;
      const bool below = r >= pady;
      const int y = below ? ph + (r - pady) : r - pady;
      const P* src = row_ptr<P>(base, pitch, below ? ph - 1 : 0);
      P* dst = row_ptr<P>(base, pitch, y) - padx + k * V;
      const int x0 = k * V - padx;
      P tmp[V];
#pragma unroll
      for (int j = 0; j < V; j++) tmp[j] = src[min(max(x0 + j, 0), pw - 1)];
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(tmp);
    }
  }
}

static void launch_extend_borders(const Surface& s, cudaStream_t st)
{
  dim3 grid(132 * 2, s.chroma ? 3 : 1);  // two CTAs per SM of an H100 SXM
  if (bytes_per_sample(s.bd_y) == 2)
    k_extend_borders<uint16_t><<<grid, 256, 0, st>>>(s.plane[0], s.plane[1], s.plane[2], s.pitch[0], s.pitch[1], s.w, s.h, s.cw, s.ch);
  else
    k_extend_borders<uint8_t><<<grid, 256, 0, st>>>(s.plane[0], s.plane[1], s.plane[2], s.pitch[0], s.pitch[1], s.w, s.h, s.cw, s.ch);
}

// ---- the store -----------------------------------------------------------------------------------
// DPB slots are NAMES (what the records' ref_slot / dst_slot say); the pictures live in a pool of physical surfaces.  A picture
// that writes slot d while earlier pictures on other streams still read (or write) d's current surface gets another, idle
// surface and the name moves — like register renaming, WAR / WAW hazards between pictures cost nothing, whatever slot policy
// the host's DPB has (libde265 reuses the first free image, dpb.cc: the hazard is the common case).  Only true (RAW)
// dependencies remain.  B200_RENAME=0 keeps every name on one surface.
#define B200_MAX_PHYS (B200_MAX_SLOTS + 32)  // physical surfaces: every name plus the renamed pictures in flight

// Per surface: an access issued on stream k waits only for those on other streams (same-stream accesses are ordered anyway).
// Exports (b200_engine_export_slot) read on the caller's streams, which are none of the engine's: one external-read event per
// surface covers all of them, because each export's stream waits for the previous one before it records the event again.
struct SlotSync {
  cudaEvent_t written = nullptr;
  int writer = -1;                       // stream of the last writer, -1: none in flight
  cudaEvent_t read[B200_MAX_CTX] = {};   // last read of this surface issued on each stream
  bool read_pending[B200_MAX_CTX] = {};
  cudaEvent_t ext_read = nullptr;        // last export of this surface, on the caller's stream
  bool ext_pending = false;
};

struct Dpb {
  Surface surf[B200_MAX_PHYS];
  SlotSync sync[B200_MAX_PHYS];
  int lmap[B200_MAX_SLOTS];       // name -> physical surface, -1: never written
  int owner[B200_MAX_PHYS];       // physical surface -> name it currently carries, -1: free (may still have readers in flight)
  int last_owner[B200_MAX_PHYS];  // the name it carried last (dpb_wait_events also waits for reads of a renamed-away surface)
  bool rename = true;
  uint64_t n_renamed = 0;
  SurfaceFormat issued{};  // format of the last picture issued
};

static int dpb_init(Dpb& d)
{
  memset(d.lmap, -1, sizeof(d.lmap));
  memset(d.owner, -1, sizeof(d.owner));
  memset(d.last_owner, -1, sizeof(d.last_owner));
  if (const char* e = getenv("B200_RENAME")) d.rename = atoi(e) != 0;
  for (auto& ss : d.sync) {
    CU(cudaEventCreateWithFlags(&ss.written, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ss.ext_read, cudaEventDisableTiming));
    for (auto& e : ss.read) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  return B200_OK;
}

// `report`: B200_HOST_PROF's line on slot renaming first.
static void dpb_destroy(Dpb& d, bool report)
{
  int n_surf = 0;
  for (const auto& sf : d.surf) n_surf += sf.plane[0] != nullptr;
  if (report)
    fprintf(stderr, "[b200] %llu pictures took their destination name to another surface (slot renaming); %d surfaces allocated\n",
            (unsigned long long)d.n_renamed, n_surf);
  for (auto& s : d.surf) surface_free(s);
  for (auto& ss : d.sync) {
    if (ss.written) cudaEventDestroy(ss.written);
    if (ss.ext_read) cudaEventDestroy(ss.ext_read);
    for (auto& e : ss.read)
      if (e) cudaEventDestroy(e);
  }
}

// The surface that holds the picture named `name`, or null.
static Surface* dpb_picture(Dpb& d, int name)
{
  const int ph = d.lmap[name];
  return ph >= 0 && d.surf[ph].valid ? &d.surf[ph] : nullptr;
}

// The references a picture sees: resolved against the names as they are BEFORE the picture takes its destination name.
static RefTable dpb_refs(Dpb& d, const b200_pic_params& p)
{
  RefTable refs;
  memset(&refs, 0, sizeof(refs));
  for (int i = 0; i < B200_MAX_SLOTS; i++) {
    const Surface* s = i == p.dst_slot ? nullptr : dpb_picture(d, i);
    if (s && usable_reference(*s, p))
      for (int c = 0; c < 3; c++) refs.plane[i][c] = s->plane[c];
  }
  return refs;
}

// Blocks until the exports of surface `ph` have finished (before it is freed or reallocated).
static int dpb_wait_export(Dpb& d, int ph)
{
  SlotSync& ss = d.sync[ph];
  if (ss.ext_pending) CU(cudaEventSynchronize(ss.ext_read));
  ss.ext_pending = false;
  return B200_OK;
}

// Blocks until every export has finished.
static int dpb_wait_exports(Dpb& d)
{
  for (int ph = 0; ph < B200_MAX_PHYS; ph++) {
    const int rc = dpb_wait_export(d, ph);
    if (rc) return rc;
  }
  return B200_OK;
}

// Format change (new SPS): drain `streams`, then drop every surface that carries no name — surfaces of another format cannot
// be reused as they are, and converting them one rename at a time (free + allocate, each a device-wide synchronisation) was
// measured to leave the second format at 75 % of its speed for a long time.
static int dpb_set_format(Dpb& d, const b200_pic_params& p, const cudaStream_t* streams, int n_streams)
{
  const SurfaceFormat f = format_of(p);
  if (d.issued.w && !(d.issued == f)) {
    for (int c = 0; c < n_streams; c++) CU(cudaStreamSynchronize(streams[c]));
    for (int ph = 0; ph < B200_MAX_PHYS; ph++)
      if (d.owner[ph] < 0 && d.surf[ph].plane[0] && !(format_of(d.surf[ph]) == f)) {
        const int rc = dpb_wait_export(d, ph);
        if (rc) return rc;
        surface_free(d.surf[ph]);
      }
  }
  d.issued = f;
  return B200_OK;
}

// Is every access to surface `ph` issued on a stream other than `k` (exports included) complete?  The completed ones are
// forgotten on the way.
static bool dpb_idle(Dpb& d, int ph, int k)
{
  SlotSync& ss = d.sync[ph];
  if (ss.writer >= 0 && ss.writer != k) {
    if (cudaEventQuery(ss.written) != cudaSuccess) return false;
    ss.writer = -1;
  }
  if (ss.ext_pending) {
    if (cudaEventQuery(ss.ext_read) != cudaSuccess) return false;
    ss.ext_pending = false;
  }
  for (int c = 0; c < B200_MAX_CTX; c++)
    if (c != k && ss.read_pending[c]) {
      if (cudaEventQuery(ss.read[c]) != cudaSuccess) return false;
      ss.read_pending[c] = false;
    }
  cudaGetLastError();  // cudaErrorNotReady is not sticky, but leave nothing behind
  return true;
}

// The surface a picture issued on stream `k` writes for the name `name` (null: none).  `overlap`: pictures on different
// streams may run at the same time; otherwise the name never moves.
static Surface* dpb_acquire(Dpb& d, int name, int k, const b200_pic_params& p, bool overlap)
{
  const int cur = d.lmap[name];
  if (cur >= 0 && (!d.rename || !overlap || dpb_idle(d, cur, k))) {
    // the name keeps its surface: one of another format is reallocated in place (surface_ensure), not behind its exports
    if (!(format_of(d.surf[cur]) == format_of(p))) dpb_wait_export(d, cur);
    return &d.surf[cur];
  }
  int best = -1, empty = -1, other = -1;
  for (int ph = 0; ph < B200_MAX_PHYS && best < 0; ph++) {
    if (d.owner[ph] >= 0) continue;
    const Surface& s = d.surf[ph];
    if (!s.plane[0]) { if (empty < 0) empty = ph; continue; }
    if (!dpb_idle(d, ph, k)) continue;
    if (format_of(s) == format_of(p)) best = ph;
    else if (other < 0) other = ph;
  }
  if (best < 0) best = empty >= 0 ? empty : other;  // a new surface, or an idle one of another format (surface_ensure reallocates it)
  if (best < 0) {  // pool exhausted: write in place behind the readers (dpb_order_before waits)
    if (cur >= 0 && !(format_of(d.surf[cur]) == format_of(p))) dpb_wait_export(d, cur);
    return cur >= 0 ? &d.surf[cur] : nullptr;
  }
  if (cur >= 0) {
    d.owner[cur] = -1;
    d.n_renamed++;
  }
  d.lmap[name] = best;
  d.owner[best] = name;
  d.last_owner[best] = name;
  return &d.surf[best];
}

// Before a picture issued on stream `k` (`st`) that writes the name `dst` (dpb_acquire): wait for the writers of its reference
// surfaces and for every earlier reader / writer of its destination surface that ran on another stream (none when the
// destination was renamed to an idle surface), exports included: the destination's name never moves with one stream, while
// timing is on or with B200_RENAME=0.
static int dpb_order_before(Dpb& d, int k, cudaStream_t st, uint32_t ref_mask, int dst)
{
  for (int r = 0; r < B200_MAX_SLOTS; r++) {
    if (!((ref_mask >> r) & 1) || r == dst || d.lmap[r] < 0) continue;
    SlotSync& ss = d.sync[d.lmap[r]];
    if (ss.writer >= 0 && ss.writer != k) CU(cudaStreamWaitEvent(st, ss.written, 0));
  }
  SlotSync& sd = d.sync[d.lmap[dst]];
  if (sd.writer >= 0 && sd.writer != k) CU(cudaStreamWaitEvent(st, sd.written, 0));
  for (int c = 0; c < B200_MAX_CTX; c++)
    if (c != k && sd.read_pending[c]) CU(cudaStreamWaitEvent(st, sd.read[c], 0));
  if (sd.ext_pending) CU(cudaStreamWaitEvent(st, sd.ext_read, 0));
  return B200_OK;
}

// An export of the picture named `name` on the caller's stream `st`: dpb_export_before orders it after the picture's writer,
// dpb_export_after after the earlier exports of the surface (whichever streams they ran on), then records the external read
// that later writers wait for.
static int dpb_export_before(Dpb& d, int name, cudaStream_t st)
{
  const SlotSync& ss = d.sync[d.lmap[name]];
  if (ss.writer >= 0) CU(cudaStreamWaitEvent(st, ss.written, 0));
  return B200_OK;
}
static int dpb_export_after(Dpb& d, int name, cudaStream_t st)
{
  SlotSync& ss = d.sync[d.lmap[name]];
  if (ss.ext_pending) CU(cudaStreamWaitEvent(st, ss.ext_read, 0));
  CU(cudaEventRecord(ss.ext_read, st));
  ss.ext_pending = true;
  return B200_OK;
}

// A read of the picture named `name` issued on stream `k`: later writers on other streams wait for it.
static int dpb_mark_read(Dpb& d, int name, int k, cudaStream_t st)
{
  SlotSync& ss = d.sync[d.lmap[name]];
  CU(cudaEventRecord(ss.read[k], st));
  ss.read_pending[k] = true;
  return B200_OK;
}

// A write of the picture named `name` issued on stream `k` after every earlier access to its surface, exports included
// (dpb_order_before, or a full synchronise with dpb_wait_exports).
static int dpb_mark_written(Dpb& d, int name, int k, cudaStream_t st)
{
  SlotSync& ss = d.sync[d.lmap[name]];
  CU(cudaEventRecord(ss.written, st));
  ss.writer = k;
  for (auto& rp : ss.read_pending) rp = false;  // later accesses wait for this write instead
  ss.ext_pending = false;
  return B200_OK;
}

// After a picture issued on stream `k`: its reads of the references (`record_reads`: more than one stream may need them) and
// its write.
static int dpb_order_after(Dpb& d, int k, cudaStream_t st, uint32_t ref_mask, int dst, bool record_reads)
{
  for (int r = 0; r < B200_MAX_SLOTS && record_reads; r++) {
    if (!((ref_mask >> r) & 1) || r == dst || d.lmap[r] < 0) continue;
    const int rc = dpb_mark_read(d, r, k, st);
    if (rc) return rc;
  }
  return dpb_mark_written(d, dst, k, st);
}

// The stream a read-back of the name goes on: its last writer's (ordered after the write without an event), else stream 0.
static int dpb_read_stream(const Dpb& d, int name)
{
  const int ph = d.lmap[name];
  return ph >= 0 && d.sync[ph].writer >= 0 ? d.sync[ph].writer : 0;
}

// What the host waits for before it touches the picture named `name`: the write of the surface that carries the name, and the
// reads and exports pending on it and on surfaces that carried the name before (a read-back requested from them may still be in
// flight).
static void dpb_wait_events(const Dpb& d, int name, std::vector<cudaEvent_t>& evs)
{
  for (int ph = 0; ph < B200_MAX_PHYS; ph++) {
    const bool current = d.lmap[name] == ph;
    if (!current && !(d.owner[ph] < 0 && d.last_owner[ph] == name)) continue;
    if (current && d.sync[ph].writer >= 0) evs.push_back(d.sync[ph].written);
    for (int c = 0; c < B200_MAX_CTX; c++)
      if (d.sync[ph].read_pending[c]) evs.push_back(d.sync[ph].read[c]);
    if (d.sync[ph].ext_pending) evs.push_back(d.sync[ph].ext_read);
  }
}

// After every stream was synchronised and dpb_wait_exports: nothing is in flight.
static void dpb_forget_pending(Dpb& d)
{
  for (auto& ss : d.sync) {
    ss.writer = -1;
    for (auto& r : ss.read_pending) r = false;
  }
}
