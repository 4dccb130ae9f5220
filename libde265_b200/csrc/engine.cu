// engine.cu — host side of the B200 reconstruction engine (b200hevc.h part 2) + kernel launches.
//
// Per picture: validate the records, build the work lists (MC units, k_residual classes, intra tasks in topological
// order) and pack everything into one pinned staging buffer on a small host thread pool (planner.cuh), ONE host->device copy, then
//   k_inter_pred8 -> k_residual -> k_mark_pending + k_intra -> k_deblock<V> -> k_deblock<H> -> k_sao_prep + k_sao
// on one of the engine's streams; pictures are pipelined over the streams with per-slot event ordering.
// Reference pictures never leave the device (DPB slots are device surfaces).
// There is no CPU fallback: without a CUDA device b200_engine_create fails with B200_ERR_NO_DEVICE.

#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "b200hevc.h"
#include "dev_common.cuh"
#include "kernels_filter.cuh"
#include "kernels_mc.cuh"
#include "kernels_mc8.cuh"
#include "kernels_mct.cuh"
#include "kernels_recon.cuh"

// ---- error reporting -----------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int set_err(int code, const char* fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
extern "C" const char* b200_last_error(void) { return g_err; }

#define CU(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) return set_err(B200_ERR_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static inline double prof_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

#define B200_MAX_CTX 12  // pipeline streams (PipeCtx)
#include "dpb.cuh"
#include "export.cuh"

// ---- engine --------------------------------------------------------------------------------------
struct StagingSet {
  uint8_t* host = nullptr;  // pinned
  uint8_t* dev = nullptr;
  size_t cap = 0;
  cudaEvent_t done = nullptr;  // recorded after the last kernel that reads `dev`
  bool in_flight = false;
  std::atomic<size_t>* cap_hint = nullptr;  // the owning engine's largest capacity so far (ensure_staging)
};

// A few host threads for the per-picture host work (validation / work-list building of the PUs next to that of the TUs,
// copying the record arrays into the pinned staging buffer): submit_picture is host-bound on large pictures otherwise.
struct HostPool {
  // Jobs belong to a group; wait(group) returns when that group's jobs are done, so several planners (the engine's and the
  // asynchronous ones) can share one pool.
  struct Group { int pending = 0; };
  std::vector<std::thread> th;
  std::mutex m;
  std::condition_variable cv, done_cv;
  std::deque<std::pair<Group*, std::function<void()>>> q;
  bool stop = false;
  void start(int n)
  {
    for (int i = 0; i < n; i++)
      th.emplace_back([this] {
        for (;;) {
          std::pair<Group*, std::function<void()>> job;
          {
            std::unique_lock<std::mutex> lk(m);
            cv.wait(lk, [this] { return stop || !q.empty(); });
            if (stop && q.empty()) return;
            job = std::move(q.front());
            q.pop_front();
          }
          job.second();
          {
            std::lock_guard<std::mutex> lk(m);
            if (--job.first->pending == 0) done_cv.notify_all();
          }
        }
      });
  }
  void run(Group* g, std::function<void()> f)
  {
    if (th.empty()) { f(); return; }
    {
      std::lock_guard<std::mutex> lk(m);
      q.emplace_back(g, std::move(f));
      g->pending++;
    }
    cv.notify_one();
  }
  void wait(Group* g)
  {
    std::unique_lock<std::mutex> lk(m);
    done_cv.wait(lk, [g] { return g->pending == 0; });
  }
  ~HostPool()
  {
    {
      std::lock_guard<std::mutex> lk(m);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : th) t.join();
  }
};

#include "planner.cuh"
#include "submit_queue.cuh"

// One pipeline context = one CUDA stream with everything a picture in flight needs privately.  Pictures are issued
// round-robin onto the contexts; cross-context ordering comes from per-surface events (Dpb, dpb.cuh): a picture waits for
// the writers of its reference slots and for every earlier reader / writer of its destination slot.  So pictures that do
// not depend on each other (the B pictures of one hierarchy level, the next intra period's I picture) overlap, and a
// latency-bound kernel (the intra DAG) of one picture leaves the SMs to the others.
#define B200_STAGE_SETS 40
struct PipeCtx {
  cudaStream_t stream = nullptr;
  Surface scratch;              // pre-SAO picture
  uint8_t* sync_buf = nullptr;  // [256 B ticket | pending map Y | Cb | Cr | SAO masks]
  size_t sync_cap = 0;
  cudaEvent_t tail = nullptr;   // b200_engine_join
};

struct b200_engine {
  int device = 0;
  std::atomic<size_t> stage_cap_hint{0};
  std::mutex issue_m;  // held by the asynchronous sequencer while it issues a command (it mutates the Dpb / stream state b200_engine_wait_slot reads)
  std::unique_ptr<SubmitQueue> async;  // b200_engine_submit_picture_async (created on first use)
  std::unique_ptr<Planner[]> async_planners;  // one per planner thread of `async`
  PipeCtx ctx[B200_MAX_CTX];
  // Record staging: pinned host buffer + device arena per picture in flight, handed out round-robin whatever stream the picture
  // runs on (a set is reused when the kernels of the picture that used it B200_STAGE_SETS pictures ago have finished)
  StagingSet stage_pool[B200_STAGE_SETS];
  unsigned next_stage = 0;
  int n_ctx = 1, next_ctx = 0;
  Dpb dpb;  // the DPB slots' surfaces and their cross-stream ordering
  int intra_width_pct = 0;  // off: warps beyond the DAG's width still pay (they run the dependency-free part of later levels ahead: measured)
  bool sao_legacy = false;  // B200_SAO_LEGACY=1: k_sao for 8-bit pictures too
  HostPool pool;
  Planner planner;  // b200_engine_submit_picture / _prepare_picture, every picture on `pool`
  int num_sms = 132;
  long long slot_depth[B200_MAX_SLOTS] = {}, tail_depth[B200_MAX_CTX] = {}, key_depth = 0;  // pick_ctx: dependency depths
  bool sched_rr = false;        // B200_SCHED=rr: plain round-robin placement (A/B measurements)
  int n_ind = 2, next_ind = 0, ind_run = 0;  // streams for pictures that read no reference (intra pictures), used round-robin (B200_IND_STREAMS)
  int intra_i_grid = 64;        // grid cap of k_intra for such pictures: the DAG is at most ~160 tasks wide, 64 CTAs (512 warps) cover it and leave the other SMs to the P/B pictures (0: one CTA per SM; B200_INTRA_I_GRID)
  unsigned int *intra_err = nullptr, *intra_err_host = nullptr;  // k_intra gave up a dependency wait (device word; mapped host copy)
  unsigned long long spin_limit_ns = 2000000000ull;              // B200_INTRA_SPIN_LIMIT_MS
  int intra_ctas = 3, poll_ns = 256;  // k_intra: persistent CTAs per SM, back-off cap of the flag polling (B200_INTRA_CTAS / B200_POLL_NS)
  // B200_TIMELINE=<file>: a CUDA event before and after every launch; the intervals of all streams (ms since the first launch)
  // are appended to the file at b200_engine_sync / destroy: which kernels of which pictures really overlap (tools/timeline.py)
  struct TlEntry { cudaEvent_t e0, e1; const char* name; int poc, ctx; };
  std::vector<TlEntry> tl;
  const char* tl_path = nullptr;
  cudaEvent_t tl_base = nullptr;
  int mc_ctas = 3;         // k_inter_pred_tma: persistent CTAs per SM (B200_MC_CTAS)
  bool timing = false;
  std::vector<cudaEvent_t> tev;  // timing ring: TIMING_RING pictures x 7 events
  unsigned tcount = 0;           // pictures recorded since enable / reset
  cudaEvent_t* ev = nullptr;     // events of the picture being submitted
  uint64_t launches = 0;
  // B200_HOST_PROF=1 prints at destroy: submit_picture's host time (after the first B200_HOST_PROF_SKIP pictures) ...
  double host_validate = 0, host_plan = 0, host_launch = 0;  // validate + staging wait, plan + pack, launches
  uint64_t host_n = 0;
  int host_skip = 0;  // B200_HOST_PROF_SKIP: warm-up pictures left, counted down by both paths (the queue's sequencer while it runs)
  // ... and run_layout's segments of the pictures the asynchronous queue profiles
  double seg_surfaces = 0, seg_order_before = 0, seg_kernels = 0, seg_order_after = 0;  // surfaces + H2D copy, order_before, kernels, border + order_after
};

#define TIMING_RING 256

static void tl_begin(b200_engine* en, cudaStream_t st, const char* name, int poc, int ctx)
{
  b200_engine::TlEntry e{nullptr, nullptr, name, poc, ctx};
  cudaEventCreate(&e.e0);
  cudaEventCreate(&e.e1);
  if (!en->tl_base) { cudaEventCreate(&en->tl_base); cudaEventRecord(en->tl_base, st); }
  cudaEventRecord(e.e0, st);
  en->tl.push_back(e);
}
static void tl_end(b200_engine* en, cudaStream_t st) { cudaEventRecord(en->tl.back().e1, st); }
static void tl_flush(b200_engine* en)  // after all streams were synchronised
{
  if (!en->tl_path || en->tl.empty()) return;
  if (FILE* f = fopen(en->tl_path, "a")) {
    for (auto& e : en->tl) {
      float t0 = 0, t1 = 0;
      cudaEventElapsedTime(&t0, en->tl_base, e.e0);
      cudaEventElapsedTime(&t1, en->tl_base, e.e1);
      fprintf(f, "%d %s %d %.4f %.4f\n", e.ctx, e.name, e.poc, t0, t1);
    }
    fclose(f);
  }
  for (auto& e : en->tl) { cudaEventDestroy(e.e0); cudaEventDestroy(e.e1); }
  en->tl.clear();
}
#define TL(name, launch)                                                              \
  do {                                                                                \
    if (en->tl_path) tl_begin(en, st, name, L.params.poc, (int)(&cx - en->ctx));      \
    launch;                                                                           \
    if (en->tl_path) tl_end(en, st);                                                  \
  } while (0)

struct b200_prepared {
  uint8_t* dev = nullptr;
  PicLayout L;
};

static bool g_tables_ready[64] = {};

static int init_tables(int device)
{
  if (device < 64 && g_tables_ready[device]) return B200_OK;
  // HEVC core transform: mat[k][n] = +-T((2n+1)k mod 128) with T = first matrix column (cosine symmetry);
  // the 32 base magnitudes are the transform's definition (fallback-dct.cc:512-545 column 0).
  static const int8_t T[33] = {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                               61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9,  4,  0};
  int8_t m[32][32];
  for (int k = 0; k < 32; k++)
    for (int n = 0; n < 32; n++) {
      int j = ((2 * n + 1) * k) % 128, sign = 1;
      if (j > 64) j = 128 - j;
      if (j > 32) { j = 64 - j; sign = -1; }
      m[k][n] = (int8_t)(sign * T[j]);
    }
  CU(cudaMemcpyToSymbol(c_dct, m, sizeof(m)));
  {  // packed transform matrices of the sub-warp residual paths (kernels_residual.cuh): 4 rows of one column per word
    static ResTables rt;
    auto col4 = [&](int nT, int jq, int i) {
      uint32_t w = 0;
      for (int b = 0; b < 4; b++) w |= (uint32_t)(uint8_t)m[(32 / nT) * (4 * jq + b)][i] << (8 * b);
      return w;
    };
    for (int i = 0; i < 4; i++) rt.m4[i] = col4(4, 0, i);
    for (int jq = 0; jq < 2; jq++) for (int i = 0; i < 8; i++) rt.m8[jq][i] = col4(8, jq, i);
    for (int jq = 0; jq < 4; jq++) for (int i = 0; i < 16; i++) rt.m16[jq][i] = col4(16, jq, i);
    for (int jq = 0; jq < 8; jq++) for (int i = 0; i < 32; i++) rt.m32[jq][i] = col4(32, jq, i);
    // DST-VII: M[j][i] = round(128 * 2/3 * sin((2j+1)(i+1)pi/9)) (fallback-dct.cc:260-265 holds the same 16 numbers)
    for (int i = 0; i < 4; i++) {
      uint32_t w = 0;
      for (int j = 0; j < 4; j++) w |= (uint32_t)(uint8_t)(int8_t)lround(128.0 * 2.0 / 3.0 * sin((2 * j + 1) * (i + 1) * M_PI / 9.0)) << (8 * j);
      rt.dst4[i] = w;
    }
    CU(cudaMemcpyToSymbol(c_res, &rt, sizeof(rt)));
  }
  {  // packed tap tables of the 8-bit MC kernels (kernels_mc8.cuh mc8_build_tables)
    static Mc8Tables tb;
    mc8_build_tables(tb);
    CU(cudaMemcpyToSymbol(c_mc8, &tb, sizeof(tb)));
  }
  {  // prediction plans of k_intra's small-TU fast path (kernels_recon.cuh)
    static uint32_t plan[INTRA_PLAN_CLASSES][64];
    for (int c = 0; c < INTRA_PLAN_CLASSES; c++)
      for (int lane = 0; lane < 32; lane++) {
        uint32_t w[2];
        intra_plan_words(c, lane, w);
        plan[c][lane] = w[0];
        plan[c][lane + 32] = w[1];
      }
    CU(cudaMemcpyToSymbol(g_intra_plan, plan, sizeof(plan)));
  }
  if (device < 64) g_tables_ready[device] = true;
  return B200_OK;
}

extern "C" int b200_engine_create(b200_engine** out, int device)
{
  if (!out) return set_err(B200_ERR_INVALID, "null out");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return set_err(B200_ERR_NO_DEVICE, "no CUDA device available (%s); the B200 engine has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= n) return set_err(B200_ERR_INVALID, "device %d out of range (0..%d)", device, n - 1);
  CU(cudaSetDevice(device));
  b200_engine* en = new (std::nothrow) b200_engine();
  if (!en) return set_err(B200_ERR_NOMEM, "out of memory");
  en->device = device;
  int rc = init_tables(device);
  if (rc) { delete en; return rc; }
  en->n_ctx = 8;
  {
    int nt = 8;
    if (const char* e = getenv("B200_HOST_THREADS")) nt = std::max(0, std::min(16, atoi(e)));
    en->pool.start(nt);
  }
  en->planner.opt = plan_options_from_env();
  en->planner.pool = &en->pool;
  if (const char* e = getenv("B200_INTRA_CTAS")) en->intra_ctas = std::max(1, std::min(4, atoi(e)));
  if (const char* e = getenv("B200_SCHED")) en->sched_rr = !strcmp(e, "rr");
  if (const char* e = getenv("B200_IND_STREAMS")) en->n_ind = std::max(1, std::min(4, atoi(e)));
  if (const char* e = getenv("B200_INTRA_I_GRID")) en->intra_i_grid = std::max(0, atoi(e));
  if (const char* e = getenv("B200_INTRA_WIDTH_PCT")) en->intra_width_pct = std::max(0, atoi(e));
  if (const char* e = getenv("B200_SAO_LEGACY")) en->sao_legacy = atoi(e) != 0;
  if (const char* e = getenv("B200_POLL_NS")) en->poll_ns = std::max(32, std::min(100000, atoi(e)));
  if (const char* e = getenv("B200_INTRA_SPIN_LIMIT_MS")) en->spin_limit_ns = 1000000ull * (unsigned long long)std::max(1, std::min(60000, atoi(e)));
  en->tl_path = getenv("B200_TIMELINE");
  if (const char* e = getenv("B200_HOST_PROF_SKIP")) en->host_skip = std::max(0, atoi(e));
  if (const char* e = getenv("B200_MC_CTAS")) en->mc_ctas = std::max(1, std::min(8, atoi(e)));
  if (const char* e = getenv("B200_STREAMS")) en->n_ctx = std::max(1, std::min(B200_MAX_CTX, atoi(e)));
  for (int k = 0; k < B200_MAX_CTX; k++) {
    PipeCtx& cx = en->ctx[k];
    CU(cudaStreamCreateWithFlags(&cx.stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&cx.tail, cudaEventDisableTiming));
  }
  for (auto& st : en->stage_pool) {
    CU(cudaEventCreateWithFlags(&st.done, cudaEventDisableTiming | cudaEventBlockingSync));
    st.cap_hint = &en->stage_cap_hint;
  }  // planner threads sleep, not spin, on a busy set
  CU(cudaMalloc(&en->intra_err, 256));
  CU(cudaMemset(en->intra_err, 0, 256));
  CU(cudaHostAlloc(&en->intra_err_host, 64, cudaHostAllocMapped));
  *en->intra_err_host = 0;
  rc = dpb_init(en->dpb);
  if (rc) return rc;
  CU(cudaFuncSetAttribute(k_inter_pred_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MctShared)));
  CU(cudaFuncSetAttribute(k_intra<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(IntraSmem<uint8_t>)));
  CU(cudaFuncSetAttribute(k_intra<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(IntraSmem<uint16_t>)));
  CU(cudaDeviceGetAttribute(&en->num_sms, cudaDevAttrMultiProcessorCount, device));
  *out = en;
  return B200_OK;
}

extern "C" void b200_engine_destroy(b200_engine* en)
{
  if (!en) return;
  cudaSetDevice(en->device);
  if (en->async) en->async->stop();
  cudaDeviceSynchronize();
  tl_flush(en);
  if (en->tl_base) cudaEventDestroy(en->tl_base);
  dpb_destroy(en->dpb, getenv("B200_HOST_PROF") != nullptr);  // prints the first line of B200_HOST_PROF's report
  if (getenv("B200_HOST_PROF") && en->async && en->async->prof.pictures) {
    const SubmitQueue::Prof& a = en->async->prof;
    const unsigned long long n = a.pictures;
    fprintf(stderr, "[b200] submit_picture_async host ms/picture over %llu pictures: planner busy (all threads) %.3f | sequencer: waiting for a plan %.3f  "
            "pictures %.3f (surfaces+H2D %.3f  order_before %.3f  kernels %.3f  borders+order_after %.3f)  read-backs %.3f\n",
            n, 1e3 * a.plan_busy / n, 1e3 * a.wait_plan / n, 1e3 * a.issue_pictures / n, 1e3 * en->seg_surfaces / n, 1e3 * en->seg_order_before / n,
            1e3 * en->seg_kernels / n, 1e3 * en->seg_order_after / n, 1e3 * a.issue_reads / n);
  }
  if (getenv("B200_HOST_PROF") && en->host_n)
    fprintf(stderr, "[b200] submit_picture host ms/picture over %llu pictures: validate+staging-wait %.3f  plan+pack (threaded) %.3f  launch %.3f\n",
            (unsigned long long)en->host_n, 1e3 * en->host_validate / en->host_n, 1e3 * en->host_plan / en->host_n, 1e3 * en->host_launch / en->host_n);
  for (auto& cx : en->ctx) {
    surface_free(cx.scratch);
    if (cx.sync_buf) cudaFree(cx.sync_buf);
    if (cx.tail) cudaEventDestroy(cx.tail);
    if (cx.stream) cudaStreamDestroy(cx.stream);
  }
  for (auto& st : en->stage_pool) {
    if (st.host) cudaFreeHost(st.host);
    if (st.dev) cudaFree(st.dev);
    if (st.done) cudaEventDestroy(st.done);
  }
  for (auto& e : en->tev)
    if (e) cudaEventDestroy(e);
  if (en->intra_err) cudaFree(en->intra_err);
  if (en->intra_err_host) cudaFreeHost(en->intra_err_host);
  delete en;
}

extern "C" void* b200_engine_stream(b200_engine* en) { return en ? (void*)en->ctx[0].stream : nullptr; }

// After a synchronisation point: did k_intra give up a dependency wait (ReconArgs::err)?  Reported once, then cleared.
static int check_intra_err(b200_engine* en)
{
  if (!en->intra_err_host || !*(volatile unsigned int*)en->intra_err_host) return B200_OK;
  const unsigned int t = *(volatile unsigned int*)en->intra_err_host - 1;
  for (int k = 0; k < B200_MAX_CTX; k++) cudaStreamSynchronize(en->ctx[k].stream);
  *(volatile unsigned int*)en->intra_err_host = 0;
  cudaMemset(en->intra_err, 0, sizeof(unsigned int));
  return set_err(B200_ERR_INVALID, "intra task %u: a neighbour named by the avail bits is never reconstructed before it (dependency wait gave up); picture damaged", t);
}

static int sync_all(b200_engine* en)
{
  for (int k = 0; k < B200_MAX_CTX; k++) CU(cudaStreamSynchronize(en->ctx[k].stream));
  const int rc = dpb_wait_exports(en->dpb);  // fill_slot / upload_slot write behind sync_all without an event
  if (rc) return rc;
  tl_flush(en);
  dpb_forget_pending(en->dpb);
  return check_intra_err(en);
}

// The prologue of the entry points that act after everything queued so far (the synchronous paths keep submission order with
// the queued pictures): select the device and flush the queue.  Returns (and clears) the first error of a queued command.
static int flush_queue(b200_engine* en) { return en->async ? en->async->wait(SubmitQueue::all) : B200_OK; }
static int flushed(b200_engine* en)
{
  CU(cudaSetDevice(en->device));
  return flush_queue(en);
}

extern "C" int b200_engine_set_streams(b200_engine* en, int n)
{
  if (!en || n < 1 || n > B200_MAX_CTX) return set_err(B200_ERR_INVALID, "stream count must be 1..%d", B200_MAX_CTX);
  int rc = flushed(en);
  if (!rc) rc = sync_all(en);
  if (rc) return rc;
  en->n_ctx = n;
  en->next_ctx = 0;
  en->next_ind = 0;
  return B200_OK;
}

// Makes stream 0 (b200_engine_stream) wait for everything issued so far on the other streams: an event recorded on
// stream 0 afterwards marks the completion of all submitted pictures.
extern "C" int b200_engine_join(b200_engine* en)
{
  if (!en) return set_err(B200_ERR_INVALID, "null engine");
  const int rc = flushed(en);
  if (rc) return rc;
  for (int k = 1; k < B200_MAX_CTX; k++) {
    CU(cudaEventRecord(en->ctx[k].tail, en->ctx[k].stream));
    CU(cudaStreamWaitEvent(en->ctx[0].stream, en->ctx[k].tail, 0));
  }
  return B200_OK;
}
extern "C" uint64_t b200_engine_launch_count(const b200_engine* en) { return en ? en->launches : 0; }

extern "C" int b200_engine_enable_timing(b200_engine* en, int on)
{
  if (!en) return set_err(B200_ERR_INVALID, "null engine");
  CU(cudaSetDevice(en->device));
  if (on && en->tev.empty()) {
    en->tev.assign((size_t)TIMING_RING * 7, nullptr);
    for (auto& e : en->tev) CU(cudaEventCreate(&e));
  }
  en->timing = on != 0;
  en->tcount = 0;
  return B200_OK;
}

static int timing_of(b200_engine* en, unsigned idx, float ms[6])
{
  cudaEvent_t* ev = &en->tev[(size_t)(idx % TIMING_RING) * 7];
  CU(cudaEventSynchronize(ev[6]));
  for (int i = 0; i < 5; i++) CU(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
  CU(cudaEventElapsedTime(&ms[5], ev[0], ev[6]));
  return B200_OK;
}

extern "C" int b200_engine_last_timing(b200_engine* en, float ms[6])
{
  if (!en || !ms) return set_err(B200_ERR_INVALID, "null argument");
  if (!en->timing || en->tcount == 0) return set_err(B200_ERR_INVALID, "no timed picture yet");
  CU(cudaSetDevice(en->device));
  return timing_of(en, en->tcount - 1, ms);
}

extern "C" int b200_engine_timing_sum(b200_engine* en, float ms[6], int* n_pictures, int reset)
{
  if (!en || !ms || !n_pictures) return set_err(B200_ERR_INVALID, "null argument");
  CU(cudaSetDevice(en->device));
  for (int i = 0; i < 6; i++) ms[i] = 0;
  const unsigned n = en->timing ? (en->tcount < TIMING_RING ? en->tcount : TIMING_RING) : 0;
  for (unsigned k = 0; k < n; k++) {
    float one[6];
    int rc = timing_of(en, en->tcount - 1 - k, one);
    if (rc) return rc;
    for (int i = 0; i < 6; i++) ms[i] += one[i];
  }
  *n_pictures = (int)n;
  if (reset) en->tcount = 0;
  return B200_OK;
}

static DevPic make_devpic(const b200_pic_params& p, const Surface& cur, const Surface& out)
{
  DevPic d{};
  d.w = p.width; d.h = p.height;
  d.cw = cur.cw; d.ch = cur.ch;
  d.bd_y = p.bit_depth_luma; d.bd_c = p.bit_depth_chroma;
  d.log2ctb = p.log2_ctb_size;
  const int S = 1 << d.log2ctb;
  d.wctb = (p.width + S - 1) / S; d.hctb = (p.height + S - 1) / S;
  d.w4 = (p.width + 3) / 4; d.h4 = (p.height + 3) / 4;
  d.w8 = (p.width + 7) / 8; d.h8 = (p.height + 7) / 8;
  d.chroma = p.chroma_format_idc;
  d.cb_qp_off = p.pps_cb_qp_offset; d.cr_qp_off = p.pps_cr_qp_offset;
  d.flags = p.flags;
  for (int c = 0; c < 3; c++) { d.cur[c] = cur.plane[c]; d.out[c] = out.plane[c]; d.pitch[c] = cur.pitch[c]; }
  return d;
}

// sync_buf layout: [256 B ticket | pending map Y | Cb | Cr | (256-aligned) SAO neighbour-availability masks]
static size_t sync_sao_offset(const b200_pic_params& p)
{
  const size_t cw4 = p.chroma_format_idc ? (size_t)((p.width / 2 + 3) / 4) : 0, ch4 = p.chroma_format_idc ? (size_t)((p.height / 2 + 3) / 4) : 0;
  return (256 + (size_t)((p.width + 3) / 4) * ((p.height + 3) / 4) + 2 * cw4 * ch4 + 255) & ~(size_t)255;
}

template <typename P>
static int launch_picture(b200_engine* en, PipeCtx& cx, const PicLayout& L, const DevPic& dp, const RefTable& refs, const uint8_t* dbase)
{
  cudaStream_t st = cx.stream;
  const size_t* off = L.off;
  const int n_tiles = L.n_tiles;
  const bool run_deblock = L.run_deblock, run_sao = L.run_sao;
  if (en->timing) CU(cudaEventRecord(en->ev[1], st));
  if (n_tiles > 0) {
    if (L.mc_units == MC_CLASS_BATCHES) {
      // reference windows staged by TMA: the tensor maps of the slots this picture reads travel as a kernel parameter
      MctMaps maps;
      memset(&maps, 0, sizeof(maps));
      int n = 0;
      for (int i = 0; i < B200_MAX_SLOTS; i++) {
        maps.index_of_slot[i] = -1;
        if (!((L.ref_mask >> i) & 1) || !refs.plane[i][0]) continue;  // a reference in the table holds a picture
        const Surface& s = *dpb_picture(en->dpb, i);
        if (!s.has_tm) continue;
        if (n == MCT_MAX_REFS) return set_err(B200_ERR_UNSUPPORTED, "picture references more than %d DPB slots", MCT_MAX_REFS);
        for (int k = 0; k < 2; k++) { maps.luma[k][n] = s.tm_luma[k]; maps.chroma[k][n] = s.tm_chroma[k]; }
        maps.index_of_slot[i] = (int8_t)n++;
        maps.valid_slots |= 1u << i;
      }
      const uint32_t* tw = (const uint32_t*)(dbase + off[12]);  // tile words, then the batch table
      TL("mc", (k_inter_pred_tma<<<std::min(L.n_batches, en->num_sms * en->mc_ctas), MCT_CTA_THREADS, sizeof(MctShared), st>>>(
                   dp, maps, (const b200_pu*)(dbase + off[0]), (const b200_weight_entry*)(dbase + off[1]), tw, tw + n_tiles, L.n_batches)));
    } else if (L.mc_units == MC_UNITS8x16)
      k_inter_pred8<<<std::min((n_tiles + MC8_UNITS_PER_CTA - 1) / MC8_UNITS_PER_CTA, en->num_sms * 5), MC8_WARPS * 32, 0, st>>>(dp, refs, (const b200_pu*)(dbase + off[0]), (const b200_weight_entry*)(dbase + off[1]),
                                                         (const uint32_t*)(dbase + off[12]), n_tiles);
    else
      k_inter_pred<P><<<(n_tiles + 3) / 4, 128, 0, st>>>(dp, refs, (const b200_pu*)(dbase + off[0]), (const b200_weight_entry*)(dbase + off[1]),
                                                           (const uint32_t*)(dbase + off[12]), n_tiles);
    en->launches++;
  }
  if (en->timing) CU(cudaEventRecord(en->ev[2], st));
  if ((L.n_a > 0 || L.n_b > 0) && L.params.stop_after_stage != B200_STAGE_INTER_PRED) {
    ReconArgs ra;
    ra.tus = (const b200_tu*)(dbase + off[2]);
    ra.coeffs = (const b200_coeff*)(dbase + off[5]);
    ra.scaling = L.has_scaling ? dbase + off[11] : nullptr;
    ra.ticket = (unsigned int*)cx.sync_buf;
    ra.region = L.region;
    ra.poll_ns = en->poll_ns;
    ra.err = en->intra_err;
    ra.err_host = en->intra_err_host;
    ra.spin_limit_ns = en->spin_limit_ns;
    const size_t cw4 = (size_t)((dp.cw + 3) / 4), ch4 = (size_t)((dp.ch + 3) / 4);
    ra.pend[0] = cx.sync_buf + 256;
    ra.pend[1] = ra.pend[0] + (size_t)dp.w4 * dp.h4;
    ra.pend[2] = ra.pend[1] + cw4 * ch4;
    ra.pend_w[0] = dp.w4;
    ra.pend_w[1] = ra.pend_w[2] = (int)cw4;
    ra.mark_list = nullptr;
    ra.n_mark = 0;
    if (L.n_b > 0) CU(cudaMemsetAsync(cx.sync_buf, 0, 256 + (size_t)dp.w4 * dp.h4 + 2 * cw4 * ch4, st));  // ticket + pending flags
    if (L.n_a > 0) {
      ra.list = (const uint32_t*)(dbase + off[3]);
      ra.n_list = L.n_a;
      ra.n_listw = L.n_aw;
      ra.n_list8 = L.n_a8;
      if (L.n_b > 0) {  // k_residual also sets the pending flags of the intra TUs
        ra.mark_list = (const uint32_t*)(dbase + off[4]);
        ra.n_mark = L.n_b;
      }
      const int items = L.n_aw + (L.n_a8 + 3) / 4 + (L.n_a - L.n_aw - L.n_a8 + 31) / 32;
      TL("residual", (k_residual<P><<<std::min((items + RC_WARPS - 1) / RC_WARPS, en->num_sms * 4), RC_THREADS, 0, st>>>(dp, ra)));
      en->launches++;
    }
    ra.trace = nullptr;
    if (L.n_b > 0) {
      unsigned long long* trace_dev = nullptr;
      const char* trace_path = getenv("B200_TRACE_INTRA");  // debug: per-task timing trace of k_intra appended to this file
      if (trace_path && L.n_task > 0) {
        CU(cudaMalloc(&trace_dev, sizeof(unsigned long long) * RC_TRACE_WORDS * (size_t)L.n_task));
        CU(cudaMemsetAsync(trace_dev, 0, sizeof(unsigned long long) * RC_TRACE_WORDS * (size_t)L.n_task, st));
        ra.trace = trace_dev;
      }
      ra.list = (const uint32_t*)(dbase + off[4]);
      ra.n_list = L.n_b;
      if (L.n_a == 0) {
        TL("mark", (k_mark_pending<<<(L.n_b + 255) / 256, 256, 0, st>>>(ra)));
        en->launches++;
      }
      ra.task_start = (const uint32_t*)(dbase + off[13]);
      ra.n_task = L.n_task;
      int grid = (L.n_task + RC_WARPS - 1) / RC_WARPS;
      // an intra picture's DAG is latency-bound (one CTA per SM is as fast) and should leave room for the pictures it overlaps with
      const bool background = L.ref_mask == 0 && en->n_ctx > 1;
      int cap = background ? (en->intra_i_grid ? en->intra_i_grid : en->num_sms) : en->num_sms * en->intra_ctas;
      // tickets in level order: the widest level bounds how many tasks can ever run at once; more warps than that only spin and
      // keep other pictures' CTAs off the SMs (B200_INTRA_WIDTH_PCT: warps per task of the widest level, in percent; 0 = off)
      if (L.intra_width > 0 && en->intra_width_pct > 0)
        cap = std::min(cap, std::max(4, (int)(((long long)L.intra_width * en->intra_width_pct / 100 + RC_WARPS - 1) / RC_WARPS)));
      if (grid > cap) grid = cap;
      TL("intra", (k_intra<P><<<grid, RC_THREADS, sizeof(IntraSmem<P>), st>>>(dp, ra)));
      en->launches++;
      if (trace_dev) {
        // record: n_task, n_list (u64), the per-task stamps, then task_start[n_task + 1] and list[n_list] (u32) so that a reader
        // can rebuild which task produced each neighbour unit
        std::vector<unsigned long long> h(RC_TRACE_WORDS * (size_t)L.n_task);
        std::vector<uint32_t> tasks((size_t)L.n_task + 1 + (size_t)L.n_b);
        CU(cudaStreamSynchronize(st));
        CU(cudaMemcpy(h.data(), trace_dev, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(tasks.data(), ra.task_start, ((size_t)L.n_task + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(tasks.data() + L.n_task + 1, ra.list, (size_t)L.n_b * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        cudaFree(trace_dev);
        if (FILE* f = fopen(trace_path, "ab")) {
          const unsigned long long n[2] = {(unsigned long long)L.n_task, (unsigned long long)L.n_b};
          fwrite(n, sizeof(n), 1, f);
          fwrite(h.data(), sizeof(unsigned long long), h.size(), f);
          fwrite(tasks.data(), sizeof(uint32_t), tasks.size(), f);
          fclose(f);
        }
      }
    }
  }
  if (en->timing) CU(cudaEventRecord(en->ev[3], st));
  FilterArgs fa;
  fa.bs_map = dbase + off[8];
  fa.qp_map = (const int8_t*)(dbase + off[9]);
  fa.nofilt_map = dbase + off[10];
  fa.slices = (const b200_slice_info*)(dbase + off[6]);
  fa.ctbs = (const b200_ctb_info*)(dbase + off[7]);
  if (run_deblock) {
    const int nseg = ((dp.w4 + 1) / 2) * dp.h4 > dp.w4 * ((dp.h4 + 1) / 2) ? ((dp.w4 + 1) / 2) * dp.h4 : dp.w4 * ((dp.h4 + 1) / 2);
    dim3 grid((nseg + 127) / 128, dp.chroma ? 2 : 1);
    TL("deblock_v", (k_deblock<P, true><<<grid, 128, 0, st>>>(dp, fa)));
    TL("deblock_h", (k_deblock<P, false><<<grid, 128, 0, st>>>(dp, fa)));
    en->launches += 2;
  }
  if (en->timing) CU(cudaEventRecord(en->ev[4], st));
  if (run_sao) {
    uint16_t* avail = (uint16_t*)(cx.sync_buf + sync_sao_offset(L.params));
    fa.sao_avail = avail;
    const bool sao8 = sizeof(P) == 1 && dp.log2ctb >= 5 && !en->sao_legacy;
    if (!sao8) {  // k_sao8 derives the neighbour masks itself
      TL("sao_prep", (k_sao_prep<<<(2 * dp.wctb * dp.hctb + 127) / 128, 128, 0, st>>>(dp, fa, avail)));
      en->launches++;
    }
    dim3 grid((dp.w / 8 + 127) / 128, dp.h, dp.chroma ? 3 : 1);
    if (sao8) {  // byte-parallel kernel: a warp per CTB part (kernels_filter.cuh)
      Sao8Layout lay;
      lay.n_ctb = dp.wctb * dp.hctb;
      const int S = 1 << dp.log2ctb, rows_l = (32 >> (dp.log2ctb - 4)) * SAO8_R, rows_c = (32 >> (dp.log2ctb - 5)) * SAO8_R;
      lay.ipl = (S + rows_l - 1) / rows_l;
      lay.ipc = dp.chroma ? (S / 2 + rows_c - 1) / rows_c : 0;
      const int items = lay.n_ctb * (lay.ipl + 2 * lay.ipc);
      TL("sao", (k_sao8<<<(items + SAO8_WARPS - 1) / SAO8_WARPS, SAO8_WARPS * 32, 0, st>>>(dp, fa, lay)));
    } else {
      TL("sao", (k_sao<P><<<grid, 128, 0, st>>>(dp, fa)));
    }
    en->launches++;
  }
  if (en->timing) CU(cudaEventRecord(en->ev[5], st));
  CU(cudaGetLastError());
  return B200_OK;
}

// cap_hint = the largest staging capacity any set of the engine has needed: a set that has to grow goes straight to it, so that
// every set is reallocated at most once after the first large (intra) picture instead of whenever such a picture happens to land
// on it (page-locking tens of MB and cudaFree both stall the other threads' CUDA calls).

static int ensure_staging(StagingSet& ss, size_t total)
{
  if (ss.in_flight) { CU(cudaEventSynchronize(ss.done)); ss.in_flight = false; }
  std::atomic<size_t> local{0};
  std::atomic<size_t>& cap_hint = ss.cap_hint ? *ss.cap_hint : local;
  size_t hint = cap_hint.load(std::memory_order_relaxed);
  const size_t want = align_up(total + total / 2, 1 << 20);
  while (want > hint && !cap_hint.compare_exchange_weak(hint, want, std::memory_order_relaxed)) {}
  if (ss.cap < total) {
    if (ss.host) cudaFreeHost(ss.host);
    if (ss.dev) cudaFree(ss.dev);
    ss.host = nullptr; ss.dev = nullptr;
    ss.cap = std::max(want, cap_hint.load(std::memory_order_relaxed));
    CU(cudaMallocHost(&ss.host, ss.cap));
    CU(cudaMalloc(&ss.dev, ss.cap));
  }
  return B200_OK;
}

// Host side of one picture: validate, build the work lists, fill the pinned staging buffer (plan_build: on the planner's pool).
static int plan_and_pack(Planner& pl, const b200_picture* pic, PicLayout* L, StagingSet& ss, double* t_plan_pack)
{
  const double t0 = prof_now();
  size_t cap = 0;
  int rc = plan_begin(pl, pic, L, &cap);
  if (rc) return rc;
  rc = ensure_staging(ss, cap);
  if (rc) return rc;
  const double t1 = prof_now();
  rc = plan_build(pl, pic, L, ss.host);
  if (rc) return rc;
  if (t_plan_pack) { t_plan_pack[0] = t1 - t0; t_plan_pack[1] = prof_now() - t1; }
  return B200_OK;
}

extern "C" int b200_plan_picture_host(const b200_picture* pic, uint32_t counts[8], uint32_t* mc_units, size_t cap_units, uint32_t* list_a, size_t cap_a,
                                      uint32_t* list_b, size_t cap_b, uint32_t* task_start, size_t cap_tasks)
{
  if (!pic || !counts) return set_err(B200_ERR_INVALID, "null argument");
  Planner pl;  // no pool, no CUDA call
  pl.opt = plan_options_from_env();
  PicLayout L;
  size_t cap = 0;
  int rc = plan_begin(pl, pic, &L, &cap);
  if (!rc) rc = plan_build(pl, pic, &L, nullptr);
  if (rc) return rc;
  counts[0] = (uint32_t)L.n_tiles; counts[1] = (uint32_t)L.n_a; counts[2] = (uint32_t)L.n_aw; counts[3] = (uint32_t)L.n_a8;
  counts[4] = (uint32_t)L.n_b; counts[5] = (uint32_t)L.n_task; counts[6] = L.ref_mask; counts[7] = 0;
  auto copy = [](uint32_t* dst, size_t cap_, const std::vector<uint32_t>& v, size_t n) {
    if (dst) memcpy(dst, v.data(), sizeof(uint32_t) * std::min(cap_, n));
  };
  copy(mc_units, cap_units, pl.tiles, (size_t)L.n_tiles);
  copy(list_a, cap_a, pl.list_a, (size_t)L.n_a);
  copy(list_b, cap_b, pl.list_b, (size_t)L.n_b);
  copy(task_start, cap_tasks, pl.task_start, L.n_task ? (size_t)L.n_task + 1 : 0);
  return B200_OK;
}

// Everything after the records are in device memory at `dbase`.  `upload_from`: pinned source to copy first (or null).
static int run_layout(b200_engine* en, int k, const PicLayout& L, uint8_t* dbase, const uint8_t* upload_from)
{
  PipeCtx& cx = en->ctx[k];
  const b200_pic_params& p = L.params;
  const bool prof = en->async && en->async->profiling();
  double tseg[5] = {prof ? prof_now() : 0.0, 0, 0, 0, 0};
  const RefTable refs = dpb_refs(en->dpb, p);
  cudaStream_t streams[B200_MAX_CTX];
  for (int c = 0; c < B200_MAX_CTX; c++) streams[c] = en->ctx[c].stream;
  int rc = dpb_set_format(en->dpb, p, streams, B200_MAX_CTX);
  if (rc) return rc;
  Surface* dstp = dpb_acquire(en->dpb, p.dst_slot, k, p, en->n_ctx > 1 && !en->timing);
  if (!dstp) {  // first use of the name with every surface taken: cannot happen (B200_MAX_PHYS > B200_MAX_SLOTS), but stay safe
    return set_err(B200_ERR_NOMEM, "no free picture surface");
  }
  Surface& dst = *dstp;
  rc = surface_ensure(dst, p, cx.stream);
  if (rc) return rc;
  Surface* cur = &dst;
  if (L.run_sao) {
    rc = surface_ensure(cx.scratch, p, cx.stream);
    if (rc) return rc;
    cur = &cx.scratch;
  }
  {
    const size_t n_ctb = (size_t)((p.width + (1 << p.log2_ctb_size) - 1) >> p.log2_ctb_size) * ((p.height + (1 << p.log2_ctb_size) - 1) >> p.log2_ctb_size);
    const size_t need = sync_sao_offset(p) + 2 * n_ctb * sizeof(uint16_t);
    if (cx.sync_cap < need) {
      if (cx.sync_buf) { CU(cudaStreamSynchronize(cx.stream)); cudaFree(cx.sync_buf); }
      cx.sync_buf = nullptr;
      CU(cudaMalloc(&cx.sync_buf, need));
      cx.sync_cap = need;
    }
  }
  cudaStream_t st = cx.stream;
  en->ev = en->timing ? &en->tev[(size_t)(en->tcount % TIMING_RING) * 7] : nullptr;
  if (en->timing) CU(cudaEventRecord(en->ev[0], st));
  if (upload_from && L.direct) {  // raw record arrays straight from the caller's page-locked memory, the planner's lists from the staging buffer
    for (int i : k_raw_sections)
      if (L.raw_sz[i]) CU(cudaMemcpyAsync(dbase + L.off[i], L.raw_src[i], L.raw_sz[i], cudaMemcpyHostToDevice, st));
    if (L.total > L.raw_total) CU(cudaMemcpyAsync(dbase + L.raw_total, upload_from + L.raw_total, L.total - L.raw_total, cudaMemcpyHostToDevice, st));
  } else if (upload_from) {
    CU(cudaMemcpyAsync(dbase, upload_from, L.total, cudaMemcpyHostToDevice, st));  // records first: overlaps the waits below
  }
  if (prof) tseg[1] = prof_now();
  rc = dpb_order_before(en->dpb, k, st, L.ref_mask, p.dst_slot);
  if (rc) return rc;
  if (prof) tseg[2] = prof_now();
  const DevPic dp = make_devpic(p, *cur, dst);
  if (p.bit_depth_luma > 8) rc = launch_picture<uint16_t>(en, cx, L, dp, refs, dbase);
  else rc = launch_picture<uint8_t>(en, cx, L, dp, refs, dbase);
  if (rc) return rc;
  if (prof) tseg[3] = prof_now();
  TL("extend", launch_extend_borders(dst, st));  // the finished picture may be referenced: replicate its edges into the border
  en->launches++;
  CU(cudaGetLastError());
  if (en->timing) { CU(cudaEventRecord(en->ev[6], st)); en->tcount++; }
  rc = dpb_order_after(en->dpb, k, st, L.ref_mask, p.dst_slot, en->n_ctx > 1);
  if (rc) return rc;
  dst.valid = true;
  if (prof) {
    tseg[4] = prof_now();
    en->seg_surfaces += tseg[1] - tseg[0];
    en->seg_order_before += tseg[2] - tseg[1];
    en->seg_kernels += tseg[3] - tseg[2];
    en->seg_order_after += tseg[4] - tseg[3];
  }
  return B200_OK;
}

// Per-stage timing needs the stages of consecutive pictures not to overlap: one stream while it is on.
// Pictures that read no reference (intra pictures) go to a stream of their own: nothing queued in front of them, so the
// long intra DAG of the next intra period's I picture runs in the background of the current period's P/B pictures.
//
// The other pictures are placed by DEPENDENCY DEPTH (depth = 1 + the largest depth among the pictures in the slots it reads): a
// stream is a FIFO, so a picture queued behind an unrelated picture that still waits for ITS references is held up for nothing
// (round-robin puts the next GOP's key picture behind the current GOP's leaf B pictures: 16 picture times per 4 GOPs instead
// of 7).  A picture goes to the stream whose last picture has the largest depth still below its own (that picture finishes
// before this one could start anyway); if there is none, to the stream whose last picture is the shallowest.
static int pick_ctx(b200_engine* en, uint32_t ref_mask, int dst_slot)
{
  if (en->timing || en->n_ctx <= 1) return 0;
  long long depth = 1;
  for (int r = 0; r < B200_MAX_SLOTS; r++)
    if ((ref_mask >> r) & 1) depth = std::max(depth, en->slot_depth[r] + 1);
  int k;
  if (ref_mask == 0 && en->n_ctx + en->n_ind <= B200_MAX_CTX) {  // the long intra DAGs of consecutive intra pictures overlap each other too
    // an all-intra stream (several pictures in a row that read no reference) spreads over ALL streams: every picture is a
    // latency-bound DAG on a quarter of the SMs, so many of them fit side by side
    en->ind_run++;
    const int pool = en->ind_run > 2 ? en->n_ctx + en->n_ind : en->n_ind, base = en->ind_run > 2 ? 0 : en->n_ctx;
    k = base + en->next_ind % pool;
    en->next_ind = (en->next_ind + 1) % pool;
    depth = en->key_depth + 1;  // what references it comes after the pictures already queued
  } else if (en->sched_rr) {
    k = en->next_ctx;
    en->next_ctx = (en->next_ctx + 1) % en->n_ctx;
  } else {
    int best = -1, shallow = 0;
    for (int c = 0; c < en->n_ctx; c++) {
      if (en->tail_depth[c] < depth && (best < 0 || en->tail_depth[c] > en->tail_depth[best])) best = c;
      if (en->tail_depth[c] < en->tail_depth[shallow]) shallow = c;
    }
    k = best >= 0 ? best : shallow;
  }
  if (ref_mask != 0) en->ind_run = 0;
  en->tail_depth[k] = depth;
  if (dst_slot >= 0 && dst_slot < B200_MAX_SLOTS) en->slot_depth[dst_slot] = depth;
  en->key_depth = std::max(en->key_depth, depth);
  return k;
}

// Issues a planned picture whose records are at `dbase` (uploaded first from `ss`'s pinned buffer when `ss` is given) on the
// stream pick_ctx chooses; `ss` is busy until the picture's kernels are done.
static int issue_picture(b200_engine* en, const PicLayout& L, uint8_t* dbase, StagingSet* ss)
{
  const int k = pick_ctx(en, L.ref_mask, L.params.dst_slot);
  const int rc = run_layout(en, k, L, dbase, ss ? ss->host : nullptr);
  if (rc) return rc;
  if (ss) {
    CU(cudaEventRecord(ss->done, en->ctx[k].stream));
    ss->in_flight = true;
  }
  return B200_OK;
}

// ---- asynchronous submission (submit_queue.cuh) -----------------------------------------------------------------------------
// Staging sets are handed out round-robin in submission order.  A queued picture's planner writes its set before the picture is
// issued (and the set marked in flight), so the queue must hold fewer pictures than there are sets: then the picture that used
// the set before has been issued, and ensure_staging waits for its kernels.
static_assert(B200_ASYNC_DEPTH < B200_STAGE_SETS, "a staging set would be handed out again before its previous picture was issued");
static StagingSet& next_staging(b200_engine* en) { return en->stage_pool[en->next_stage++ % B200_STAGE_SETS]; }

// A queued picture (its records, layout and staging set) or read-back (where the planes go).
struct QueuedCmd : SubmitCmd {
  b200_picture pic{};
  PicLayout L;
  StagingSet* ss = nullptr;
  void* planes[3] = {nullptr, nullptr, nullptr};
  size_t strides[3] = {0, 0, 0};
};

static int read_slot_async_now(b200_engine* en, int slot, void* const planes[3], const size_t strides[3]);

// Started on first use: an engine that never submits asynchronously starts no threads.  Each planner thread has a Planner of its
// own (the engine's options, private scratch); the sequencer issues under issue_m exactly as the synchronous path does, so
// stream placement, DPB ordering and results are the same.
static int async_start(b200_engine* en)
{
  if (en->async) return B200_OK;
  const int n = SubmitQueue::planner_threads();
  en->async_planners.reset(new (std::nothrow) Planner[n]);
  if (!en->async_planners) return set_err(B200_ERR_NOMEM, "out of memory");
  for (int i = 0; i < n; i++) {
    en->async_planners[i].opt = en->planner.opt;
    // a picture with a long plan (a large intra picture) borrows the engine's pool so that the in-order sequencer is not held up by it
    en->async_planners[i].pool = &en->pool;
    en->async_planners[i].pool_min_tus = 200000;
  }
  en->async.reset(new (std::nothrow) SubmitQueue());
  if (!en->async) return set_err(B200_ERR_NOMEM, "out of memory");
  en->async->plan = [en](int w, SubmitCmd& c) {
    QueuedCmd& q = static_cast<QueuedCmd&>(c);
    return plan_and_pack(en->async_planners[w], &q.pic, &q.L, *q.ss, nullptr);
  };
  en->async->issue = [en](SubmitCmd& c) {
    QueuedCmd& q = static_cast<QueuedCmd&>(c);
    std::lock_guard<std::mutex> issue(en->issue_m);
    return q.kind == CmdKind::picture ? issue_picture(en, q.L, q.ss->dev, q.ss) : read_slot_async_now(en, q.slot, q.planes, q.strides);
  };
  en->async->thread_start = [en] { cudaSetDevice(en->device); };
  en->async->prof_on = getenv("B200_HOST_PROF") != nullptr;
  en->async->prof_skip = &en->host_skip;
  const int rc = en->async->start(n);
  if (rc) en->async.reset();
  return rc;
}

extern "C" int b200_engine_submit_picture_async(b200_engine* en, const b200_picture* pic)
{
  if (!en || !pic) return set_err(B200_ERR_INVALID, "null argument");
  CU(cudaSetDevice(en->device));
  const int rc = async_start(en);
  if (rc) return rc;
  QueuedCmd* cmd = new (std::nothrow) QueuedCmd();
  if (!cmd) return set_err(B200_ERR_NOMEM, "out of memory");
  cmd->slot = pic->params.dst_slot;
  cmd->pic = *pic;  // the record ARRAYS must stay valid until b200_engine_flush / _sync returns
  cmd->ss = &next_staging(en);
  en->async->enqueue(cmd);
  return B200_OK;
}

extern "C" unsigned long long b200_engine_last_ticket(b200_engine* en) { return en && en->async ? en->async->last_ticket() : 0; }

extern "C" int b200_engine_wait_ticket(b200_engine* en, unsigned long long ticket)
{
  if (!en) return set_err(B200_ERR_INVALID, "null engine");
  return en->async ? en->async->wait(ticket) : B200_OK;
}

extern "C" int b200_engine_flush(b200_engine* en)
{
  if (!en) return set_err(B200_ERR_INVALID, "null engine");
  return flush_queue(en);
}

extern "C" int b200_engine_submit_picture(b200_engine* en, const b200_picture* pic)
{
  if (!en || !pic) return set_err(B200_ERR_INVALID, "null argument");
  int rc = flushed(en);
  if (rc) return rc;
  PicLayout L;
  StagingSet& ss = next_staging(en);
  double tp[2] = {0, 0};
  rc = plan_and_pack(en->planner, pic, &L, ss, tp);
  if (rc) return rc;
  const double t3 = prof_now();
  rc = issue_picture(en, L, ss.dev, &ss);
  if (rc) return rc;
  if (en->host_skip > 0) en->host_skip--;  // B200_HOST_PROF_SKIP: leave the warm-up (first-use allocations) out of the profile
  else { en->host_validate += tp[0]; en->host_plan += tp[1]; en->host_launch += prof_now() - t3; en->host_n++; }
  return B200_OK;
}

extern "C" int b200_engine_prepare_picture(b200_engine* en, const b200_picture* pic, b200_prepared** out)
{
  if (!en || !pic || !out) return set_err(B200_ERR_INVALID, "null argument");
  int rc = flushed(en);
  if (rc) return rc;
  b200_prepared* pp = new (std::nothrow) b200_prepared();
  if (!pp) return set_err(B200_ERR_NOMEM, "out of memory");
  PipeCtx& cx = en->ctx[0];
  StagingSet& ss = next_staging(en);
  b200_picture staged = *pic;
  staged.params.flags &= ~B200_PIC_RECORDS_PINNED;  // a prepared picture keeps its own device copy of everything
  rc = plan_and_pack(en->planner, &staged, &pp->L, ss, nullptr);
  if (rc) { delete pp; return rc; }
  cudaError_t e = cudaMalloc(&pp->dev, pp->L.total);
  if (e == cudaSuccess) e = cudaMemcpyAsync(pp->dev, ss.host, pp->L.total, cudaMemcpyHostToDevice, cx.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(cx.stream);
  if (e != cudaSuccess) {
    if (pp->dev) cudaFree(pp->dev);
    delete pp;
    return set_err(B200_ERR_CUDA, "prepare: %s", cudaGetErrorString(e));
  }
  *out = pp;
  return B200_OK;
}

extern "C" int b200_engine_run_prepared(b200_engine* en, b200_prepared* pp)
{
  if (!en || !pp) return set_err(B200_ERR_INVALID, "null argument");
  const int rc = flushed(en);
  return rc ? rc : issue_picture(en, pp->L, pp->dev, nullptr);
}

extern "C" void b200_engine_free_prepared(b200_engine* en, b200_prepared* pp)
{
  if (!en || !pp) return;
  cudaSetDevice(en->device);
  flush_queue(en);
  sync_all(en);
  if (pp->dev) cudaFree(pp->dev);
  delete pp;
}

extern "C" int b200_engine_sync(b200_engine* en)
{
  if (!en) return set_err(B200_ERR_INVALID, "null engine");
  const int rc = flushed(en);
  return rc ? rc : sync_all(en);
}

template <typename P>
__global__ void k_fill(uint8_t* base, int pitch, int w, int h, int value)
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x < w && y < h) row_ptr<P>(base, pitch, y)[x] = (P)value;
}

// The utility writes (fill_slot, upload_slot): check the arguments, quiesce, then take the surface the name `slot` is written to
// on stream 0, allocated in the format of `p`.
static int utility_write_begin(b200_engine* en, int slot, const b200_pic_params* p, Surface** s)
{
  if (!en || !p || slot < 0 || slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "bad argument");
  int rc = check_params(*p);
  if (rc) return rc;
  rc = flushed(en);
  if (!rc) rc = sync_all(en);
  if (rc) return rc;
  *s = dpb_acquire(en->dpb, slot, 0, *p, false);  // everything is idle after sync_all: the name keeps its surface, or gets its first one
  if (!*s) return set_err(B200_ERR_NOMEM, "no free picture surface");
  return surface_ensure(**s, *p, en->ctx[0].stream);
}

extern "C" int b200_engine_fill_slot(b200_engine* en, int slot, const b200_pic_params* p, int vy, int vc)
{
  Surface* sp;
  int rc = utility_write_begin(en, slot, p, &sp);
  if (rc) return rc;
  cudaStream_t st = en->ctx[0].stream;
  Surface& s = *sp;
  for (int c = 0; c < (s.chroma ? 3 : 1); c++) {
    const int w = c ? s.cw : s.w, h = c ? s.ch : s.h;
    dim3 grid((w + 255) / 256, h);
    if (p->bit_depth_luma > 8) k_fill<uint16_t><<<grid, 256, 0, st>>>(s.plane[c], s.pitch[c], w, h, c ? vc : vy);
    else k_fill<uint8_t><<<grid, 256, 0, st>>>(s.plane[c], s.pitch[c], w, h, c ? vc : vy);
    en->launches++;
  }
  launch_extend_borders(s, st);
  en->launches++;
  CU(cudaGetLastError());
  rc = dpb_mark_written(en->dpb, slot, 0, st);
  if (rc) return rc;
  s.valid = true;
  return B200_OK;
}

extern "C" int b200_engine_upload_slot(b200_engine* en, int slot, const b200_pic_params* p, const void* const planes[3], const size_t strides[3])
{
  if (!planes || !strides) return set_err(B200_ERR_INVALID, "bad argument");
  Surface* sp;
  const int rc = utility_write_begin(en, slot, p, &sp);
  if (rc) return rc;
  cudaStream_t st = en->ctx[0].stream;
  Surface& s = *sp;
  for (int c = 0; c < (s.chroma ? 3 : 1); c++) {
    const int w = c ? s.cw : s.w, h = c ? s.ch : s.h, bps = bytes_per_sample(c ? s.bd_c : s.bd_y);
    if (!planes[c]) return set_err(B200_ERR_INVALID, "plane %d missing", c);
    CU(cudaMemcpy2DAsync(s.plane[c], s.pitch[c], planes[c], strides[c], (size_t)w * bps, h, cudaMemcpyHostToDevice, st));
  }
  launch_extend_borders(s, st);
  en->launches++;
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));  // the source may be pageable / reused by the caller
  s.valid = true;
  return B200_OK;
}

extern "C" int b200_engine_read_slot_async(b200_engine* en, int slot, void* const planes[3], const size_t strides[3])
{
  if (!en || !planes || !strides || slot < 0 || slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "bad argument");
  if (en->async) {  // pictures are queued: the read takes its place behind them (the picture it reads may not be launched yet)
    QueuedCmd* cmd = new (std::nothrow) QueuedCmd();
    if (!cmd) return set_err(B200_ERR_NOMEM, "out of memory");
    cmd->kind = CmdKind::read;
    cmd->slot = slot;
    for (int c = 0; c < 3; c++) { cmd->planes[c] = planes[c]; cmd->strides[c] = strides[c]; }
    en->async->enqueue(cmd);
    return B200_OK;
  }
  return read_slot_async_now(en, slot, planes, strides);
}

static int read_slot_async_now(b200_engine* en, int slot, void* const planes[3], const size_t strides[3])
{
  const Surface* sp = dpb_picture(en->dpb, slot);
  if (!sp) return set_err(B200_ERR_INVALID, "slot %d holds no picture", slot);
  const Surface& s = *sp;
  CU(cudaSetDevice(en->device));
  const int k = dpb_read_stream(en->dpb, slot);
  cudaStream_t st = en->ctx[k].stream;
  for (int c = 0; c < (s.chroma ? 3 : 1); c++) {
    if (!planes[c]) continue;
    const int w = c ? s.cw : s.w, h = c ? s.ch : s.h, bps = bytes_per_sample(c ? s.bd_c : s.bd_y);
    CU(cudaMemcpy2DAsync(planes[c], strides[c], s.plane[c], s.pitch[c], (size_t)w * bps, h, cudaMemcpyDeviceToHost, st));
  }
  return dpb_mark_read(en->dpb, slot, k, st);
}

extern "C" int b200_engine_read_slot(b200_engine* en, int slot, void* const planes[3], const size_t strides[3])
{
  int rc = b200_engine_read_slot_async(en, slot, planes, strides);
  if (!rc) rc = flushed(en);
  if (rc) return rc;
  CU(cudaStreamSynchronize(en->ctx[dpb_read_stream(en->dpb, slot)].stream));
  return check_intra_err(en);
}

extern "C" int b200_engine_wait_slot(b200_engine* en, int slot)
{
  if (!en || slot < 0 || slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "bad argument");
  CU(cudaSetDevice(en->device));
  if (en->async) {  // not a flush: only the commands that touch this slot (later pictures may still be with the planners)
    const int rc = en->async->wait(en->async->slot_ticket(slot));
    if (rc) return rc;
  }
  std::vector<cudaEvent_t> evs;
  {
    std::lock_guard<std::mutex> issue(en->issue_m);  // the sequencer may be issuing later pictures
    dpb_wait_events(en->dpb, slot, evs);
  }
  for (cudaEvent_t e : evs) CU(cudaEventSynchronize(e));
  return check_intra_err(en);
}

extern "C" void* b200_host_alloc(size_t bytes)
{
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
extern "C" void b200_host_free(void* p)
{
  if (p) cudaFreeHost(p);
}

// Ordered against the engine through the picture store's external reader (dpb_export_before / _after).
extern "C" int b200_engine_export_slot(b200_engine* en, int slot, const b200_export* ex, void* const dst[3], const size_t dst_pitch[3], void* stream)
{
  if (!en || !ex || !dst || !dst_pitch || slot < 0 || slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "bad argument");
  if (ex->format > B200_EXPORT_RGB_BT2020) return set_err(B200_ERR_INVALID, "unknown export format %d", ex->format);
  if (ex->flags & ~B200_EXPORT_FULL_RANGE) return set_err(B200_ERR_INVALID, "unknown export flags 0x%x", ex->flags);
  if (ex->reserved[0] || ex->reserved[1]) return set_err(B200_ERR_INVALID, "reserved export bytes must be 0");
  CU(cudaSetDevice(en->device));
  if (en->async) {  // the slot's picture may still be queued: wait until it has been issued (not until it is finished)
    const int rc = en->async->wait(en->async->slot_ticket(slot));
    if (rc) return rc;
  }
  std::lock_guard<std::mutex> issue(en->issue_m);  // the sequencer may be issuing later pictures
  const Surface* sp = dpb_picture(en->dpb, slot);
  if (!sp) return set_err(B200_ERR_INVALID, "slot %d holds no picture", slot);
  const Surface& s = *sp;
  const int x = ex->x, y = ex->y, w = ex->width, h = ex->height;
  if (w == 0 || h == 0 || x + w > s.w || y + h > s.h)
    return set_err(B200_ERR_INVALID, "export window %dx%d at (%d, %d) is empty or outside the %dx%d picture", w, h, x, y, s.w, s.h);
  if (s.chroma && ((x | y | w | h) & 1)) return set_err(B200_ERR_INVALID, "4:2:0 export window (%d, %d) %dx%d is not even", x, y, w, h);
  const bool rgb = ex->format != B200_EXPORT_YUV;
  const int n_out = rgb || s.chroma ? 3 : 1;
  for (int c = 0; c < n_out; c++) {
    const size_t row = rgb ? (size_t)w : (size_t)(c ? w / 2 : w) * bytes_per_sample(c ? s.bd_c : s.bd_y);
    if (!dst[c]) return set_err(B200_ERR_INVALID, "export plane %d missing", c);
    if (dst_pitch[c] < row) return set_err(B200_ERR_INVALID, "export plane %d: pitch %zu below the row's %zu bytes", c, dst_pitch[c], row);
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = dpb_export_before(en->dpb, slot, st);
  if (rc) return rc;
  const uint8_t* src[3] = {nullptr, nullptr, nullptr};
  for (int c = 0; c < (s.chroma ? 3 : 1); c++) {
    const int cx = c ? x / 2 : x, cy = c ? y / 2 : y;
    src[c] = s.plane[c] + (size_t)cy * s.pitch[c] + (size_t)cx * bytes_per_sample(c ? s.bd_c : s.bd_y);
  }
  if (!rgb) {
    for (int c = 0; c < n_out; c++) {
      const int bps = bytes_per_sample(c ? s.bd_c : s.bd_y);
      CU(cudaMemcpy2DAsync(dst[c], dst_pitch[c], src[c], s.pitch[c], (size_t)(c ? w / 2 : w) * bps, c ? h / 2 : h, cudaMemcpyDeviceToDevice, st));
    }
  } else {
    ExportArgs a;
    for (int c = 0; c < 3; c++) {
      a.src[c] = src[c];
      a.src_pitch[c] = s.pitch[c];
      a.dst[c] = (uint8_t*)dst[c];
      a.dst_pitch[c] = dst_pitch[c];
    }
    a.w = w;
    a.h = h;
    a.c = export_coefs(ex->format, (ex->flags & B200_EXPORT_FULL_RANGE) != 0, s.bd_y, s.chroma ? s.bd_c : 8);
    launch_export_rgb(a, bytes_per_sample(s.bd_y), bytes_per_sample(s.bd_c), !s.chroma, st);
    en->launches++;
    CU(cudaGetLastError());
  }
  return dpb_export_after(en->dpb, slot, st);
}

extern "C" int b200_engine_slot_device_planes(b200_engine* en, int slot, void* planes[3], size_t strides[3])
{
  if (!en || !planes || !strides || slot < 0 || slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "bad argument");
  const Surface* s = dpb_picture(en->dpb, slot);
  if (!s) return set_err(B200_ERR_INVALID, "slot %d holds no picture", slot);
  for (int c = 0; c < 3; c++) { planes[c] = s->plane[c]; strides[c] = (size_t)s->pitch[c]; }
  return B200_OK;
}
#include "dsp_table.cuh"
