// planner.cuh — the host planner: turns one picture's records into the work lists the kernels consume.
//
// Validates the records, cuts the PUs into MC units, sorts the non-intra TUs into the k_residual classes, forms the intra tasks
// and puts their tickets in topological order, and packs the record arrays and the lists into one staging buffer.  Host code
// only: a Planner owns nothing but its options and scratch, so the engine, the asynchronous planner threads and
// b200_plan_picture_host (no device) run the very same sequence.  Included by engine.cu (one translation unit).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

// The planner's switches, read from the environment once per engine (and per b200_plan_picture_host call).
struct PlanOptions {
  int region = 16;  // luma size of an intra region task (16 or 8; B200_REGION)
  // 2: tickets of every picture by DAG level, 1: intra pictures only (B200_INTRA_ORDER=level_i), 0: CTB anti-diagonal order everywhere (=diag)
  int intra_level_order = 2;
  // one intra task per plane and region in every picture (default).  B200_INTRA_SPLIT=0: pictures with inter prediction merge the
  // planes of a region into one task — fewer tasks, but each runs its segments in sequence (three dependent L2 round trips)
  bool intra_split_planes = true;
  bool mc_legacy = false;  // B200_MC_LEGACY=1: 8x16 MC units for the first-generation 8-bit MC kernel (k_inter_pred8), for A/B measurements
};

static PlanOptions plan_options_from_env()
{
  PlanOptions o;
  if (const char* e = getenv("B200_REGION")) o.region = (atoi(e) == 8) ? 8 : 16;
  if (const char* e = getenv("B200_INTRA_ORDER")) o.intra_level_order = !strcmp(e, "diag") ? 0 : !strcmp(e, "level_i") ? 1 : 2;
  if (const char* e = getenv("B200_INTRA_SPLIT")) o.intra_split_planes = atoi(e) != 0;
  if (const char* e = getenv("B200_MC_LEGACY")) o.mc_legacy = atoi(e) != 0;
  return o;
}

// What the words of the MC section are; launch_picture runs the kernel that reads them.
enum McUnits : uint8_t {
  MC_TILES16,        // > 8 bit: <= 16x16 tiles, one warp each (k_inter_pred<uint16_t>, kernels_mc.cuh)
  MC_CLASS_BATCHES,  // 8 bit: <= 16x16 tiles tagged with their class, in class-pure batches + the batch table (k_inter_pred_tma, kernels_mct.cuh)
  MC_UNITS8x16,      // 8 bit with B200_MC_LEGACY=1: <= 8x16 units, one quarter-warp each (k_inter_pred8, kernels_mc8.cuh)
};

// A planned picture: section offsets of its staging buffer / device arena, the list sizes, and how it was planned.
struct PicLayout {
  size_t off[14] = {}, total = 0, raw_total = 0, unit_cap = 0;
  uint32_t ref_mask = 0;  // slots the picture's PUs read
  int n_tiles = 0, n_batches = 0, n_a = 0, n_aw = 0, n_a8 = 0, n_b = 0, n_task = 0;
  bool direct = false;                   // B200_PIC_RECORDS_PINNED: raw sections are uploaded from raw_src (the caller's arrays)
  const void* raw_src[14] = {};
  size_t raw_sz[14] = {};
  int intra_levels = 0, intra_width = 0;  // tickets in DAG-level order: number of levels, tasks in the widest level (0: anti-diagonal order)
  int region = 16;                        // luma size of the intra region tasks (k_intra's ReconArgs::region)
  McUnits mc_units = MC_CLASS_BATCHES;
  bool run_deblock = false, run_sao = false, has_scaling = false;
  b200_pic_params params{};
  uint32_t n_tu = 0;
};

static int check_params(const b200_pic_params& p)
{
  if (p.width == 0 || p.height == 0) return set_err(B200_ERR_INVALID, "empty picture");
  if (p.log2_ctb_size < 4 || p.log2_ctb_size > 6) return set_err(B200_ERR_INVALID, "log2_ctb_size %d", p.log2_ctb_size);
  if (p.dst_slot >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "dst_slot %d", p.dst_slot);
  if (p.chroma_format_idc > 1) return set_err(B200_ERR_UNSUPPORTED, "chroma_format_idc %d: the device path implements 4:0:0 and 4:2:0", p.chroma_format_idc);
  if (p.bit_depth_luma < 8 || p.bit_depth_luma > 12 || p.bit_depth_chroma < 8 || p.bit_depth_chroma > 12)
    return set_err(B200_ERR_UNSUPPORTED, "bit depth %d/%d (8..12 supported)", p.bit_depth_luma, p.bit_depth_chroma);
  if ((p.bit_depth_luma > 8) != (p.bit_depth_chroma > 8)) return set_err(B200_ERR_UNSUPPORTED, "mixed 8-bit / high-bit-depth planes");
  if ((p.width & 7) || (p.height & 7)) return set_err(B200_ERR_INVALID, "picture size must be a multiple of the minimum CB size (8)");
  return B200_OK;
}

#define PLAN_PU_PARTS 4
#define PLAN_INTRA_PARTS 8
struct IntraPart {
  uint32_t i0 = 0, i1 = 0, task_base = 0;
  std::vector<uint32_t> intra_idx, task_of, task_first, task_cell, diag_cnt, diag_off, fill;  // task_cell: region cell x | y << 12 | cells per side << 24 | plane << 28
};

// The options and the scratch of one planning thread, reused across pictures.  The parallel phases of a picture with at least
// pool_min_tus TUs run on `pool` (shared with other planners: each waits for its own group); without a pool, or for a smaller
// picture, everything runs on the calling thread.
struct Planner {
  PlanOptions opt;
  HostPool* pool = nullptr;
  HostPool::Group group;
  uint32_t pool_min_tus = 0;
  bool use_pool = false;  // for the picture being planned
  void run(std::function<void()> f)
  {
    if (use_pool) pool->run(&group, std::move(f));
    else f();
  }
  void wait()
  {
    if (use_pool) pool->wait(&group);
  }
  std::vector<uint32_t> part_a[PLAN_INTRA_PARTS][3];  // plan_intra_A: per range, per k_residual class
  std::vector<uint32_t> pu_tiles[PLAN_PU_PARTS];      // plan_pus_part
  size_t pu_count[PLAN_PU_PARTS][8] = {};
  uint32_t pu_ref_mask[PLAN_PU_PARTS] = {};
  IntraPart ipart[PLAN_INTRA_PARTS];                  // plan_intra_*
  std::vector<uint32_t> cell_level[3], task_level, level_off;  // plan_intra_levels
  std::vector<uint32_t> tiles, list_a, list_b, task_start, task_order;
};

// Section order in the staging buffer / device arena: the raw record arrays first (their offsets depend only on the
// counts, so copying them can start before the work lists exist), then the lists the planner builds.
//   0 pus, 1 weights, 2 tus, 5 coeffs, 6 slices, 7 ctbs, 8 bs_map, 9 qp_map, 10 nofilt_map, 11 scaling |
//   3 list_a (non-intra TU indices by k_residual class), 4 list_b (intra TU indices by task), 12 MC units / tiles, 13 task_start
static const int k_raw_sections[10] = {0, 1, 2, 5, 6, 7, 8, 9, 10, 11};
static const int k_list_sections[4] = {3, 4, 12, 13};

// Checks the picture parameters and the presence of the record arrays, lays out the raw sections and records how the picture
// is planned; *cap_total = the staging bytes plan_build may need.
static int plan_begin(Planner& pl, const b200_picture* pic, PicLayout* L, size_t* cap_total)
{
  const b200_pic_params& p = pic->params;
  int rc = check_params(p);
  if (rc) return rc;
  if ((pic->n_pu && !pic->pus) || (pic->n_tu && !pic->tus) || (pic->n_coeff && !pic->coeffs) || !pic->slices || !pic->ctbs || !pic->qp_map ||
      !pic->nofilt_map || pic->n_slices == 0)
    return set_err(B200_ERR_INVALID, "missing record arrays");
  if (pic->n_pu >= (1u << 20)) return set_err(B200_ERR_INVALID, "too many PUs");
  const int S = 1 << p.log2_ctb_size;
  const int wctb = (p.width + S - 1) / S, hctb = (p.height + S - 1) / S, n_ctb = wctb * hctb;
  const int w4 = (p.width + 3) / 4, h4 = (p.height + 3) / 4, w8 = (p.width + 7) / 8, h8 = (p.height + 7) / 8;
  L->params = p;
  L->n_tu = pic->n_tu;
  L->has_scaling = pic->scaling_factors != nullptr;
  L->run_deblock = !(p.flags & B200_PIC_SKIP_DEBLOCK) && pic->bs_map && (p.stop_after_stage == B200_STAGE_ALL || p.stop_after_stage == B200_STAGE_DEBLOCK);
  L->run_sao = (p.flags & B200_PIC_SAO_ENABLED) && !(p.flags & B200_PIC_SKIP_SAO) && p.stop_after_stage == B200_STAGE_ALL;
  L->region = pl.opt.region;
  L->mc_units = p.bit_depth_luma > 8 ? MC_TILES16 : pl.opt.mc_legacy ? MC_UNITS8x16 : MC_CLASS_BATCHES;

  for (int i = 0; i < n_ctb; i++)
    if (pic->ctbs[i].slice_idx >= pic->n_slices) return set_err(B200_ERR_INVALID, "CTB %d slice index", i);
  size_t sz[14] = {};
  sz[0] = sizeof(b200_pu) * pic->n_pu;
  sz[1] = sizeof(b200_weight_entry) * pic->n_weights;
  sz[2] = sizeof(b200_tu) * pic->n_tu;
  sz[5] = sizeof(b200_coeff) * pic->n_coeff;
  sz[6] = sizeof(b200_slice_info) * pic->n_slices;
  sz[7] = sizeof(b200_ctb_info) * (size_t)n_ctb;
  sz[8] = L->run_deblock ? (size_t)w4 * h4 : 0;
  sz[9] = (size_t)w8 * h8;
  sz[10] = (size_t)w8 * h8;
  sz[11] = L->has_scaling ? B200_SCALING_FACTOR_BYTES : 0;
  size_t total = 0;
  for (int i : k_raw_sections) { L->off[i] = total; total += align_up(sz[i], 256); }
  L->raw_total = total;
  L->direct = (p.flags & B200_PIC_RECORDS_PINNED) != 0;
  const void* src[14] = {pic->pus, pic->weights, pic->tus, nullptr, nullptr, pic->coeffs, pic->slices, pic->ctbs, pic->bs_map, pic->qp_map, pic->nofilt_map,
                         pic->scaling_factors, nullptr, nullptr};
  for (int i : k_raw_sections) { L->raw_src[i] = src[i]; L->raw_sz[i] = sz[i]; }
  // upper bound of the lists: every TU in one list, one task per TU; MC units cannot outnumber 4x8 blocks unless PUs overlap
  L->unit_cap = ((size_t)w4 * h4 / 2 + 64 + 8 * MCT_MAX_TILES) * 3 / 2 + 64;  // + the padding of the class-pure batches + the batch table
  *cap_total = total + 3 * align_up(sizeof(uint32_t) * ((size_t)pic->n_tu + 1), 256) + align_up(sizeof(uint32_t) * L->unit_cap, 256) + 256;
  return B200_OK;
}

// PU validation + MC work list for the PU range [i0, i1) into the part's own tile list (parts run on pool threads;
// plan_pus_merge sorts them into class-pure batches)
static int plan_pus_part(Planner& pl, const b200_picture* pic, McUnits units, int part, uint32_t i0, uint32_t i1)
{
  const b200_pic_params& p = pic->params;
  std::vector<uint32_t>& tiles = pl.pu_tiles[part];
  // at most 16 tiles (64x64 PU) per record: written through a raw pointer, trimmed at the end (no per-tile capacity check)
  tiles.resize((size_t)(i1 - i0) * 16);
  uint32_t* out = tiles.data();
  uint32_t ref_mask = 0;
  size_t count[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const bool wide = units == MC_TILES16;
  const bool legacy = units == MC_UNITS8x16;
  const unsigned pw = p.width, ph = p.height;
  const uint32_t n_weights = pic->n_weights;
  const b200_pu* pus = pic->pus;
  for (uint32_t i = i0; i < i1; i++) {
    const b200_pu& pu = pus[i];
    const unsigned w = pu.w, h = pu.h;
    if (w - 1u > 63u || h - 1u > 63u || ((w | h | pu.x | pu.y) & 3u) || pu.x + w > pw || pu.y + h > ph)
      return set_err(B200_ERR_INVALID, "PU %u out of range", i);
    if ((pu.flags & B200_PU_WEIGHTED) && pu.wt_idx >= n_weights) return set_err(B200_ERR_INVALID, "PU %u weight index", i);
    if (pu.ref_slot[0] >= B200_MAX_SLOTS || pu.ref_slot[1] >= B200_MAX_SLOTS) return set_err(B200_ERR_INVALID, "PU %u reference slot", i);
    const unsigned l0 = pu.flags & B200_PU_PRED_L0, l1 = pu.flags & B200_PU_PRED_L1;
    if (!(l0 | l1)) continue;
    if (l0 && pu.ref_slot[0] >= 0) ref_mask |= 1u << pu.ref_slot[0];
    if (l1 && pu.ref_slot[1] >= 0) ref_mask |= 1u << pu.ref_slot[1];
    if (wide) {  // 16-bit path: <= 16x16 tiles, one warp each (kernels_mc.cuh)
      for (unsigned ty = 0; ty * MC_TILE < h; ty++)
        for (unsigned tx = 0; tx * MC_TILE < w; tx++) *out++ = i | (tx << 20) | (ty << 22);
    } else if (legacy) {  // first-generation 8-bit path: <= 8x16 units, one quarter-warp each (kernels_mc8.cuh)
      tiles.resize((size_t)(out - tiles.data()));  // (rare debug path: up to 32 units per PU, keep the simple form)
      for (unsigned uy = 0; uy * MC8_UH < h; uy++)
        for (unsigned ux = 0; ux * MC8_UW < w; ux++) tiles.push_back(MC8_UNIT(i, ux, uy));
      const size_t used = tiles.size();
      tiles.resize(used + (size_t)(i1 - i - 1) * 32 + 32);
      out = tiles.data() + used;
    } else {     // 8-bit path: <= 16x16 tiles with their class (kernels_mct.cuh), sorted into class-pure batches by the merge
      const unsigned bi = (l0 && l1) ? MCT_CLASS_BI : 0;
      for (unsigned ty = 0; ty * 16 < h; ty++) {
        const unsigned tall = (h - 16 * ty > 8) ? MCT_CLASS_TALL : 0;
        for (unsigned tx = 0; tx * 16 < w; tx++) {
          const unsigned cls = bi | tall | ((w - 16 * tx > 8) ? MCT_CLASS_WIDE : 0);
          *out++ = MCT_TILE_WORD(i, tx, ty, cls);
          count[cls]++;
        }
      }
    }
  }
  tiles.resize((size_t)(out - tiles.data()));
  for (int c = 0; c < 8; c++) pl.pu_count[part][c] = count[c];
  pl.pu_ref_mask[part] = ref_mask;
  return B200_OK;
}

// Concatenates the parts; 8-bit: counting sort by class, every class padded to whole batches (MCT_CLASS_TILES tiles of one class,
// padding = MCT_INVALID), the batch table (first tile index | class) behind the tile words in the same section.
static int plan_pus_merge(Planner& pl, PicLayout* L)
{
  std::vector<uint32_t>& tiles = pl.tiles;
  L->n_batches = 0;
  for (int part = 0; part < PLAN_PU_PARTS; part++) L->ref_mask |= pl.pu_ref_mask[part];
  size_t n_words;
  if (L->mc_units != MC_CLASS_BATCHES) {
    tiles.clear();
    for (int part = 0; part < PLAN_PU_PARTS; part++) tiles.insert(tiles.end(), pl.pu_tiles[part].begin(), pl.pu_tiles[part].end());
    n_words = tiles.size();
  } else {
    size_t count[8] = {}, start[8], total = 0, nb = 0;
    for (int part = 0; part < PLAN_PU_PARTS; part++)
      for (int c = 0; c < 8; c++) count[c] += pl.pu_count[part][c];
    for (int c = 0; c < 8; c++) {
      const size_t per = MCT_CLASS_TILES(c), batches = (count[c] + per - 1) / per;
      start[c] = total;
      total += batches * per;
      nb += batches;
    }
    tiles.assign(total + nb, MCT_INVALID);
    size_t bi = total;
    for (int c = 0; c < 8; c++)
      for (size_t f = start[c]; f < start[c] + (count[c] + MCT_CLASS_TILES(c) - 1) / MCT_CLASS_TILES(c) * MCT_CLASS_TILES(c); f += MCT_CLASS_TILES(c))
        tiles[bi++] = MCT_BATCH_WORD(f, c);
    for (int part = 0; part < PLAN_PU_PARTS; part++)
      for (uint32_t t : pl.pu_tiles[part]) tiles[start[(t >> 24) & 7]++] = t;
    n_words = total;
    L->n_batches = (int)nb;
  }
  if (tiles.size() > L->unit_cap) return set_err(B200_ERR_INVALID, "PUs overlap (more MC units than the picture has 4x8 blocks)");
  L->n_tiles = (int)n_words;  // tile words; pl.tiles also holds the n_batches batch words behind them
  return B200_OK;
}

// TU validation + the k_residual work classes for the TU range [i0, i1) into the part's own lists (two parts run on pool
// threads; merge_list_a concatenates them).  Classes: warp per TU (16x16, 32x32, PCM) | quarter-warp per 8x8 | lane per 4x4.
#define PLAN_TU_PARTS PLAN_INTRA_PARTS  // validation and the intra task formation share one pass over a range of TUs
// One TU record against the picture; B200_OK or the error (message set).  `dims`: plane sizes per cIdx (0 when the plane does not exist).
struct TuDims { int pw[3], ph[3]; };
static inline TuDims tu_dims(const b200_pic_params& p)
{
  TuDims d;
  d.pw[0] = p.width; d.ph[0] = p.height;
  d.pw[1] = d.pw[2] = p.chroma_format_idc ? p.width / 2 : 0;
  d.ph[1] = d.ph[2] = p.chroma_format_idc ? p.height / 2 : 0;
  return d;
}
static inline int tu_check(const TuDims& d, const b200_picture* pic, uint32_t i, const b200_tu& tu)
{
  const unsigned l2 = tu.log2_size, c = tu.cidx;
  if (l2 - 2u > 3u || c > 2u) return set_err(B200_ERR_INVALID, "TU %u out of range", i);
  const int nT = 1 << l2, pw = d.pw[c], ph = d.ph[c];
  if (tu.x + nT > pw || tu.y + nT > ph || ((tu.x | tu.y) & (nT - 1))) return set_err(B200_ERR_INVALID, "TU %u out of range", i);  // nT >= 4: also the 4-sample grid
  if ((size_t)tu.coeff_off + tu.n_coeff > pic->n_coeff || tu.n_coeff > nT * nT) return set_err(B200_ERR_INVALID, "TU %u coefficient range", i);
  if ((tu.flags & B200_TU_PCM) && tu.n_coeff != nT * nT) return set_err(B200_ERR_INVALID, "PCM TU %u sample count", i);
  if (tu.flags & B200_TU_INTRA) {
    if (tu.intra_mode > 34) return set_err(B200_ERR_INVALID, "TU %u intra mode", i);
    // avail bits must name samples inside the picture (k_intra reads the border and the pending flags at those positions)
    const int half = nT >> 1;  // groups of 4 samples per side
    const uint32_t gm = half >= 32 ? 0xffffffffu : (1u << half) - 1u;
    const uint32_t left = (uint32_t)tu.avail & 0xffffu, top = (uint32_t)(tu.avail >> B200_AVAIL_TOP_BIT0) & 0xffffu;
    const bool corner = (tu.avail >> B200_AVAIL_CORNER_BIT) & 1;
    const int rows_below = (ph - tu.y) >> 2, cols_right = (pw - tu.x) >> 2;  // groups that still lie inside the plane
    const uint32_t lm = rows_below >= 16 ? 0xffffu : (1u << rows_below) - 1u, tm = cols_right >= 16 ? 0xffffu : (1u << cols_right) - 1u;
    if ((left & ~gm) || (top & ~gm) || (tu.avail >> (B200_AVAIL_TOP_BIT0 + 16)) || (left && tu.x == 0) || (top && tu.y == 0) ||
        (corner && (tu.x == 0 || tu.y == 0)) || (left & ~lm) || (top & ~tm))
      return set_err(B200_ERR_INVALID, "TU %u intra availability names samples outside the picture", i);
  }
  return B200_OK;
}

// TU validation, the k_residual classes of the non-intra TUs and the intra work list, in one pass over the TU records.  Intra tasks: the TUs of one plane inside one aligned 16x16-luma / 8x8-chroma region (contiguous per plane in
// decode order); a TU at least as large as the region is a task of its own.  Tasks are emitted in a topological order: CTB
// anti-diagonal x + 2y, ties in decode order.  The TU list is cut at CTB boundaries into PLAN_INTRA_PARTS ranges (a region
// never crosses a CTB, so no task spans two ranges) and the phases A, C, E run per range on the pool threads:
//   A  per range: intra TUs, their (range-local) task ids, tasks per diagonal          B  serial: task / rank offsets of the ranges
//   C  per range: rank of every task, TUs per task                                      D  serial: prefix sum -> task_start
//   E  per range: list_b (TU indices grouped by task in rank order)

static inline size_t plan_diag_of(const b200_pic_params& p, const b200_tu& tu)
{
  const int sh = tu.cidx ? 1 : 0;
  return (size_t)((tu.x << sh) >> p.log2_ctb_size) + 2 * (size_t)((tu.y << sh) >> p.log2_ctb_size);
}
static inline uint32_t plan_ctb_of(const b200_pic_params& p, const b200_tu& tu)
{
  const int sh = (tu.cidx && tu.cidx <= 2) ? 1 : 0;
  return (uint32_t)(((uint32_t)tu.x << sh) >> p.log2_ctb_size) | ((uint32_t)(((uint32_t)tu.y << sh) >> p.log2_ctb_size) << 16);
}

static void plan_intra_ranges(Planner& pl, const b200_picture* pic)
{
  const b200_pic_params& p = pic->params;
  uint32_t prev = 0;
  for (int k = 0; k < PLAN_INTRA_PARTS; k++) {
    uint32_t end = (k == PLAN_INTRA_PARTS - 1) ? pic->n_tu : (uint32_t)((uint64_t)pic->n_tu * (k + 1) / PLAN_INTRA_PARTS);
    if (end < prev) end = prev;
    // move the cut forward to the next CTB change (all TUs of a CTB are contiguous in decode order)
    while (end > 0 && end < pic->n_tu && plan_ctb_of(p, pic->tus[end]) == plan_ctb_of(p, pic->tus[end - 1])) end++;
    pl.ipart[k].i0 = prev;
    pl.ipart[k].i1 = end;
    prev = end;
  }
}

static int plan_intra_A(Planner& pl, const b200_picture* pic, int k, int n_diag, int wctb, int hctb)
{
  const b200_pic_params& p = pic->params;
  IntraPart& ip = pl.ipart[k];
  std::vector<uint32_t>&la = pl.part_a[k][0], &la8 = pl.part_a[k][1], &la4 = pl.part_a[k][2];  // non-intra TUs with a residual, by k_residual class
  la.clear();
  la8.clear();
  la4.clear();
  ip.intra_idx.clear();
  ip.task_of.clear();
  ip.task_first.clear();
  ip.task_cell.clear();
  ip.diag_cnt.assign((size_t)n_diag, 0);
  // Pictures with inter prediction have few, scattered intra blocks: the per-task overhead of k_intra dominates there, so the
  // small TUs of ALL planes of a region form one task (luma, then Cb, then Cr) when they are at most 16; intra pictures keep
  // one task per plane (three shorter dependency chains side by side).
  const bool merged = pic->n_pu > 0 && !pl.opt.intra_split_planes;
  const int lg_region = pl.opt.region == 16 ? 4 : 3;
  const TuDims dims = tu_dims(p);
  long long cur_key[3] = {-1, -1, -1};
  uint32_t cur_task[3] = {0, 0, 0};
  uint32_t run[48];  // merged mode: the small intra TUs of the current region (at most 16 + 4 + 4, sized generously)
  int n_run = 0;
  long long run_key = -1;
  auto new_task = [&](uint32_t first_tu) {
    const b200_tu& ft = pic->tus[first_tu];
    ip.task_first.push_back(first_tu);
    ip.diag_cnt[plan_diag_of(p, ft)]++;
    const uint32_t sh = ft.cidx ? 1 : 0;  // what plan_intra_levels needs of the task, kept here so that pass reads no TU record
    const uint32_t R = std::max(1u, ((1u << ft.log2_size) << sh) >> lg_region);
    ip.task_cell.push_back((((uint32_t)ft.x << sh) >> lg_region) | ((((uint32_t)ft.y << sh) >> lg_region) << 12) | (R << 24) | ((uint32_t)ft.cidx << 28));
    return (uint32_t)ip.task_first.size() - 1;
  };
  auto flush_run = [&]() {
    if (!n_run) return;
    int cnt[3] = {0, 0, 0};
    for (int j = 0; j < n_run; j++) cnt[pic->tus[run[j]].cidx]++;
    const bool one = n_run <= 16;
    uint32_t t = 0;
    if (one) t = new_task(run[0]);
    for (int c = 0; c < 3; c++) {  // plane by plane, decode order inside a plane
      if (!cnt[c]) continue;
      bool first = true;
      for (int j = 0; j < n_run; j++) {
        if (pic->tus[run[j]].cidx != c) continue;
        if (!one && first) t = new_task(run[j]);
        first = false;
        ip.intra_idx.push_back(run[j]);
        ip.task_of.push_back(t);
      }
    }
    n_run = 0;
  };
  for (uint32_t i = ip.i0; i < ip.i1; i++) {
    const b200_tu& tu = pic->tus[i];
    if (const int rc = tu_check(dims, pic, i, tu)) return rc;
    if (!(tu.flags & B200_TU_INTRA)) {
      if (tu.flags & (B200_TU_CBF | B200_TU_PCM)) {
        if ((tu.flags & B200_TU_PCM) || tu.log2_size > 3) la.push_back(i);
        else if (tu.log2_size == 3) la8.push_back(i);
        else la4.push_back(i);
      }
      continue;
    }
    const int c = tu.cidx, G = pl.opt.region >> (c ? 1 : 0), nT = 1 << tu.log2_size;
    if (merged) {
      if (nT >= G) {  // a TU at least as large as the region is a task of its own
        flush_run();
        run_key = -1;
        ip.intra_idx.push_back(i);
        ip.task_of.push_back(new_task(i));
        continue;
      }
      const int sh = c ? 1 : 0;
      const long long key = (((long long)((tu.y << sh) >> lg_region)) << 20) | ((tu.x << sh) >> lg_region);
      if (key != run_key || n_run == 48) {
        flush_run();
        run_key = key;
      }
      run[n_run++] = i;
      continue;
    }
    ip.intra_idx.push_back(i);
    const long long key = (nT >= G) ? -2 - (long long)i : (((long long)(tu.y >> (lg_region - (c ? 1 : 0)))) << 20) | (tu.x >> (lg_region - (c ? 1 : 0)));
    if (key != cur_key[c]) {
      cur_key[c] = key;
      cur_task[c] = new_task(i);
    }
    ip.task_of.push_back(cur_task[c]);
  }
  flush_run();
  return B200_OK;
}

static void plan_intra_B(Planner& pl, int n_diag, uint32_t* n_task, uint32_t* n_intra)
{
  uint32_t nt = 0, ni = 0;
  for (int k = 0; k < PLAN_INTRA_PARTS; k++) {
    pl.ipart[k].task_base = nt;
    nt += (uint32_t)pl.ipart[k].task_first.size();
    ni += (uint32_t)pl.ipart[k].intra_idx.size();
    pl.ipart[k].diag_off.assign((size_t)n_diag, 0);
  }
  uint32_t run = 0;
  for (int d = 0; d < n_diag; d++)
    for (int k = 0; k < PLAN_INTRA_PARTS; k++) {  // ranges are in decode order: within a diagonal, earlier ranges rank first
      pl.ipart[k].diag_off[d] = run;
      run += pl.ipart[k].diag_cnt[d];
    }
  *n_task = nt;
  *n_intra = ni;
  pl.task_order.resize(nt);
  pl.task_start.assign((size_t)nt + 1, 0);
  pl.list_b.resize(ni);
}

// Ticket order by DAG LEVEL (default; B200_INTRA_ORDER=diag keeps the CTB anti-diagonal order).  A level is assigned per task in
// ONE pass over the tasks in decode order through a map "region cell (16x16 luma) -> highest level of a task covering it":
//   level(task) = 1 + max over the cells its TUs may read (the column left of it from one cell above to 2x its height below —
//   corner, left and bottom-left neighbours — and the row above it to 2x its width — top and top-right), cells not written yet
//   (decoded later, or not intra) count 0.
// That is a superset of the true dependencies (availability bits), which is all a valid layering needs: every neighbour a task
// waits for has a lower level.  Tasks of one level are independent, so with tickets sorted by level the lowest unfinished
// tickets are exactly the ready tasks: the persistent warps of k_intra hold ready work instead of spinning on tasks far down
// the anti-diagonal, and the grid is sized to the DAG's width (the widest level) instead of the whole GPU — the other SMs stay
// free for the pictures it overlaps with.  (The anti-diagonal order is topological too, but of the ~500 consecutive tickets
// the warps hold only the first task of every CTB chain is ready.)  Intra pictures keep one map per plane (their tasks are
// per plane); pictures with inter prediction one map (tasks span the planes).
static void plan_intra_levels(Planner& pl, const b200_picture* pic, PicLayout* L, uint32_t n_task)
{
  const b200_pic_params& p = pic->params;
  const int lg = pl.opt.region == 16 ? 4 : 3;
  const int cw = (p.width + (1 << lg) - 1) >> lg, ch = (p.height + (1 << lg) - 1) >> lg;
  const bool per_plane = pic->n_pu == 0 || pl.opt.intra_split_planes;
  for (int c = 0; c < (per_plane ? 3 : 1); c++) pl.cell_level[c].assign((size_t)cw * ch, 0);
  std::vector<uint32_t>& level = pl.task_level;
  level.resize(n_task);
  uint32_t max_level = 0;
  for (int k = 0; k < PLAN_INTRA_PARTS; k++) {
    const IntraPart& ip = pl.ipart[k];
    for (size_t t = 0; t < ip.task_first.size(); t++) {
      const uint32_t tc = ip.task_cell[t];
      const int cx = (int)(tc & 0xfff), cy = (int)((tc >> 12) & 0xfff);
      const int R = (int)((tc >> 24) & 0xf);  // cells per side: 1 (region task) or the large TU's size
      uint32_t* map = pl.cell_level[per_plane ? (tc >> 28) : 0].data();
      uint32_t lvl = 0;
      if (cx > 0)
        for (int y = std::max(cy - 1, 0); y < std::min(cy + 2 * R, ch); y++) lvl = std::max(lvl, map[(size_t)y * cw + cx - 1]);
      if (cy > 0)
        for (int x = cx; x < std::min(cx + 2 * R, cw); x++) lvl = std::max(lvl, map[(size_t)(cy - 1) * cw + x]);
      lvl++;
      level[ip.task_base + t] = lvl;
      if (lvl > max_level) max_level = lvl;
      for (int y = cy; y < std::min(cy + R, ch); y++)
        for (int x = cx; x < std::min(cx + R, cw); x++) {
          uint32_t& m = map[(size_t)y * cw + x];
          if (lvl > m) m = lvl;  // several tasks may cover a cell (planes of a merged region that were split, large chroma TUs)
        }
    }
  }
  // rank = position in (level, decode order): counting sort over the levels; the widest level sizes the grid
  std::vector<uint32_t>& off = pl.level_off;
  off.assign((size_t)max_level + 2, 0);
  for (uint32_t t = 0; t < n_task; t++) off[level[t] + 1]++;
  uint32_t width = 0;
  for (size_t l = 1; l < off.size(); l++) {
    if (off[l] > width) width = off[l];
    off[l] += off[l - 1];
  }
  uint32_t* order = pl.task_order.data();
  for (uint32_t t = 0; t < n_task; t++) order[t] = off[level[t]]++;
  L->intra_levels = (int)max_level;
  L->intra_width = (int)width;
}

static void plan_intra_C(Planner& pl, const b200_picture* pic, int k, bool by_level)
{
  const b200_pic_params& p = pic->params;
  IntraPart& ip = pl.ipart[k];
  uint32_t* order = pl.task_order.data() + ip.task_base;
  if (!by_level)
    for (size_t t = 0; t < ip.task_first.size(); t++) order[t] = ip.diag_off[plan_diag_of(p, pic->tus[ip.task_first[t]])]++;
  uint32_t* ts = pl.task_start.data();
  for (size_t j = 0; j < ip.task_of.size(); j++) ts[order[ip.task_of[j]] + 1]++;  // a task belongs to exactly one range: no two threads touch one entry
}

static void plan_intra_E(Planner& pl, int k)
{
  IntraPart& ip = pl.ipart[k];
  const uint32_t* order = pl.task_order.data() + ip.task_base;
  const uint32_t* ts = pl.task_start.data();
  ip.fill.resize(ip.task_first.size());
  for (size_t t = 0; t < ip.task_first.size(); t++) ip.fill[t] = ts[order[t]];
  uint32_t* lb = pl.list_b.data();
  for (size_t j = 0; j < ip.intra_idx.size(); j++) lb[ip.fill[ip.task_of[j]]++] = ip.intra_idx[j];
}

// Runs `f(k)` for k = 0..n-1 on the pool (or inline without one) and waits.
template <typename F>
static void plan_parallel(Planner& pl, int n, F f)
{
  for (int k = 0; k < n; k++) pl.run([=] { f(k); });
  pl.wait();
}

// The serial glue of the intra planner after phase A has run for every range (in plan_build, next to the other planning work).
static void plan_intra_finish(Planner& pl, const b200_picture* pic, PicLayout* L, int n_diag)
{
  uint32_t n_task = 0, n_intra = 0;
  plan_intra_B(pl, n_diag, &n_task, &n_intra);
  const bool by_level = n_task && (pl.opt.intra_level_order == 2 || (pl.opt.intra_level_order == 1 && pic->n_pu == 0));
  L->intra_levels = L->intra_width = 0;
  if (by_level) plan_intra_levels(pl, pic, L, n_task);
  plan_parallel(pl, PLAN_INTRA_PARTS, [&pl, pic, by_level](int k) { plan_intra_C(pl, pic, k, by_level); });
  uint32_t* ts = pl.task_start.data();
  for (uint32_t t = 0; t < n_task; t++) ts[t + 1] += ts[t];
  plan_parallel(pl, PLAN_INTRA_PARTS, [&pl](int k) { plan_intra_E(pl, k); });
  L->n_task = (int)n_task;
  L->n_b = (int)n_intra;
}

static void plan_finish(PicLayout* L)
{
  size_t sz[14] = {};
  sz[3] = sizeof(uint32_t) * (size_t)L->n_a;
  sz[4] = sizeof(uint32_t) * (size_t)L->n_b;
  sz[12] = sizeof(uint32_t) * (size_t)(L->n_tiles + L->n_batches);
  sz[13] = L->n_task ? sizeof(uint32_t) * (size_t)(L->n_task + 1) : 0;
  size_t total = L->raw_total;
  for (int i : k_list_sections) { L->off[i] = total; total += align_up(sz[i], 256); }
  L->total = total ? total : 256;
}

// part 0..2: the raw record arrays in three roughly equal shares (pool threads)
static void pack_raw(const b200_picture* pic, const PicLayout& L, uint8_t* hb, int part)
{
  const b200_pic_params& p = pic->params;
  const size_t* off = L.off;
  const int S = 1 << p.log2_ctb_size;
  const int wctb = (p.width + S - 1) / S, hctb = (p.height + S - 1) / S, n_ctb = wctb * hctb;
  const int w4 = (p.width + 3) / 4, h4 = (p.height + 3) / 4, w8 = (p.width + 7) / 8, h8 = (p.height + 7) / 8;
  if (part == 0) {
    if (pic->n_coeff) memcpy(hb + off[5], pic->coeffs, sizeof(b200_coeff) * pic->n_coeff);
  } else if (part == 1) {
    if (pic->n_tu) memcpy(hb + off[2], pic->tus, sizeof(b200_tu) * pic->n_tu);
    memcpy(hb + off[6], pic->slices, sizeof(b200_slice_info) * pic->n_slices);
    memcpy(hb + off[7], pic->ctbs, sizeof(b200_ctb_info) * (size_t)n_ctb);
  } else {
    if (pic->n_pu) memcpy(hb + off[0], pic->pus, sizeof(b200_pu) * pic->n_pu);
    if (pic->n_weights) memcpy(hb + off[1], pic->weights, sizeof(b200_weight_entry) * pic->n_weights);
    if (L.run_deblock) memcpy(hb + off[8], pic->bs_map, (size_t)w4 * h4);
    memcpy(hb + off[9], pic->qp_map, (size_t)w8 * h8);
    memcpy(hb + off[10], pic->nofilt_map, (size_t)w8 * h8);
    if (L.has_scaling) memcpy(hb + off[11], pic->scaling_factors, B200_SCALING_FACTOR_BYTES);
  }
}

static void pack_lists(Planner& pl, const PicLayout& L, uint8_t* hb)
{
  const size_t* off = L.off;
  if (L.n_a) memcpy(hb + off[3], pl.list_a.data(), sizeof(uint32_t) * (size_t)L.n_a);
  if (L.n_b) memcpy(hb + off[4], pl.list_b.data(), sizeof(uint32_t) * (size_t)L.n_b);
  if (L.n_task) memcpy(hb + off[13], pl.task_start.data(), sizeof(uint32_t) * (size_t)(L.n_task + 1));
  if (L.n_tiles) memcpy(hb + off[12], pl.tiles.data(), sizeof(uint32_t) * (size_t)(L.n_tiles + L.n_batches));
}

// list_a = class by class (warp | 8x8 | 4x4), the validation parts in order
static void merge_list_a(Planner& pl, PicLayout* L)
{
  std::vector<uint32_t>& la = pl.list_a;
  la.clear();
  for (int cls = 0; cls < 3; cls++) {
    for (int part = 0; part < PLAN_TU_PARTS; part++) la.insert(la.end(), pl.part_a[part][cls].begin(), pl.part_a[part][cls].end());
    if (cls == 0) L->n_aw = (int)la.size();
    if (cls == 1) L->n_a8 = (int)la.size() - L->n_aw;
  }
  L->n_a = (int)la.size();
}
// The rest of the picture after plan_begin: the TU ranges (validation, residual classes, intra tasks), the PU parts (validation,
// MC units) and the copies of the raw record arrays side by side, then the serial tail.  With `hb` (at least the plan_begin
// capacity) the raw arrays, unless the picture uploads them from the caller's memory, and the lists are packed into it;
// hb == nullptr packs nothing.  Errors: the first failing TU range, else the first failing PU part, else overlapping PUs.
static int plan_build(Planner& pl, const b200_picture* pic, PicLayout* L, uint8_t* hb)
{
  const b200_pic_params& pp = pic->params;
  const int S = 1 << pp.log2_ctb_size, wctb = (pp.width + S - 1) / S, hctb = (pp.height + S - 1) / S, n_diag = wctb + 2 * hctb;
  pl.use_pool = pl.pool && pic->n_tu >= pl.pool_min_tus;
  int rc_pu[PLAN_PU_PARTS] = {}, rc_tv[PLAN_TU_PARTS] = {};
  std::string err_pu[PLAN_PU_PARTS], err_tv[PLAN_TU_PARTS];
  plan_intra_ranges(pl, pic);
  for (int k = 0; k < PLAN_INTRA_PARTS; k++)  // the longest items first: TU validation + residual classes + intra tasks of one range
    pl.run([&, k] {
      rc_tv[k] = plan_intra_A(pl, pic, k, n_diag, wctb, hctb);
      if (rc_tv[k]) err_tv[k] = g_err;  // the worker's thread-local message
    });
  for (int part = 0; part < PLAN_PU_PARTS; part++) {
    const uint32_t i0 = (uint32_t)((uint64_t)pic->n_pu * part / PLAN_PU_PARTS), i1 = (uint32_t)((uint64_t)pic->n_pu * (part + 1) / PLAN_PU_PARTS);
    pl.run([&, part, i0, i1] {
      rc_pu[part] = plan_pus_part(pl, pic, L->mc_units, part, i0, i1);
      if (rc_pu[part]) err_pu[part] = g_err;  // the worker's thread-local message
    });
  }
  if (hb && !L->direct)
    for (int part = 0; part < 3; part++) pl.run([=] { pack_raw(pic, *L, hb, part); });
  pl.wait();
  for (int part = 0; part < PLAN_TU_PARTS; part++)
    if (rc_tv[part]) return set_err(rc_tv[part], "%s", err_tv[part].c_str());
  for (int part = 0; part < PLAN_PU_PARTS; part++)
    if (rc_pu[part]) return set_err(rc_pu[part], "%s", err_pu[part].c_str());
  plan_intra_finish(pl, pic, L, n_diag);
  merge_list_a(pl, L);
  const int rc = plan_pus_merge(pl, L);
  if (rc) return rc;
  plan_finish(L);
  if (hb) pack_lists(pl, *L, hb);
  return B200_OK;
}
