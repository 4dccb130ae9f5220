// ref_replay.cc — record-replay executor over the UNMODIFIED reference's own reconstruction functions.
// TEST / BASELINE INFRASTRUCTURE ONLY (linked against oracle/_ref/libde265_ref.so, built from /root/reference by
// oracle/Makefile).  Nothing in the product path touches it.
//
// Why: the reference has no record replay and no 4K stream exists offline, so the CPU arm of bench.py (and a second,
// independent pin of the oracle's PICTURE-LEVEL driver) replays the very b200 command records the GPU engine consumes
// through the reference's own code:
//   PUs   -> generate_inter_prediction_samples            (motion.cc:288-707: mc_luma / mc_chroma edge handling, every
//            put_hevc_qpel / put_hevc_epel entry and the four weighting entries of the DSP table)
//   TUs   -> decode_intra_prediction + scale_coefficients (intrapred.cc:277-345, transform.cc:361-642: border availability
//            from the image's slice / tile / z-scan metadata, smoothing, prediction, dequant, IDCT/DST, skip, bypass, RDPCM)
//   PCM   -> the sample copy of read_pcm_samples_internal (slice.cc:4211-4255)
//   deblocking -> edge_filtering_luma / edge_filtering_chroma, all vertical edges then all horizontal (deblock.cc:908-946)
//   SAO   -> apply_sample_adaptive_offset_sequential      (sao.cc:327-382)
// dispatching through the DSP table base_context::set_acceleration_functions selects (decctx.cc:239-270):
// simd=0 the scalar fallback-*.cc table, simd=1 de265_acceleration_AUTO = SSE4.1 + AVX2 + AVX-512 on this host
// (x86/sse.cc:86-169) — "the reference's own SSE path" of BASELINE.json.  Parsing (CABAC) is NOT part of it: the replay
// is the reference's reconstruction work only, i.e. the same work the GPU engine does.
//
// Interface mirrors the oracle's (orc_create / orc_reconstruct / orc_upload_slot / orc_read_slot / orc_fill_slot).
#include <stdint.h>
#include <string.h>

#include <memory>
#include <vector>

#include "b200hevc.h"
#include "libde265/decctx.h"
#include "libde265/deblock.h"
#include "libde265/image.h"
#include "libde265/intrapred.h"
#include "libde265/motion.h"
#include "libde265/pps.h"
#include "libde265/sao.h"
#include "libde265/slice.h"
#include "libde265/sps.h"
#include "libde265/transform.h"

// non-static in deblock.cc but not declared in deblock.h
void edge_filtering_luma(de265_image* img, bool vertical, int yStart, int yEnd, int xStart, int xEnd);
void edge_filtering_chroma(de265_image* img, bool vertical, int yStart, int yEnd, int xStart, int xEnd);

#define EXPORT extern "C" __attribute__((visibility("default")))

namespace {

struct Replay : public base_context {
  decoder_context dctx;  // holder of the DSP table for the functions that go through img->decctx / tctx->decctx
  de265_image* slot[B200_MAX_SLOTS] = {};
  std::unique_ptr<thread_context> tctx;
  slice_segment_header pu_hdr;  // scratch header handed to generate_inter_prediction_samples, rewritten per PU
  bool constrained_intra = false;  // rr_set_options
  bool check_avail = false;
  struct {  // first intra TU of the last rr_reconstruct whose record mask differs from the reference's own
    bool found;
    uint32_t tu;
    uint64_t rec, ref;
  } mismatch = {};

  const de265_image* get_image(uint16_t id) const override { return id < B200_MAX_SLOTS ? slot[id] : nullptr; }
  bool has_image(uint16_t id) const override { return id < B200_MAX_SLOTS && slot[id] != nullptr; }
  ~Replay() override
  {
    for (auto& s : slot) delete s;
  }
};

struct Headers {
  std::shared_ptr<seq_parameter_set> sps;
  std::shared_ptr<pic_parameter_set> pps;
};

int make_headers(const b200_picture* pic, int tile_cols, int tile_rows, Headers* h)
{
  const b200_pic_params& p = pic->params;
  h->sps = std::make_shared<seq_parameter_set>();
  seq_parameter_set* sps = h->sps.get();
  sps->set_defaults();
  sps->pic_width_in_luma_samples = p.width;
  sps->pic_height_in_luma_samples = p.height;
  sps->chroma_format_idc = p.chroma_format_idc;
  sps->bit_depth_luma = p.bit_depth_luma;
  sps->bit_depth_chroma = p.bit_depth_chroma;
  sps->log2_min_luma_coding_block_size = 3;
  sps->log2_diff_max_min_luma_coding_block_size = p.log2_ctb_size - 3;
  sps->log2_min_transform_block_size = 2;
  sps->log2_diff_max_min_transform_block_size = (p.log2_ctb_size < 5 ? p.log2_ctb_size : 5) - 2;
  sps->max_transform_hierarchy_depth_inter = 1;
  sps->max_transform_hierarchy_depth_intra = 1;
  sps->sample_adaptive_offset_enabled_flag = (p.flags & B200_PIC_SAO_ENABLED) != 0;
  sps->strong_intra_smoothing_enable_flag = (p.flags & B200_PIC_STRONG_INTRA_SMOOTHING) != 0;
  sps->range_extension.intra_smoothing_disabled_flag = (p.flags & B200_PIC_INTRA_SMOOTHING_OFF) != 0;
  sps->pcm_loop_filter_disable_flag = 0;  // the records fold (pcm && pcm_loop_filter_disable) into the no-filter bit
  sps->scaling_list_enable_flag = (p.flags & B200_PIC_SCALING_LIST) && pic->scaling_factors;
  if (sps->compute_derived_values(true) != DE265_OK) return B200_ERR_INVALID;
  h->pps = std::make_shared<pic_parameter_set>();
  pic_parameter_set* pps = h->pps.get();
  pps->set_defaults();
  pps->sps = h->sps;
  pps->pic_cb_qp_offset = p.pps_cb_qp_offset;
  pps->pic_cr_qp_offset = p.pps_cr_qp_offset;
  pps->loop_filter_across_tiles_enabled_flag = (p.flags & B200_PIC_LF_ACROSS_TILES) != 0;
  pps->tiles_enabled_flag = tile_cols * tile_rows > 1;
  pps->num_tile_columns = tile_cols;
  pps->num_tile_rows = tile_rows;
  pps->uniform_spacing_flag = 1;
  pps->set_derived_values(sps);
  if (sps->scaling_list_enable_flag) {
    const uint8_t* f = pic->scaling_factors;
    memcpy(pps->scaling_list.ScalingFactor_Size0, f, 6 * 16);
    memcpy(pps->scaling_list.ScalingFactor_Size1, f + 6 * 16, 6 * 64);
    memcpy(pps->scaling_list.ScalingFactor_Size2, f + 6 * 16 + 6 * 64, 6 * 256);
    memcpy(pps->scaling_list.ScalingFactor_Size3, f + 6 * 16 + 6 * 64 + 6 * 256, 6 * 1024);
  }
  return B200_OK;
}

de265_chroma chroma_of(int idc)
{
  return idc == 0 ? de265_chroma_mono : idc == 1 ? de265_chroma_420 : idc == 2 ? de265_chroma_422 : de265_chroma_444;
}

// (Re)allocates the slot's image when the format changed; the samples of an existing image are kept.  A new CTB size alone
// keeps the samples too, but needs a new image: the per-CTB metadata is allocated for the CTB grid of the image's first SPS.
int ensure_slot(Replay* r, int s, const b200_pic_params& p, const std::shared_ptr<seq_parameter_set>& sps)
{
  de265_image*& img = r->slot[s];
  const bool same_format = img && img->get_width(0) == p.width && img->get_height(0) == p.height &&
                           img->get_chroma_format() == chroma_of(p.chroma_format_idc) && img->get_bit_depth(0) == p.bit_depth_luma &&
                           img->get_bit_depth(1) == p.bit_depth_chroma;
  if (same_format && img->number_of_ctbs() == (uint32_t)sps->PicSizeInCtbsY) return B200_OK;
  de265_image* fresh = new de265_image();
  if (fresh->alloc_image(p.width, p.height, chroma_of(p.chroma_format_idc), sps, true, &r->dctx, 0, nullptr, false) != DE265_OK) {
    delete fresh;
    return B200_ERR_NOMEM;
  }
  fresh->fill_image(0, 0, 0);  // new surfaces start at zero like the engine's and the oracle's
  if (same_format)
    for (int c = 0; c < (p.chroma_format_idc ? 3 : 1); c++) {
      const int bpp = img->get_bytes_per_pixel(c);
      for (int y = 0; y < img->get_height(c); y++)
        memcpy(fresh->get_image_plane(c) + (size_t)y * fresh->get_image_stride(c) * bpp,
               img->get_image_plane(c) + (size_t)y * img->get_image_stride(c) * bpp, (size_t)img->get_width(c) * bpp);
    }
  delete img;
  img = fresh;
  img->PicState = UsedForShortTermReference;
  return B200_OK;
}

// The availability mask of an intra TU as the reference derives it (intra_border_computer::preproc + fill_from_image,
// intrapred.h:436-633, from the image's slice / tile / z-scan metadata and, with constrained_intra_pred_flag, its
// prediction modes), packed like b200_tu.avail.  The sample values it gathers are ignored.
template <class pixel_t>
uint64_t reference_avail_mask(const de265_image* img, int xB, int yB, int nT, int cIdx)
{
  pixel_t border_mem[4 * MAX_INTRA_PRED_BLOCK_SIZE + 1];
  intra_border_computer<pixel_t> c;
  c.init(&border_mem[2 * MAX_INTRA_PRED_BLOCK_SIZE], img, nT, cIdx, xB, yB);
  c.preproc();
  c.fill_from_image();
  uint64_t m = 0;
  for (int k = 0; k < nT / 2; k++) {
    if (c.available[-4 * k - 1]) m |= 1ull << k;
    if (c.available[4 * k + 1]) m |= 1ull << (B200_AVAIL_TOP_BIT0 + k);
  }
  if (c.available[0]) m |= 1ull << B200_AVAIL_CORNER_BIT;
  return m;
}

int tile_grid(const b200_picture* pic, int* cols, int* rows)
{
  const b200_pic_params& p = pic->params;
  const int S = 1 << p.log2_ctb_size, wctb = (p.width + S - 1) / S, hctb = (p.height + S - 1) / S;
  int c = 1, r = 1;
  for (int x = 1; x < wctb; x++) c += pic->ctbs[x].tile_id != pic->ctbs[x - 1].tile_id;
  for (int y = 1; y < hctb; y++) r += pic->ctbs[y * wctb].tile_id != pic->ctbs[(y - 1) * wctb].tile_id;
  *cols = c;
  *rows = r;
  return B200_OK;
}

}  // namespace

EXPORT void* rr_create(int simd)
{
  Replay* r = new Replay();
  const de265_acceleration level = simd ? de265_acceleration_AUTO : de265_acceleration_SCALAR;
  r->set_acceleration_functions(level);
  r->dctx.set_acceleration_functions(level);
  r->tctx.reset(new thread_context());
  r->tctx->decctx = &r->dctx;
  return r;
}

EXPORT void rr_destroy(void* h) { delete (Replay*)h; }

// Present from the version whose ensure_slot reallocates a slot's image on a CTB-size change.  A library built from an older
// ref_replay.cc lacks it: it keeps the image, whose per-CTB metadata is then too small for a smaller CTB, and corrupts the heap.
EXPORT int rr_handles_ctb_change(void) { return 1; }

// constrained_intra: replay with constrained_intra_pred_flag set, so the reference derives the availability of every intra
// TU's neighbours from the prediction modes of the records (inter where a PU lies, intra where a luma intra / PCM TU lies).
// check_avail: fail rr_reconstruct on the first intra TU whose record mask differs from the one the reference derives
// (rr_avail_mismatch reports it).  Both are off after rr_create.
EXPORT int rr_set_options(void* h, int constrained_intra, int check_avail)
{
  Replay* r = (Replay*)h;
  if (!r) return B200_ERR_INVALID;
  r->constrained_intra = constrained_intra != 0;
  r->check_avail = check_avail != 0;
  return B200_OK;
}

// 1 when the last rr_reconstruct stopped at an availability mismatch: the TU's index, the record's and the reference's masks.
EXPORT int rr_avail_mismatch(void* h, uint32_t* tu, uint64_t* rec, uint64_t* ref)
{
  Replay* r = (Replay*)h;
  if (!r || !r->mismatch.found) return 0;
  *tu = r->mismatch.tu;
  *rec = r->mismatch.rec;
  *ref = r->mismatch.ref;
  return 1;
}

EXPORT int rr_fill_slot(void* h, int s, const b200_pic_params* p, int vy, int vc)
{
  Replay* r = (Replay*)h;
  if (!r || s < 0 || s >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  b200_picture tmp{};
  tmp.params = *p;
  Headers hd;
  int rc = make_headers(&tmp, 1, 1, &hd);
  if (rc) return rc;
  rc = ensure_slot(r, s, *p, hd.sps);
  if (rc) return rc;
  r->slot[s]->fill_image(vy, vc, vc);  // generate_unavailable_reference_picture's fill (decctx.cc:1308-1310)
  return B200_OK;
}

EXPORT int rr_upload_slot(void* h, int s, const b200_pic_params* p, const void* const planes[3], const size_t strides[3])
{
  Replay* r = (Replay*)h;
  if (!r || s < 0 || s >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  b200_picture tmp{};
  tmp.params = *p;
  Headers hd;
  int rc = make_headers(&tmp, 1, 1, &hd);
  if (rc) return rc;
  rc = ensure_slot(r, s, *p, hd.sps);
  if (rc) return rc;
  de265_image* img = r->slot[s];
  for (int c = 0; c < (p->chroma_format_idc ? 3 : 1); c++) {
    const int bpp = img->get_bytes_per_pixel(c);
    for (int y = 0; y < img->get_height(c); y++)
      memcpy(img->get_image_plane(c) + (size_t)y * img->get_image_stride(c) * bpp, (const uint8_t*)planes[c] + y * strides[c], (size_t)img->get_width(c) * bpp);
  }
  return B200_OK;
}

EXPORT int rr_read_slot(void* h, int s, void* const planes[3], const size_t strides[3])
{
  Replay* r = (Replay*)h;
  if (!r || s < 0 || s >= B200_MAX_SLOTS || !r->slot[s]) return B200_ERR_INVALID;
  de265_image* img = r->slot[s];
  for (int c = 0; c < (img->get_chroma_format() == de265_chroma_mono ? 1 : 3); c++) {
    if (!planes[c]) continue;
    const int bpp = img->get_bytes_per_pixel(c);
    for (int y = 0; y < img->get_height(c); y++)
      memcpy((uint8_t*)planes[c] + y * strides[c], img->get_image_plane(c) + (size_t)y * img->get_image_stride(c) * bpp, (size_t)img->get_width(c) * bpp);
  }
  return B200_OK;
}

EXPORT int rr_reconstruct(void* h, const b200_picture* pic)
{
  Replay* r = (Replay*)h;
  if (!r || !pic) return B200_ERR_INVALID;
  const b200_pic_params& p = pic->params;
  if (p.dst_slot >= B200_MAX_SLOTS) return B200_ERR_INVALID;
  int tcols = 1, trows = 1;
  tile_grid(pic, &tcols, &trows);
  Headers hd;
  int rc = make_headers(pic, tcols, trows, &hd);
  if (rc) return rc;
  rc = ensure_slot(r, p.dst_slot, p, hd.sps);
  if (rc) return rc;
  de265_image* img = r->slot[p.dst_slot];
  seq_parameter_set* sps = hd.sps.get();
  pic_parameter_set* pps = hd.pps.get();
  pps->constrained_intra_pred_flag = r->constrained_intra;
  r->mismatch.found = false;
  img->set_headers(nullptr, hd.sps, hd.pps);
  img->clear_metadata();
  img->integrity = INTEGRITY_CORRECT;

  // ---- picture metadata the reference's parser would have written (slice.cc read_coding_unit / read_sao) ----
  std::vector<std::unique_ptr<slice_segment_header>> hdrs;
  for (uint32_t i = 0; i < pic->n_slices; i++) {
    const b200_slice_info& s = pic->slices[i];
    hdrs.emplace_back(new slice_segment_header());
    slice_segment_header* sh = hdrs.back().get();
    sh->SliceAddrRS = s.slice_addr_rs;
    sh->slice_segment_address = s.slice_addr_rs;
    sh->slice_beta_offset = s.beta_offset;
    sh->slice_tc_offset = s.tc_offset;
    sh->slice_deblocking_filter_disabled_flag = (s.flags & B200_SLICE_DEBLOCK_DISABLED) != 0;
    sh->slice_loop_filter_across_slices_enabled_flag = (s.flags & B200_SLICE_LF_ACROSS_SLICES) != 0;
    sh->slice_sao_luma_flag = (s.flags & B200_SLICE_SAO_LUMA) != 0;
    sh->slice_sao_chroma_flag = (s.flags & B200_SLICE_SAO_CHROMA) != 0;
    img->add_slice_segment_header(sh);
  }
  struct SliceGuard {  // the image must not own (delete) our headers
    de265_image* i;
    ~SliceGuard() { i->slices.clear(); }
  } guard{img};
  const int S = 1 << p.log2_ctb_size, wctb = sps->PicWidthInCtbsY, hctb = sps->PicHeightInCtbsY;
  const int w8 = (p.width + 7) / 8, h8 = (p.height + 7) / 8, w4 = (p.width + 3) / 4, h4 = (p.height + 3) / 4;
  for (int cy = 0; cy < hctb; cy++)
    for (int cx = 0; cx < wctb; cx++) {
      const b200_ctb_info& ci = pic->ctbs[cx + cy * wctb];
      if (ci.slice_idx >= pic->n_slices) return B200_ERR_INVALID;
      if (ci.tile_id != pps->scan->TileIdRS[cx + cy * wctb]) return B200_ERR_UNSUPPORTED;  // only uniformly spaced tiles can be rebuilt
      img->set_SliceHeaderIndex(cx * S, cy * S, ci.slice_idx);
      img->set_SliceAddrRS(cx, cy, pic->slices[ci.slice_idx].slice_addr_rs);
      sao_info sao;
      sao.SaoTypeIdx = ci.sao_type;
      sao.SaoEoClass = ci.sao_eo_class;
      for (int c = 0; c < 3; c++) {
        sao.sao_band_position[c] = ci.sao_band_pos[c];
        for (int k = 0; k < 4; k++) sao.saoOffsetVal[c][k] = ci.sao_offset[c][k];
      }
      img->set_sao_info(cx, cy, &sao);
    }
  for (int y = 0; y < h8; y++)
    for (int x = 0; x < w8; x++) {
      img->set_QPY(8 * x, 8 * y, 3, pic->qp_map[x + y * w8]);
      if (pic->nofilt_map[x + y * w8] & 1) img->set_cu_transquant_bypass(8 * x, 8 * y, 3, 1);
    }

  // ---- inter prediction: one generate_inter_prediction_samples call per PU record ----
  {
    slice_segment_header& sh = r->pu_hdr;
    sh.slice_type = SLICE_TYPE_B;
    sh.pps = hd.pps;
    const int sh1_l = p.bit_depth_luma < 12 ? 14 - p.bit_depth_luma : 2, sh1_c = p.bit_depth_chroma < 12 ? 14 - p.bit_depth_chroma : 2;
    for (uint32_t i = 0; i < pic->n_pu; i++) {
      const b200_pu& pu = pic->pus[i];
      if (!(pu.flags & (B200_PU_PRED_L0 | B200_PU_PRED_L1))) continue;
      PBMotion vi;
      for (int l = 0; l < 2; l++) {
        vi.predFlag[l] = (pu.flags & (l ? B200_PU_PRED_L1 : B200_PU_PRED_L0)) ? 1 : 0;
        vi.refIdx[l] = 0;
        vi.mv[l].x = pu.mv[l][0];
        vi.mv[l].y = pu.mv[l][1];
        sh.RefPicList[l][0] = pu.ref_slot[l] >= 0 ? pu.ref_slot[l] : 0xFFFF;  // missing reference: no such image (motion.cc:387-391)
      }
      const bool wgt = pu.flags & B200_PU_WEIGHTED;
      pps->weighted_pred_flag = pps->weighted_bipred_flag = wgt;
      if (wgt) {
        if (pu.wt_idx >= pic->n_weights) return B200_ERR_INVALID;
        const b200_weight_entry& w = pic->weights[pu.wt_idx];
        sh.luma_log2_weight_denom = w.log2wd_luma - sh1_l;
        sh.ChromaLog2WeightDenom = w.log2wd_chroma - sh1_c;
        for (int l = 0; l < 2; l++) {
          sh.LumaWeight[l][0] = w.w[l][0];
          sh.luma_offset[l][0] = w.o[l][0] >> sps->WpOffsetBdShiftY;
          for (int c = 0; c < 2; c++) {
            sh.ChromaWeight[l][0][c] = w.w[l][1 + c];
            sh.ChromaOffset[l][0][c] = w.o[l][1 + c] >> sps->WpOffsetBdShiftC;
          }
        }
      }
      generate_inter_prediction_samples(r, &sh, img, pu.x, pu.y, 0, 0, 64, pu.w, pu.h, &vi);
    }
    sh.pps.reset();
  }
  if (p.stop_after_stage == B200_STAGE_INTER_PRED) return B200_OK;

  // ---- transform units in decode order: intra prediction, then the residual ----
  thread_context* t = r->tctx.get();
  t->img = img;
  t->ResScaleVal = 0;
  t->explicit_rdpcm_flag = 0;
  if (r->constrained_intra) {
    // The prediction mode of every 8x8 block, as read_coding_unit would have stored it: CUs are at least 8x8 and 8-aligned, so
    // each 8x8 belongs to one CU, inter where a PU lies, intra where a luma intra or PCM TU lies.
    for (uint32_t i = 0; i < pic->n_pu; i++) {
      const b200_pu& pu = pic->pus[i];
      for (int y = pu.y & ~7; y < pu.y + pu.h; y += 8)
        for (int x = pu.x & ~7; x < pu.x + pu.w; x += 8) img->set_pred_mode(x, y, 3, MODE_INTER);
    }
    for (uint32_t i = 0; i < pic->n_tu; i++) {
      const b200_tu& tu = pic->tus[i];
      if (tu.cidx || !(tu.flags & (B200_TU_INTRA | B200_TU_PCM))) continue;
      const int nT = 1 << tu.log2_size;
      for (int y = tu.y & ~7; y < tu.y + nT; y += 8)
        for (int x = tu.x & ~7; x < tu.x + nT; x += 8) img->set_pred_mode(x, y, 3, MODE_INTRA);
    }
  }
  for (uint32_t i = 0; i < pic->n_tu; i++) {
    const b200_tu& tu = pic->tus[i];
    const int nT = 1 << tu.log2_size, c = tu.cidx;
    if (tu.log2_size < 2 || tu.log2_size > 5 || c > 2 || (size_t)tu.coeff_off + tu.n_coeff > pic->n_coeff) return B200_ERR_INVALID;
    const b200_coeff* co = pic->coeffs + tu.coeff_off;
    if (tu.flags & B200_TU_PCM) {  // slice.cc:4211-4255: samples already shifted to the picture's bit depth
      const int bpp = img->get_bytes_per_pixel(c);
      uint8_t* base = img->get_image_plane(c);
      const ptrdiff_t stride = img->get_image_stride(c);
      for (int k = 0; k < tu.n_coeff; k++) {
        const size_t off = (size_t)(tu.x + co[k].pos % nT) + (size_t)(tu.y + co[k].pos / nT) * stride;
        if (bpp == 1) base[off] = (uint8_t)co[k].level;
        else ((uint16_t*)base)[off] = (uint16_t)co[k].level;
      }
      continue;
    }
    const int xl = tu.x << (c ? 1 : 0), yl = tu.y << (c ? 1 : 0);  // luma position of the TU (4:2:0)
    if (tu.flags & B200_TU_INTRA) {
      if (r->check_avail) {
        const uint64_t ref = img->high_bit_depth(c) ? reference_avail_mask<uint16_t>(img, tu.x, tu.y, nT, c)
                                                    : reference_avail_mask<uint8_t>(img, tu.x, tu.y, nT, c);
        if (ref != tu.avail) {
          r->mismatch = {true, i, tu.avail, ref};
          return B200_ERR_INVALID;
        }
      }
      // disableIntraBoundaryFilter = implicit_rdpcm_enabled_flag && cu_transquant_bypass at (xB0, yB0) (intrapred.cc:308-310)
      const bool nbf = tu.flags & B200_TU_NO_BOUNDARY_FILTER;
      sps->range_extension.implicit_rdpcm_enabled_flag = nbf;
      int saved = 0;
      if (nbf) { saved = img->get_cu_transquant_bypass(tu.x, tu.y); img->set_cu_transquant_bypass(tu.x & ~7, tu.y & ~7, 3, 1); }
      decode_intra_prediction(img, tu.x, tu.y, (enum IntraPredMode)tu.intra_mode, nT, c);
      if (nbf) img->set_cu_transquant_bypass(tu.x & ~7, tu.y & ~7, 3, saved);
      sps->range_extension.implicit_rdpcm_enabled_flag = 0;
    }
    if (!(tu.flags & B200_TU_CBF)) continue;
    // scale_coefficients reads the CU's prediction mode at (xT, yT) for the DST / rotation decisions (transform.cc:400-404,
    // 601-606) and the scaling-list matrix from its `intra` argument: make them say what the record says.  (At component
    // coordinates for chroma: with constrained_intra the 8x8's own mode is put back afterwards, later TUs read it.)
    const PredMode cu_mode = img->get_pred_mode(tu.x & ~7, tu.y & ~7);
    img->set_pred_mode(tu.x & ~7, tu.y & ~7, 3, (tu.flags & (B200_TU_DST | B200_TU_ROTATE)) ? MODE_INTRA : MODE_INTER);
    sps->range_extension.transform_skip_rotation_enabled_flag = (tu.flags & B200_TU_ROTATE) != 0;
    t->cu_transquant_bypass_flag = (tu.flags & B200_TU_BYPASS) != 0;
    t->qPYPrime = t->qPCbPrime = t->qPCrPrime = tu.qp;
    t->nCoeff[c] = tu.n_coeff;
    for (int k = 0; k < tu.n_coeff; k++) {
      t->coeffList[c][k] = co[k].level;
      t->coeffPos[c][k] = (int16_t)co[k].pos;
    }
    const bool matrix_intra = (tu.flags & B200_TU_SCALING_LIST) ? !(tu.flags & B200_TU_INTER_MATRIX) : (tu.flags & B200_TU_INTRA) != 0;
    const int rdpcm = (tu.flags & B200_TU_RDPCM_H) ? 1 : (tu.flags & B200_TU_RDPCM_V) ? 2 : 0;
    scale_coefficients(t, tu.x, tu.y, tu.x, tu.y, nT, c, (tu.flags & B200_TU_TSKIP) != 0, matrix_intra, rdpcm);
    if (r->constrained_intra) img->set_pred_mode(tu.x & ~7, tu.y & ~7, 3, cu_mode);
    (void)xl; (void)yl;
  }
  sps->range_extension.transform_skip_rotation_enabled_flag = 0;
  if (p.stop_after_stage == B200_STAGE_RECON) return B200_OK;

  // ---- deblocking: bS from the records (what derive_boundaryStrength stored), the reference's edge filters ----
  if (!(p.flags & B200_PIC_SKIP_DEBLOCK) && pic->bs_map) {
    for (int pass = 0; pass < 2; pass++) {
      const bool vertical = pass == 0;
      for (int y = 0; y < h4; y++)
        for (int x = 0; x < w4; x++) {
          const uint8_t b = pic->bs_map[x + y * w4];
          img->set_deblk_bS(4 * x, 4 * y, vertical ? B200_BS_V(b) : B200_BS_H(b));
        }
      edge_filtering_luma(img, vertical, 0, img->get_deblk_height(), 0, img->get_deblk_width());
      if (p.chroma_format_idc) edge_filtering_chroma(img, vertical, 0, img->get_deblk_height(), 0, img->get_deblk_width());
    }
  }
  if (p.stop_after_stage == B200_STAGE_DEBLOCK) return B200_OK;
  if ((p.flags & B200_PIC_SAO_ENABLED) && !(p.flags & B200_PIC_SKIP_SAO)) apply_sample_adaptive_offset_sequential(img);
  return B200_OK;
}
