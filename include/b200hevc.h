/*
 * b200hevc.h — C ABI of the HEVC reconstruction engine for the H100 (sm_90a).
 *
 * This is the drop-in boundary for the per-CTB reconstruction hot path of
 * strukturag/libde265 (dequant + inverse DCT/DST + add-residual, luma/chroma MC
 * interpolation + weighted prediction, intra DC/planar/angular, deblocking, SAO).
 * NAL/CABAC parsing stays in the host decoder; the host *records* what it would
 * have reconstructed and the engine *replays* the records on the GPU.
 *
 * Two nested boundaries are exported (SURVEY.md §8b):
 *
 *   B2  per-picture execution boundary (this file, part 1 + 2): command records
 *       and b200_engine_*.  It replaces the reference's driver calls
 *         decode_TU                        libde265/slice.cc:3460
 *         generate_inter_prediction_samples libde265/motion.cc:288
 *         read_pcm_samples_internal        libde265/slice.cc:4211
 *         run_postprocessing_filters_*     libde265/decctx.cc:1783-1833
 *       The recorder (part 3, b200_rec_*) is what the reference-side hooks call.
 *
 *   B1  per-block DSP boundary (b200hevc_dsp.h): same contracts as the entries
 *       of `struct acceleration_functions` (libde265/acceleration.h:29-231).
 *
 * All structs are plain little-endian POD; no C++/torch types cross this ABI.
 * All functions return 0 on success or a negative B200_ERR_* code; nothing throws.
 */
#ifndef B200HEVC_H
#define B200HEVC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#define B200_ABI_VERSION 1

enum {
  B200_OK = 0,
  B200_ERR_INVALID = -1,     /* bad argument / malformed record */
  B200_ERR_CUDA = -2,        /* CUDA runtime error, see b200_last_error() */
  B200_ERR_NOMEM = -3,
  B200_ERR_UNSUPPORTED = -4, /* e.g. bit depth > 12 */
  B200_ERR_NO_DEVICE = -5    /* no CUDA device: the engine never falls back to the CPU */
};

/* DPB slots mirror libde265's decoded_picture_buffer indices (dpb.h:101, max 30). */
#define B200_MAX_SLOTS 32

/* ------------------------------------------------------------------------------------------
 * Part 1 — command records (SURVEY.md App. C.2)
 * ---------------------------------------------------------------------------------------- */

/* b200_pic_params.flags */
#define B200_PIC_SAO_ENABLED            0x0001 /* sps.sample_adaptive_offset_enabled_flag (sao.cc:333) */
#define B200_PIC_STRONG_INTRA_SMOOTHING 0x0002 /* sps.strong_intra_smoothing_enable_flag (intrapred.h:216) */
#define B200_PIC_PCM_LF_DISABLE         0x0004 /* informational; folded into nofilt_map by the host */
#define B200_PIC_LF_ACROSS_TILES        0x0008 /* pps.loop_filter_across_tiles_enabled_flag (sao.cc:157) */
#define B200_PIC_INTRA_SMOOTHING_OFF    0x0010 /* sps.range_extension.intra_smoothing_disabled_flag (intrapred.cc:289) */
#define B200_PIC_SKIP_DEBLOCK           0x0020 /* DE265_DECODER_PARAM_DISABLE_DEBLOCKING or no slice enables it (deblock.cc:914) */
#define B200_PIC_SKIP_SAO               0x0040 /* DE265_DECODER_PARAM_DISABLE_SAO (decctx.cc:1798) */
#define B200_PIC_SCALING_LIST           0x0080 /* sps.scaling_list_enable_flag: b200_picture.scaling_factors is valid */
#define B200_PIC_RECORDS_PINNED         0x0100 /* the record arrays are page-locked (b200_host_alloc / cudaHostRegister) AND stay unchanged
                                                  until the picture has been reconstructed (b200_engine_wait_slot / _sync): the engine
                                                  uploads them straight from where they lie instead of through its staging copy */

typedef struct b200_pic_params {
  uint16_t width, height;      /* luma samples, sps.pic_{width,height}_in_luma_samples */
  uint8_t  chroma_format_idc;  /* 0 mono, 1 4:2:0, 2 4:2:2, 3 4:4:4 */
  uint8_t  bit_depth_luma;     /* 8..12 */
  uint8_t  bit_depth_chroma;
  uint8_t  log2_ctb_size;      /* 4..6 */
  uint16_t flags;              /* B200_PIC_* */
  int8_t   pps_cb_qp_offset;   /* pps.pic_cb_qp_offset (deblock.cc:673) */
  int8_t   pps_cr_qp_offset;
  uint8_t  dst_slot;           /* DPB slot that receives the finished picture */
  uint8_t  stop_after_stage;   /* 0 = run everything; else B200_STAGE_* (stage dump, SURVEY §5) */
  uint8_t  reserved[2];
  int32_t  poc;                /* informational */
} b200_pic_params;             /* 20 bytes */

enum {
  B200_STAGE_ALL = 0,
  B200_STAGE_INTER_PRED = 1,   /* MC + weighting only */
  B200_STAGE_RECON = 2,        /* + intra + residual ("pre-lf" in decctx.cc:1785) */
  B200_STAGE_DEBLOCK = 3       /* + deblocking ("pre-sao" in decctx.cc:1794) */
};

/* One prediction unit = one call of generate_inter_prediction_samples (motion.cc:288). */
#define B200_PU_PRED_L0   0x01
#define B200_PU_PRED_L1   0x02
#define B200_PU_WEIGHTED  0x04  /* explicit weighting, weights[wt_idx] (motion.cc:494,555,636) */

typedef struct b200_pu {
  uint16_t x, y;        /* luma position xP,yP */
  uint8_t  w, h;        /* luma size nPbW,nPbH (4..64) */
  uint8_t  flags;       /* B200_PU_* (after the identical-MV bi->uni collapse, motion.cc:348-357) */
  uint8_t  reserved;
  int8_t   ref_slot[2]; /* DPB slot per list; <0 => reference missing, predict mid-grey 1<<13 (motion.cc:362) */
  uint16_t wt_idx;      /* index into b200_picture.weights */
  int16_t  mv[2][2];    /* [list][x,y] quarter-sample units */
  uint32_t pad;
} b200_pu;              /* 24 bytes */

/* Explicit weighted-prediction parameters, already resolved per (slice, refIdx0, refIdx1)
 * exactly as motion.cc:518-529 / 585-600 compute them (offsets pre-shifted by WpOffsetBdShift). */
typedef struct b200_weight_entry {
  int16_t w[2][3];      /* [list][cIdx] */
  int16_t o[2][3];
  uint8_t log2wd_luma;  /* luma_log2_weight_denom + shift1 */
  uint8_t log2wd_chroma;
  uint8_t pad[2];
} b200_weight_entry;    /* 28 bytes */

/* One transform unit = one call of decode_TU (slice.cc:3460). */
#define B200_TU_INTRA        0x0001 /* run intra prediction first (cuPredMode==MODE_INTRA) */
#define B200_TU_CBF          0x0002 /* residual present -> scale_coefficients (transform.cc:645) */
#define B200_TU_TSKIP        0x0004 /* transform_skip_flag */
#define B200_TU_BYPASS       0x0008 /* cu_transquant_bypass_flag */
#define B200_TU_RDPCM_H      0x0010 /* rdpcmMode==1 */
#define B200_TU_RDPCM_V      0x0020 /* rdpcmMode==2 */
#define B200_TU_DST          0x0040 /* trType==1: 4x4 luma of intra CU (transform.cc:601-606) */
#define B200_TU_NO_BOUNDARY_FILTER 0x0080 /* disableIntraBoundaryFilter (intrapred.cc:308-310) */
#define B200_TU_PCM          0x0100 /* raw samples: coeff level = sample already shifted (slice.cc:4211-4255) */
#define B200_TU_ROTATE       0x0200 /* RExt transform_skip_rotation (transform.cc:402-404) */
#define B200_TU_SCALING_LIST 0x0400 /* use scaling_factors[matrix] (transform.cc:489-525) */
#define B200_TU_INTER_MATRIX 0x0800 /* scaling list matrixID for non-intra CU (+3 / +1) */

typedef struct b200_tu {
  uint16_t x, y;        /* position in *component* samples (x0,y0 of decode_TU) */
  uint8_t  log2_size;   /* 2..5 */
  uint8_t  cidx;        /* 0 Y, 1 Cb, 2 Cr */
  uint16_t flags;       /* B200_TU_* */
  uint8_t  intra_mode;  /* 0 planar, 1 DC, 2..34 angular */
  uint8_t  qp;          /* qP{Y,Cb,Cr}Prime of the TU (transform.cc:371-377) */
  uint16_t n_coeff;     /* entries in coeffs[] starting at coeff_off */
  uint32_t coeff_off;
  uint64_t avail;       /* intra neighbour availability, see below */
} b200_tu;              /* 24 bytes */

/* Intra availability mask (replaces intra_border_computer::preproc/fill_from_image's
 * metadata tests, intrapred.h:436-633).  One bit per group of 4 border samples:
 *   bit k, k = 0..(nT/2-1)      : left column rows 4k..4k+3 below the TU's top edge,
 *                                 i.e. border[-4k-1 .. -4k-4] (k >= nT/4 is the bottom-left part)
 *   bit 16                      : top-left corner border[0]
 *   bit 17+k, k = 0..(nT/2-1)   : top row columns 4k..4k+3, i.e. border[4k+1 .. 4k+4]
 *                                 (k >= nT/4 is the top-right part)
 * where border[] is indexed as in intrapred.h (border[-k] = left column going down,
 * border[+k] = top row going right). */
#define B200_AVAIL_CORNER_BIT 16
#define B200_AVAIL_TOP_BIT0   17

typedef struct b200_coeff {
  uint16_t pos;         /* x + y*nT (coeffPos, slice.cc:3445) */
  int16_t  level;       /* coeffList value (already clipped to int16 by the parser) */
} b200_coeff;           /* 4 bytes */

/* Per slice segment header (deblock.cc:521-523, sao.cc:143-152,305-311). */
#define B200_SLICE_DEBLOCK_DISABLED  0x01
#define B200_SLICE_LF_ACROSS_SLICES  0x02
#define B200_SLICE_SAO_LUMA          0x04
#define B200_SLICE_SAO_CHROMA        0x08

typedef struct b200_slice_info {
  uint32_t slice_addr_rs;   /* SliceAddrRS */
  int8_t   beta_offset;     /* slice_beta_offset (already *2) */
  int8_t   tc_offset;       /* slice_tc_offset   (already *2) */
  uint8_t  flags;           /* B200_SLICE_* */
  uint8_t  pad;
} b200_slice_info;          /* 8 bytes */

/* Per CTB (image.h:160-170, slice.h:268-276). */
typedef struct b200_ctb_info {
  uint16_t slice_idx;       /* SliceHeaderIndex -> b200_picture.slices[] */
  uint16_t tile_id;         /* pps.scan->TileIdRS[ctb] */
  uint8_t  sao_type;        /* (SaoTypeIdx >> 2*cIdx) & 3 : 0 off, 1 band, 2 edge */
  uint8_t  sao_eo_class;    /* (SaoEoClass >> 2*cIdx) & 3 */
  uint8_t  sao_band_pos[3];
  int8_t   sao_offset[3][4];/* saoOffsetVal[cIdx][0..3], pre-scaled (slice.cc:2853) */
  uint8_t  pad[3];
} b200_ctb_info;            /* 24 bytes */

/* bs_map: one byte per 4x4 luma unit, row-major, width = ceil(W/4):
 *   bits 0-1 boundary strength of the vertical edge at the unit's left border,
 *   bits 2-3 boundary strength of the horizontal edge at the unit's top border,
 * i.e. the value derive_boundaryStrength (deblock.cc:243-383) stores with
 * vertical=true resp. vertical=false.  Edges off the 8x8 luma grid are ignored. */
#define B200_BS_V(b) ((b) & 3)
#define B200_BS_H(b) (((b) >> 2) & 3)

/* Everything the engine needs to reconstruct one picture.  All pointers are HOST
 * pointers (pinned or pageable); the engine copies them to the device. */
typedef struct b200_picture {
  b200_pic_params          params;
  uint32_t                 n_pu, n_weights, n_tu, n_coeff, n_slices;
  const b200_pu*           pus;
  const b200_weight_entry* weights;
  const b200_tu*           tus;          /* any order; the engine groups by CTB keeping relative order */
  const b200_coeff*        coeffs;
  const b200_slice_info*   slices;
  const b200_ctb_info*     ctbs;         /* PicWidthInCtbs * PicHeightInCtbs, raster order */
  const uint8_t*           bs_map;       /* ceil(W/4)*ceil(H/4); may be NULL if deblocking skipped */
  const int8_t*            qp_map;       /* QP_Y per 8x8 luma block, ceil(W/8)*ceil(H/8) */
  const uint8_t*           nofilt_map;   /* per 8x8: bit0 = (pcm && pcm_loop_filter_disable) || cu_transquant_bypass */
  const uint8_t*           scaling_factors; /* B200_SCALING_FACTOR_BYTES or NULL; read only under B200_PIC_SCALING_LIST */
} b200_picture;

/* scaling_factors layout: ScalingFactor_Size0[6][16], Size1[6][64], Size2[6][256], Size3[6][1024]
 * (pps.scaling_list, transform.cc:502-506), concatenated. */
#define B200_SCALING_FACTOR_BYTES (6*16 + 6*64 + 6*256 + 6*1024)

/* ------------------------------------------------------------------------------------------
 * Part 2 — engine (one per decoder context; single owner thread like de265_decoder_context)
 * ---------------------------------------------------------------------------------------- */

typedef struct b200_engine b200_engine;

/* device: CUDA ordinal. Fails with B200_ERR_NO_DEVICE when no GPU is present. */
B200_API int  b200_engine_create(b200_engine** out, int device);
B200_API void b200_engine_destroy(b200_engine*);

/* Asynchronously: upload the records, run inter-pred -> recon -> deblock -> SAO on the
 * engine's stream, leaving the picture resident in DPB slot params.dst_slot. */
B200_API int  b200_engine_submit_picture(b200_engine*, const b200_picture*);

/* Asynchronous submission: queues the picture and returns; planner threads validate / plan / pack whole pictures in parallel and one
 * sequencer thread issues them to the GPU in submission order, exactly as b200_engine_submit_picture would (same stream placement,
 * same results).  The record ARRAYS the picture points to must stay valid until the picture has been issued: until b200_engine_flush,
 * _sync or _read_slot returns, or b200_engine_wait_ticket of the picture's ticket, or b200_engine_wait_slot of its OWN destination slot
 * (with B200_PIC_RECORDS_PINNED: until the picture has been reconstructed, i.e. _sync / _wait_slot); the b200_picture struct itself is
 * copied.  b200_engine_read_slot_async calls are queued behind the pictures submitted
 * before them.  Errors of queued pictures (malformed records) are reported by the next flush / sync: the picture is skipped.
 * For hosts that produce pictures faster than one thread can plan them (parallel parsers, cached records, bench.py e2e). */
B200_API int  b200_engine_submit_picture_async(b200_engine*, const b200_picture*);
/* Blocks until everything queued has been issued to the GPU (not until the GPU has finished: see b200_engine_sync). */
B200_API int  b200_engine_flush(b200_engine*);
/* Tickets: every queued command (picture, read-back) gets the next number.  b200_engine_last_ticket returns the one queued last;
 * b200_engine_wait_ticket returns when every command up to the ticket has been issued — from then on the record arrays of those
 * pictures are no longer read by the engine's host side (a recorder with a ring of buffers waits for the ticket of the picture
 * that used a buffer last, not for the whole queue).  b200_engine_wait_slot only waits for the commands that touch its slot. */
B200_API unsigned long long b200_engine_last_ticket(b200_engine*);
B200_API int  b200_engine_wait_ticket(b200_engine*, unsigned long long ticket);

/* Prepared pictures: validate + upload the records ONCE and keep them resident in HBM; running a prepared
 * picture only launches the kernels (bench.py `value`: inputs already resident when the timed region starts;
 * also the replay path for cached pictures).  A prepared picture keeps its own device arena until freed. */
typedef struct b200_prepared b200_prepared;
B200_API int  b200_engine_prepare_picture(b200_engine*, const b200_picture*, b200_prepared** out);
B200_API int  b200_engine_run_prepared(b200_engine*, b200_prepared*);
B200_API void b200_engine_free_prepared(b200_engine*, b200_prepared*);

/* Fill a slot with a constant (generate_unavailable_reference_picture, decctx.cc:1294). */
B200_API int  b200_engine_fill_slot(b200_engine*, int slot, const b200_pic_params*, int value_y, int value_c);

/* Upload host planes into a slot (tests / reference pictures produced elsewhere).
 * Strides in BYTES, as de265_get_image_plane reports them (de265.cc:747-752). */
B200_API int  b200_engine_upload_slot(b200_engine*, int slot, const b200_pic_params*,
                                      const void* const planes[3], const size_t strides[3]);

/* Device->host copy of a finished slot (blocks until the picture is complete). */
B200_API int  b200_engine_read_slot(b200_engine*, int slot, void* const planes[3], const size_t strides[3]);

/* Async variant + explicit wait (lets the host parse picture N+1 meanwhile). */
B200_API int  b200_engine_read_slot_async(b200_engine*, int slot, void* const planes[3], const size_t strides[3]);
B200_API int  b200_engine_sync(b200_engine*);
/* Blocks until everything issued so far that writes or reads `slot` has finished (the picture in it is complete and every
 * b200_engine_read_slot_async and b200_engine_export_slot of it has landed), without waiting for later pictures in other slots: what a decoder calls when it
 * hands a picture to the application (push_picture_to_output_queue / de265_get_next_picture, decctx.cc:1842-1881). */
B200_API int  b200_engine_wait_slot(b200_engine*, int slot);
/* Page-locked host memory for picture planes that b200_engine_read_slot_async fills without staging (the reference-side binding
 * installs them through libde265's de265_image_allocation plug-in, de265.h:350-365). */
B200_API void* b200_host_alloc(size_t bytes);
B200_API void  b200_host_free(void* p);

/* Device pointers of a slot (zero-copy consumers, bench).
 * Unordered: nothing waits for the picture that writes the slot, and later pictures may overwrite or move the surface while the
 * caller reads it; use b200_engine_export_slot for an ordered copy. */
B200_API int  b200_engine_slot_device_planes(b200_engine*, int slot, void* planes[3], size_t strides[3]);

/* Export of a decoded picture into caller-owned CUDA memory (b200_engine_export_slot). */
#define B200_EXPORT_YUV         0  /* planar Y, Cb, Cr in the picture's own sample type (1 byte <= 8 bit, 2 bytes LE above) */
#define B200_EXPORT_RGB_BT601   1  /* planar R, G, B, 8 bit */
#define B200_EXPORT_RGB_BT709   2
#define B200_EXPORT_RGB_BT2020  3  /* non-constant luminance */
#define B200_EXPORT_FULL_RANGE  0x01  /* b200_export.flags: full-range input (default: limited / "video" range); RGB only, YUV ignores it */

typedef struct b200_export {
  uint16_t x, y, width, height;  /* crop window in luma samples; 4:2:0: all four even */
  uint8_t  format;               /* B200_EXPORT_* */
  uint8_t  flags;
  uint8_t  reserved[2];          /* must be 0 */
} b200_export;                   /* 12 bytes */

/* Enqueue on `stream` (a cudaStream_t on the engine's device; NULL = the legacy default stream) a copy of the crop window of
 * the picture named `slot` into caller-owned device memory: dst[c] / dst_pitch[c] (bytes) per output plane (YUV: Y, Cb, Cr;
 * only Y for 4:0:0; RGB: R, G, B).  Returns once the work is enqueued.  Work the caller enqueues on `stream` afterwards sees
 * the exported picture, and later pictures, fill_slot or upload_slot that write the surface wait for the export.
 * RGB: nearest chroma (pixel (x, y) takes chroma sample (x >> 1, y >> 1)), integer arithmetic (libde265_b200/csrc/export.cuh).
 * With b200_engine_submit_picture_async the call blocks until the slot's picture has been issued to the GPU (not until it is
 * finished), like b200_engine_wait_slot.  A picture damaged by a given-up intra dependency wait is exported as it is; the error
 * is reported by the next b200_engine_sync / _wait_slot / _read_slot.  b200_engine_wait_slot and _sync also wait for the
 * exports of the slot / of every slot.  Invalid arguments return B200_ERR_INVALID and leave the engine usable. */
B200_API int  b200_engine_export_slot(b200_engine*, int slot, const b200_export*, void* const dst[3], const size_t dst_pitch[3], void* stream);

/* Timing of the last submitted picture in milliseconds per stage (CUDA events on the
 * engine stream): [0] H2D, [1] inter pred, [2] recon, [3] deblock V+H, [4] SAO, [5] total.
 * Only recorded when enabled. */
B200_API int  b200_engine_enable_timing(b200_engine*, int on);
B200_API int  b200_engine_last_timing(b200_engine*, float ms[6]);
/* Sum of the per-stage times over the (up to 256 most recent) pictures submitted since timing was enabled /
 * last reset; *n_pictures receives how many pictures the sums cover.  Blocks until they have finished. */
B200_API int  b200_engine_timing_sum(b200_engine*, float ms[6], int* n_pictures, int reset);
/* Number of kernels this engine has launched so far (bench.py "gpu_launches"). */
B200_API uint64_t b200_engine_launch_count(const b200_engine*);

/* Picture-level pipelining.  The engine issues pictures onto `n` CUDA streams (default 8, 1..12; environment B200_STREAMS overrides
 * the default) plus two more for pictures that read no reference, placed by dependency depth, and orders them with per-surface
 * events: a picture waits for the writers of the slots it references; a destination slot that earlier pictures still read or write
 * is renamed to an idle surface (DESIGN.md 3), so only true dependencies order pictures and pictures that do not depend on each
 * other overlap on the GPU, in the spirit of libde265 decoding several images at once (decctx.h:334 image_units, WPP /
 * frame-parallel slice threads).  Results do not depend on n.  While per-stage timing is enabled all pictures go to stream 0. */
B200_API int  b200_engine_set_streams(b200_engine*, int n);
/* Raw CUDA stream handle (cudaStream_t) of stream 0 so callers can bracket with their own events ... */
B200_API void* b200_engine_stream(b200_engine*);
/* ... after making stream 0 wait for everything issued so far on the other streams. */
B200_API int  b200_engine_join(b200_engine*);

/* Host-side planner without a device (diagnostics / tests of the host logic on machines without a GPU): runs the planning
 * b200_engine_submit_picture runs, under the planner switches b200_engine_create reads (B200_REGION, B200_INTRA_ORDER,
 * B200_INTRA_SPLIT, B200_MC_LEGACY), and returns the work lists the kernels would consume.
 * counts[8] = { n_mc_units, n_list_a, n_list_a_warp_class, n_list_a_8x8_class, n_list_b, n_tasks, ref_slot_mask, 0 }.
 * Each output array may be NULL; otherwise it must hold cap_* entries and receives min(count, cap) of them:
 *   mc_units   one word per MC unit, bits 0-19 the PU index, the rest the unit's position in the PU.  8 bit: <= 16x16 tiles tagged
 *              with their class (bits 24-26), sorted into class-pure batches padded with 0xFFFFFFFF; > 8 bit: plain <= 16x16
 *              tiles; with B200_MC_LEGACY=1 (8 bit): <= 8x16 units
 *   list_a     indices of the non-intra TUs with work: warp class | 8x8 class | 4x4 class
 *   list_b     indices of the intra TUs grouped by task, tasks in the order the intra kernel claims them (topological)
 *   task_start n_tasks + 1 offsets into list_b */
B200_API int  b200_plan_picture_host(const b200_picture*, uint32_t counts[8], uint32_t* mc_units, size_t cap_units, uint32_t* list_a,
                                     size_t cap_a, uint32_t* list_b, size_t cap_b, uint32_t* task_start, size_t cap_tasks);

B200_API const char* b200_last_error(void);
B200_API int  b200_abi_version(void);

/* ------------------------------------------------------------------------------------------
 * Part 3 — recorder: what the reference-side hooks call while parsing (INTEGRATION.md)
 * ---------------------------------------------------------------------------------------- */

typedef struct b200_recorder b200_recorder;

B200_API int  b200_rec_create(b200_recorder** out);
B200_API void b200_rec_destroy(b200_recorder*);

/* Start a new picture; clears all per-picture buffers. */
B200_API int  b200_rec_begin_picture(b200_recorder*, const b200_pic_params*);
/* Returns the index of the appended slice (== SliceHeaderIndex order) or <0. */
B200_API int  b200_rec_add_slice(b200_recorder*, const b200_slice_info*);
B200_API int  b200_rec_add_weights(b200_recorder*, const b200_weight_entry*); /* returns wt_idx */
B200_API int  b200_rec_add_pu(b200_recorder*, const b200_pu*);
/* levels/positions exactly as thread_context::coeffList/coeffPos (decctx.h:85-92). */
B200_API int  b200_rec_add_tu(b200_recorder*, const b200_tu* tu /* coeff_off ignored */,
                              const int16_t* levels, const int16_t* positions, int n);
B200_API int  b200_rec_set_ctb(b200_recorder*, int ctb_x, int ctb_y, const b200_ctb_info*);
/* Dense maps are owned by the recorder; the hook fills them in place. */
B200_API uint8_t* b200_rec_bs_map(b200_recorder*);
B200_API int8_t*  b200_rec_qp_map(b200_recorder*);
B200_API uint8_t* b200_rec_nofilt_map(b200_recorder*);
B200_API int  b200_rec_set_scaling_factors(b200_recorder*, const uint8_t* factors);
/* Finish: fills *out with pointers into the recorder's buffers (valid until the next begin). */
B200_API int  b200_rec_end_picture(b200_recorder*, b200_picture* out);

/* Serialise / deserialise a finished picture (tests, golden fixtures, bench workloads). */
B200_API size_t b200_picture_serialized_size(const b200_picture*);
B200_API size_t b200_picture_serialize(const b200_picture*, void* buf, size_t cap);
/* Points *out into buf (no copy); returns bytes consumed or 0 on malformed input. */
B200_API size_t b200_picture_deserialize(const void* buf, size_t len, b200_picture* out);

#ifdef __cplusplus
}
#endif
#endif /* B200HEVC_H */
