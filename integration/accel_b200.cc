// accel_b200.cc — reference-side binding of boundary B1 (include/b200hevc_dsp.h).
//
// Compiled INTO libde265 (it includes libde265's internal headers).  init_acceleration_functions_b200 overrides the
// entries of `struct acceleration_functions` (acceleration.h:29-231) with wrappers that run on the GPU through
// b200_dsp_run_batch, in the same way init_acceleration_functions_sse overrides the scalar table (decctx.cc:243-269):
// call init_acceleration_functions_fallback first, then this.  Every wrapper issues a batch of ONE command and
// returns when the host buffers hold the result, so the table keeps its synchronous per-block contract; that makes it
// a parity boundary (the unmodified reference decode loop + these entries reproduces the golden output), not the
// throughput path — see INTEGRATION.md.  One b200_dsp context per thread (the table is called concurrently from the
// decoder's worker threads and must be stateless towards its callers).
#include <cstdio>
#include <cstdlib>

#include "libde265/acceleration.h"
#include "libde265/decctx.h"
#include "libde265/fallback.h"
#include "b200hevc_dsp.h"

namespace {

b200_dsp* ctx()
{
  static thread_local b200_dsp* d = nullptr;
  if (!d && b200_dsp_create(&d, 0) != 0) {
    fprintf(stderr, "accel_b200: %s\n", b200_last_error());
    abort();  // the table has no error return; without a device there is nothing to fall back to by design
  }
  return d;
}

void run(b200_dsp_cmd& c)
{
  if (b200_dsp_run_batch(ctx(), &c, 1) != 0) {
    fprintf(stderr, "accel_b200: %s\n", b200_last_error());
    abort();
  }
}

b200_dsp_cmd cmd(int op, int bd, void* dst, ptrdiff_t dststride, const void* src, const void* src2, ptrdiff_t srcstride, int w, int h)
{
  b200_dsp_cmd c = {};
  c.op = op; c.bit_depth = bd; c.dst = dst; c.dststride = dststride; c.src = src; c.src2 = src2; c.srcstride = srcstride; c.w = w; c.h = h;
  return c;
}

// ---- motion compensation ----
template <int XF, int YF>
void qpel8(int16_t* dst, ptrdiff_t ds, const uint8_t* src, ptrdiff_t ss, int w, int h, int16_t*)
{
  b200_dsp_cmd c = cmd(B200_DSP_QPEL, 8, dst, ds, src, nullptr, ss, w, h);
  c.a[0] = XF; c.a[1] = YF;
  run(c);
}
template <int XF, int YF>
void qpel16(int16_t* dst, ptrdiff_t ds, const uint16_t* src, ptrdiff_t ss, int w, int h, int16_t*, int bd)
{
  b200_dsp_cmd c = cmd(B200_DSP_QPEL, bd, dst, ds, src, nullptr, ss, w, h);
  c.a[0] = XF; c.a[1] = YF;
  run(c);
}
void epel8(int16_t* dst, ptrdiff_t ds, const uint8_t* src, ptrdiff_t ss, int w, int h, int mx, int my, int16_t*)
{
  b200_dsp_cmd c = cmd(B200_DSP_EPEL, 8, dst, ds, src, nullptr, ss, w, h);
  c.a[0] = mx; c.a[1] = my;
  run(c);
}
void epel8b(int16_t* dst, ptrdiff_t ds, const uint8_t* src, ptrdiff_t ss, int w, int h, int mx, int my, int16_t* mcb, int) { epel8(dst, ds, src, ss, w, h, mx, my, mcb); }
void epel16(int16_t* dst, ptrdiff_t ds, const uint16_t* src, ptrdiff_t ss, int w, int h, int mx, int my, int16_t*, int bd)
{
  b200_dsp_cmd c = cmd(B200_DSP_EPEL, bd, dst, ds, src, nullptr, ss, w, h);
  c.a[0] = mx; c.a[1] = my;
  run(c);
}

// ---- weighting ----
void uni8(uint8_t* d, ptrdiff_t ds, const int16_t* s, ptrdiff_t ss, int w, int h) { b200_dsp_cmd c = cmd(B200_DSP_PRED_UNI, 8, d, ds, s, nullptr, ss, w, h); run(c); }
void uni16(uint16_t* d, ptrdiff_t ds, const int16_t* s, ptrdiff_t ss, int w, int h, int bd) { b200_dsp_cmd c = cmd(B200_DSP_PRED_UNI, bd, d, ds, s, nullptr, ss, w, h); run(c); }
void avg8(uint8_t* d, ptrdiff_t ds, const int16_t* s1, const int16_t* s2, ptrdiff_t ss, int w, int h) { b200_dsp_cmd c = cmd(B200_DSP_PRED_AVG, 8, d, ds, s1, s2, ss, w, h); run(c); }
void avg16(uint16_t* d, ptrdiff_t ds, const int16_t* s1, const int16_t* s2, ptrdiff_t ss, int w, int h, int bd) { b200_dsp_cmd c = cmd(B200_DSP_PRED_AVG, bd, d, ds, s1, s2, ss, w, h); run(c); }
void wp8(uint8_t* d, ptrdiff_t ds, const int16_t* s, ptrdiff_t ss, int w, int h, int wt, int o, int wd)
{
  b200_dsp_cmd c = cmd(B200_DSP_PRED_WEIGHTED, 8, d, ds, s, nullptr, ss, w, h);
  c.a[0] = wt; c.a[1] = o; c.a[2] = wd;
  run(c);
}
void wp16(uint16_t* d, ptrdiff_t ds, const int16_t* s, ptrdiff_t ss, int w, int h, int wt, int o, int wd, int bd)
{
  b200_dsp_cmd c = cmd(B200_DSP_PRED_WEIGHTED, bd, d, ds, s, nullptr, ss, w, h);
  c.a[0] = wt; c.a[1] = o; c.a[2] = wd;
  run(c);
}
void bi8(uint8_t* d, ptrdiff_t ds, const int16_t* s1, const int16_t* s2, ptrdiff_t ss, int w, int h, int w1, int o1, int w2, int o2, int wd)
{
  b200_dsp_cmd c = cmd(B200_DSP_PRED_WEIGHTED_BI, 8, d, ds, s1, s2, ss, w, h);
  c.a[0] = w1; c.a[1] = o1; c.a[2] = w2; c.a[3] = o2; c.a[4] = wd;
  run(c);
}
void bi16(uint16_t* d, ptrdiff_t ds, const int16_t* s1, const int16_t* s2, ptrdiff_t ss, int w, int h, int w1, int o1, int w2, int o2, int wd, int bd)
{
  b200_dsp_cmd c = cmd(B200_DSP_PRED_WEIGHTED_BI, bd, d, ds, s1, s2, ss, w, h);
  c.a[0] = w1; c.a[1] = o1; c.a[2] = w2; c.a[3] = o2; c.a[4] = wd;
  run(c);
}

// ---- residual ----
template <int LOG2>
void tr8(uint8_t* d, const int16_t* co, ptrdiff_t st) { b200_dsp_cmd c = cmd(B200_DSP_TRANSFORM_ADD, 8, d, st, co, nullptr, 0, 0, 0); c.a[0] = LOG2; run(c); }
template <int LOG2>
void tr16(uint16_t* d, const int16_t* co, ptrdiff_t st, int bd) { b200_dsp_cmd c = cmd(B200_DSP_TRANSFORM_ADD, bd, d, st, co, nullptr, 0, 0, 0); c.a[0] = LOG2; run(c); }
void dst8(uint8_t* d, const int16_t* co, ptrdiff_t st) { b200_dsp_cmd c = cmd(B200_DSP_DST_ADD, 8, d, st, co, nullptr, 0, 0, 0); run(c); }
void dst16(uint16_t* d, const int16_t* co, ptrdiff_t st, int bd) { b200_dsp_cmd c = cmd(B200_DSP_DST_ADD, bd, d, st, co, nullptr, 0, 0, 0); run(c); }

// ---- intra ----
template <class P>
void intra(int op, P* d, ptrdiff_t st, int bd, int nT, int cIdx, const P* border, int mode = 0, int nofilt = 0)
{
  b200_dsp_cmd c = cmd(op, bd, d, st, border, nullptr, 0, 0, 0);
  c.a[0] = nT; c.a[1] = cIdx; c.a[2] = mode; c.a[3] = nofilt;
  run(c);
}
void dc8(uint8_t* d, ptrdiff_t st, int nT, int cIdx, const uint8_t* b) { intra(B200_DSP_INTRA_DC, d, st, 8, nT, cIdx, b); }
void planar8(uint8_t* d, ptrdiff_t st, int nT, int cIdx, const uint8_t* b) { intra(B200_DSP_INTRA_PLANAR, d, st, 8, nT, cIdx, b); }
void ang8(uint8_t* d, ptrdiff_t st, int bd, int nofilt, int, int, int m, int nT, int cIdx, const uint8_t* b) { intra(B200_DSP_INTRA_ANGULAR, d, st, bd, nT, cIdx, b, m, nofilt); }
// the _16 DC / planar entries carry no bit depth (they do not clip): any depth > 8 selects the 16-bit sample type
void dc16(uint16_t* d, ptrdiff_t st, int nT, int cIdx, const uint16_t* b) { intra(B200_DSP_INTRA_DC, d, st, 12, nT, cIdx, b); }
void planar16(uint16_t* d, ptrdiff_t st, int nT, int cIdx, const uint16_t* b) { intra(B200_DSP_INTRA_PLANAR, d, st, 12, nT, cIdx, b); }
void ang16(uint16_t* d, ptrdiff_t st, int bd, int nofilt, int, int, int m, int nT, int cIdx, const uint16_t* b) { intra(B200_DSP_INTRA_ANGULAR, d, st, bd, nT, cIdx, b, m, nofilt); }

// ---- deblocking ----
void dbl8(uint8_t* p, ptrdiff_t st, int vertical, int dE, int dEp, int dEq, int tc, int fP, int fQ)
{
  b200_dsp_cmd c = cmd(B200_DSP_DEBLOCK_LUMA, 8, p, st, nullptr, nullptr, 0, 0, 0);
  c.a[0] = vertical; c.a[1] = dE; c.a[2] = dEp; c.a[3] = dEq; c.a[4] = tc; c.a[5] = fP; c.a[6] = fQ;
  run(c);
}
void dbc8(uint8_t* p, ptrdiff_t st, int vertical, int tc, int fP, int fQ)
{
  b200_dsp_cmd c = cmd(B200_DSP_DEBLOCK_CHROMA, 8, p, st, nullptr, nullptr, 0, 0, 0);
  c.a[0] = vertical; c.a[1] = tc; c.a[2] = fP; c.a[3] = fQ;
  run(c);
}

template <int X>
void fill_qpel_row(acceleration_functions* a)
{
  a->put_hevc_qpel_8[X][0] = qpel8<X, 0>; a->put_hevc_qpel_8[X][1] = qpel8<X, 1>; a->put_hevc_qpel_8[X][2] = qpel8<X, 2>; a->put_hevc_qpel_8[X][3] = qpel8<X, 3>;
  a->put_hevc_qpel_16[X][0] = qpel16<X, 0>; a->put_hevc_qpel_16[X][1] = qpel16<X, 1>; a->put_hevc_qpel_16[X][2] = qpel16<X, 2>; a->put_hevc_qpel_16[X][3] = qpel16<X, 3>;
}

}  // namespace

// Same contract as init_acceleration_functions_sse (x86/sse.h): the table has been filled by
// init_acceleration_functions_fallback before; entries this file does not provide stay scalar.
void init_acceleration_functions_b200(struct acceleration_functions* a)
{
  fill_qpel_row<0>(a); fill_qpel_row<1>(a); fill_qpel_row<2>(a); fill_qpel_row<3>(a);
  a->put_hevc_epel_8 = epel8; a->put_hevc_epel_h_8 = epel8b; a->put_hevc_epel_v_8 = epel8b; a->put_hevc_epel_hv_8 = epel8b;
  a->put_hevc_epel_16 = epel16; a->put_hevc_epel_h_16 = epel16; a->put_hevc_epel_v_16 = epel16; a->put_hevc_epel_hv_16 = epel16;
  a->put_unweighted_pred_8 = uni8; a->put_unweighted_pred_16 = uni16;
  a->put_weighted_pred_avg_8 = avg8; a->put_weighted_pred_avg_16 = avg16;
  a->put_weighted_pred_8 = wp8; a->put_weighted_pred_16 = wp16;
  a->put_weighted_bipred_8 = bi8; a->put_weighted_bipred_16 = bi16;
  a->transform_add_8[0] = tr8<2>; a->transform_add_8[1] = tr8<3>; a->transform_add_8[2] = tr8<4>; a->transform_add_8[3] = tr8<5>;
  a->transform_add_16[0] = tr16<2>; a->transform_add_16[1] = tr16<3>; a->transform_add_16[2] = tr16<4>; a->transform_add_16[3] = tr16<5>;
  a->transform_4x4_dst_add_8 = dst8; a->transform_4x4_dst_add_16 = dst16;
  a->intra_pred_dc_8 = dc8; a->intra_pred_planar_8 = planar8; a->intra_pred_angular_8 = ang8;
  a->intra_pred_dc_16 = dc16; a->intra_pred_planar_16 = planar16; a->intra_pred_angular_16 = ang16;
  a->deblock_luma_8 = dbl8; a->deblock_chroma_8 = dbc8;
}

// Explicit selection for applications / tests: what a new `de265_acceleration` level (de265.h:416-427) set through
// de265_set_parameter_int(ctx, DE265_DECODER_PARAM_ACCELERATION_CODE, ...) would do inside set_acceleration_functions.
extern "C" LIBDE265_API void de265_b200_use_dsp_table(de265_decoder_context* de265ctx)
{
  decoder_context* ctx = (decoder_context*)de265ctx;
  init_acceleration_functions_fallback(&ctx->acceleration);
  init_acceleration_functions_b200(&ctx->acceleration);
}
