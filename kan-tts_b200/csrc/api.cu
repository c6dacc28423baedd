// extern "C" surface of libkantts_b200.so (see include/kantts_b200.h).
#include "common.cuh"

namespace kt {
const char* last_error();
int validate_conv(const KtConv1dDesc* d);
int conv1d_fwd_ffma(const KtConv1dDesc*, const float*, const float*, const float*, const float*, float*, cudaStream_t);
int conv1d_bwd_data_ffma(const KtConv1dDesc*, const float*, const float*, const float*, const float*, float*, cudaStream_t);
int conv1d_bwd_weight_ffma(const KtConv1dDesc*, const float*, const float*, const float*, float*, float*, cudaStream_t);
int weight_prepare(const float*, const float*, const float*, int, int, int, int, int, int, float*, float*, float*, float*, cudaStream_t);
int weight_grad(const float*, const float*, const float*, const float*, const float*, int, int, int, int, int, int, float*, float*, int,
                const float*, float*, int, cudaStream_t);
int sinadd_fwd(const float*, float*, long long, cudaStream_t);
int sinadd_bwd(const float*, const float*, float*, long long, cudaStream_t);
int add3_scale(const float*, const float*, const float*, float, float*, long long, cudaStream_t);
int upsample_grad_reduce(const float*, const float*, int, float, float*, long long, int, int, cudaStream_t);
int dwt_fwd(const float*, float*, int, int, cudaStream_t);
int dwt_bwd(const float*, float*, int, int, cudaStream_t);
int l1_sum(const float*, const float*, long long, float, float*, cudaStream_t, bool accumulate = false);
int stft_mel_fwd(const KtMelDesc*, const float*, const float*, const float*, float*, float*, float*, cudaStream_t);
int stft_mel_bwd(const KtMelDesc*, const float*, const float*, const float*, const float*, const float*, float*, cudaStream_t);
long long wgrad_tc_workspace(const KtConv1dDesc*);
int conv1d_bwd_weight_tc(const KtConv1dDesc*, const float*, const float*, const float*, float*, float*, float*, long long, cudaStream_t);
int tc_plan(const KtConv1dDesc*, int);
void debug_wgrad_plan(const KtConv1dDesc*, int*);
long long tc_image_bytes(const KtConv1dDesc*, int);
int tc_pack_layer(const KtConv1dDesc*, int, const float*, void*, cudaStream_t);
long long conv_tc_workspace(const KtConv1dDesc*, int);
void debug_conv_tc_plan(const KtConv1dDesc*, int, long long*);
int conv1d_fwd_tc(const KtConv1dDesc*, const float*, const void*, const float*, const float*, float*, float*, long long, cudaStream_t);
int conv1d_bwd_data_tc(const KtConv1dDesc*, const float*, const float*, const void*, const float*, float*, float*, long long, cudaStream_t,
                       bool allow_tma = true);
int ar_duration_infer(const float*, const float*, const float*, const float*, const float*, const float*, const float*, const float*,
                      const float*, const float*, const float*, float, float*, int, int, int, int, int, cudaStream_t);
int conv1d_fwd_ffma_stream(const KtConv1dDesc*, const KtStreamWin*, const float*, const float*, const float*, const float*, float*,
                           cudaStream_t);
int conv1d_fwd_tc_stream(const KtConv1dDesc*, const KtStreamWin*, const float*, const void*, const float*, const float*, float*,
                         cudaStream_t);
int sinadd_fwd_win(const float*, float*, int, int, int, int, int, int, cudaStream_t);
int add3_scale_win(const float*, const float*, const float*, float, float*, int, int, int, int, int, int, cudaStream_t);
int stream_advance(const KtWindow*, int, int, int, int, cudaStream_t);
int stream_reset(const KtWindow*, int, int, const uint8_t*, int, cudaStream_t);
int resblock_plan(const KtResblockDesc*);
long long resblock_image_bytes(const KtResblockDesc*);
int resblock_pack(const KtResblockDesc*, const float*, void*, cudaStream_t);
int resblock_fwd(const KtResblockDesc*, const float*, const void*, const float*, const void*, const float*, float*, float*, cudaStream_t);
int layernorm_fwd(const float*, const float*, const float*, float*, float*, float*, int, int, float, cudaStream_t);
long long layernorm_bwd_workspace(int, int);
int layernorm_bwd(const float*, const float*, const float*, const float*, const float*, float*, float*, float*, float*,
                  long long, int, int, cudaStream_t);
int attention_fwd(const KtAttnDesc*, const float*, const float*, const float*, const unsigned char*, const unsigned char*,
                  float*, float*, float*, cudaStream_t);
int attention_bwd(const KtAttnDesc*, const float*, const float*, const float*, const float*, const unsigned char*,
                  const float*, float*, float*, float*, float*, int, cudaStream_t);
int fsmn_fwd(const float*, const float*, const unsigned char*, float*, int, int, int, int, int, cudaStream_t);
long long fsmn_bwd_workspace(int, int, int, int);
int fsmn_bwd(const float*, const float*, const float*, const unsigned char*, float*, float*, float*, long long, int, int,
             int, int, int, cudaStream_t);
int rows_gather_fwd(const float*, const int*, float*, int, int, int, int, cudaStream_t);
int rows_gather_bwd(const float*, const int*, const int*, const int*, float*, int, int, int, int, cudaStream_t);
int fp_insert_plan(const void*, int, const float*, const int*, int, int, int, int*, int*, int*, cudaStream_t);
int fp_insert_fwd(const float*, const float*, const int*, float*, int, int, int, int, int, cudaStream_t);
int fp_insert_bwd(const float*, const int*, const int*, float*, float*, float*, long long, int, int, int, int, int,
                  cudaStream_t);
int fsmn_fwd_stream(const KtStreamWin*, const float*, const float*, const int*, const float*, float*, int, int, int, int, int, int,
                    cudaStream_t);
int lstm_stream(const float*, const float*, float*, float*, int, int, int, int, int, cudaStream_t);
}  // namespace kt

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int kt_weight_prepare(const float* v, const float* g, const float* inv_sigma, int32_t mode, int32_t d0, int32_t d1,
                      int32_t k, int32_t transposed, int32_t groups, float* w_fwd, float* w_bwd, float* norm_out,
                      float* w_ref, void* stream) {
  return kt::weight_prepare(v, g, inv_sigma, mode, d0, d1, k, transposed, groups, w_fwd, w_bwd, norm_out, w_ref, ST(stream));
}

int kt_weight_grad(const float* dw_fwd, const float* v, const float* g, const float* norm, const float* inv_sigma,
                   int32_t mode, int32_t d0, int32_t d1, int32_t k, int32_t transposed, int32_t groups, float* dv,
                   float* dg, void* stream) {
  return kt::weight_grad(dw_fwd, v, g, norm, inv_sigma, mode, d0, d1, k, transposed, groups, dv, dg, 0, nullptr, nullptr, 0, ST(stream));
}

int kt_weight_grad_accum(const float* dw_fwd, const float* v, const float* g, const float* norm, const float* inv_sigma,
                         int32_t mode, int32_t d0, int32_t d1, int32_t k, int32_t transposed, int32_t groups, float* dv,
                         float* dg, const float* dbias_src, float* dbias_dst, int32_t nbias, void* stream) {
  return kt::weight_grad(dw_fwd, v, g, norm, inv_sigma, mode, d0, d1, k, transposed, groups, dv, dg, 1, dbias_src, dbias_dst, nbias,
                         ST(stream));
}

int kt_conv1d_fwd(const KtConv1dDesc* d, const float* x, const float* w_fwd, const float* bias, const float* resid,
                  float* y, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && w_fwd && y, "kt_conv1d_fwd: null pointer");
  KT_REQUIRE(d->path != KT_PATH_TC, "kt_conv1d_fwd: tensor-core path not available for this shape");
  return kt::conv1d_fwd_ffma(d, x, w_fwd, bias, resid, y, ST(stream));
}

int kt_conv1d_bwd_data(const KtConv1dDesc* d, const float* dy, const float* y, const float* w_bwd, const float* x,
                       float* dx, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(dy && w_bwd && dx, "kt_conv1d_bwd_data: null pointer");
  KT_REQUIRE(d->path != KT_PATH_TC, "kt_conv1d_bwd_data: tensor-core path not available for this shape");
  return kt::conv1d_bwd_data_ffma(d, dy, y, w_bwd, x, dx, ST(stream));
}

int kt_conv1d_bwd_weight(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw,
                         float* dbias, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && dy && dw, "kt_conv1d_bwd_weight: null pointer");
  KT_REQUIRE(d->path != KT_PATH_TC, "kt_conv1d_bwd_weight: tensor-core path not available for this shape");
  return kt::conv1d_bwd_weight_ffma(d, x, dy, y, dw, dbias, ST(stream));
}

int kt_sinadd_fwd(const float* x, float* y, int64_t n, void* stream) { return kt::sinadd_fwd(x, y, n, ST(stream)); }
int kt_sinadd_bwd(const float* x, const float* dy, float* dx, int64_t n, void* stream) { return kt::sinadd_bwd(x, dy, dx, n, ST(stream)); }
int kt_add3_scale(const float* a, const float* b, const float* c, float scale, float* y, int64_t n, void* stream) {
  return kt::add3_scale(a, b, c, scale, y, n, ST(stream));
}
int kt_debug_wgrad_plan(const KtConv1dDesc* d, int32_t* out12) {
  KT_REQUIRE(d && out12, "kt_debug_wgrad_plan: null pointer");
  kt::debug_wgrad_plan(d, out12);
  return KT_OK;
}
int kt_debug_conv_tc_plan(const KtConv1dDesc* d, int32_t dir, int64_t* out9) {
  KT_REQUIRE(d && out9, "kt_debug_conv_tc_plan: null pointer");
  long long v[9];
  kt::debug_conv_tc_plan(d, dir, v);
  for (int i = 0; i < 9; ++i) out9[i] = v[i];
  return KT_OK;
}
int kt_upsample_grad_reduce(const float* dxu, const float* x, int32_t act_in, float act_in_slope, float* dx, int64_t rows,
                            int32_t up, int32_t c, void* stream) {
  return kt::upsample_grad_reduce(dxu, x, act_in, act_in_slope, dx, rows, up, c, ST(stream));
}
int kt_dwt_db3_fwd(const float* x, float* y, int32_t batch, int32_t t, void* stream) { return kt::dwt_fwd(x, y, batch, t, ST(stream)); }
int kt_dwt_db3_bwd(const float* dy, float* dx, int32_t batch, int32_t t, void* stream) { return kt::dwt_bwd(dy, dx, batch, t, ST(stream)); }
int kt_stft_mel_fwd(const KtMelDesc* d, const float* wav, const float* window, const float* melmat, float* mel,
                    float* amp, float* spec, void* stream) {
  return kt::stft_mel_fwd(d, wav, window, melmat, mel, amp, spec, ST(stream));
}
int kt_stft_mel_bwd(const KtMelDesc* d, const float* dmel, const float* damp, const float* spec, const float* window,
                    const float* melmat, float* dwav, void* stream) {
  return kt::stft_mel_bwd(d, dmel, damp, spec, window, melmat, dwav, ST(stream));
}
int kt_l1_sum(const float* a, const float* b, int64_t n, float scale, float* out, void* stream) {
  return kt::l1_sum(a, b, n, scale, out, ST(stream));
}
int kt_l1_sum_acc(const float* a, const float* b, int64_t n, float scale, float* out, void* stream) {
  return kt::l1_sum(a, b, n, scale, out, ST(stream), true);
}

const char* kt_last_error(void) { return kt::last_error(); }
int kt_version(void) { return 4; }
int kt_has_tc(void) { return 1; }

int kt_conv1d_tc_plan(const KtConv1dDesc* d, int32_t dir) {
  if (kt::validate_conv(d)) return 0;
  return kt::tc_plan(d, dir);
}
int64_t kt_conv1d_tc_image_bytes(const KtConv1dDesc* d, int32_t dir) {
  if (kt::validate_conv(d)) return 0;
  return kt::tc_image_bytes(d, dir);
}
int kt_weight_pack_tc(const KtConv1dDesc* d, int32_t dir, const float* w, void* out, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  return kt::tc_pack_layer(d, dir, w, out, ST(stream));
}
int64_t kt_conv1d_tc_workspace(const KtConv1dDesc* d, int32_t dir) {
  if (kt::validate_conv(d)) return 0;
  return kt::conv_tc_workspace(d, dir);
}
int kt_conv1d_fwd_tc(const KtConv1dDesc* d, const float* x, const void* wimg, const float* bias, const float* resid,
                     float* y, float* workspace, int64_t workspace_floats, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && wimg && y, "kt_conv1d_fwd_tc: null pointer");
  return kt::conv1d_fwd_tc(d, x, wimg, bias, resid, y, workspace, workspace_floats, ST(stream));
}
int64_t kt_conv1d_bwd_weight_tc_workspace(const KtConv1dDesc* d) {
  if (kt::validate_conv(d)) return 0;
  return kt::wgrad_tc_workspace(d);
}
int kt_conv1d_bwd_weight_tc(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw,
                            float* dbias, float* workspace, int64_t workspace_floats, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(x && dy && dw, "kt_conv1d_bwd_weight_tc: null pointer");
  return kt::conv1d_bwd_weight_tc(d, x, dy, y, dw, dbias, workspace, workspace_floats, ST(stream));
}
int kt_conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                          float* dx, float* workspace, int64_t workspace_floats, void* stream) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(dy && wimg && dx, "kt_conv1d_bwd_data_tc: null pointer");
  return kt::conv1d_bwd_data_tc(d, dy, y, wimg, x, dx, workspace, workspace_floats, ST(stream));
}

static int validate_stream(const KtConv1dDesc* d, const KtStreamWin* w, const float* resid, const char* what) {
  int rc = kt::validate_conv(d);
  if (rc) return rc;
  KT_REQUIRE(w != nullptr, "%s: null window descriptor", what);
  KT_REQUIRE(d->nsub == 1, "%s: streams need nsub == 1", what);
  KT_REQUIRE(w->in_first >= 0 && w->in_first + d->t_in <= w->in_pitch, "%s: the chunk does not fit its input window", what);
  KT_REQUIRE(w->out_first >= 0 && w->out_first + d->t_out <= w->out_pitch, "%s: the chunk does not fit its output window", what);
  KT_REQUIRE(!resid || (w->res_first >= 0 && w->res_first + d->t_out <= w->res_pitch),
             "%s: the chunk does not fit its residual window", what);
  return KT_OK;
}
int kt_conv1d_fwd_stream(const KtConv1dDesc* d, const KtStreamWin* w, const float* x, const float* w_fwd, const float* bias,
                         const float* resid, float* y, void* stream) {
  int rc = validate_stream(d, w, resid, "kt_conv1d_fwd_stream");
  if (rc) return rc;
  KT_REQUIRE(x && w_fwd && y, "kt_conv1d_fwd_stream: null pointer");
  return kt::conv1d_fwd_ffma_stream(d, w, x, w_fwd, bias, resid, y, ST(stream));
}
int kt_conv1d_fwd_tc_stream(const KtConv1dDesc* d, const KtStreamWin* w, const float* x, const void* wimg, const float* bias,
                            const float* resid, float* y, void* stream) {
  int rc = validate_stream(d, w, resid, "kt_conv1d_fwd_tc_stream");
  if (rc) return rc;
  KT_REQUIRE(x && wimg && y, "kt_conv1d_fwd_tc_stream: null pointer");
  return kt::conv1d_fwd_tc_stream(d, w, x, wimg, bias, resid, y, ST(stream));
}
int kt_sinadd_fwd_win(const float* x, float* y, int32_t batch, int32_t rows, int32_t ch, int32_t x_pitch, int32_t y_pitch,
                      int32_t y_first, void* stream) {
  return kt::sinadd_fwd_win(x, y, batch, rows, ch, x_pitch, y_pitch, y_first, ST(stream));
}
int kt_add3_scale_win(const float* a, const float* b, const float* c, float scale, float* y, int32_t batch, int32_t rows,
                      int32_t ch, int32_t x_pitch, int32_t y_pitch, int32_t y_first, void* stream) {
  return kt::add3_scale_win(a, b, c, scale, y, batch, rows, ch, x_pitch, y_pitch, y_first, ST(stream));
}
int kt_stream_advance(const KtWindow* windows, int32_t n, int32_t batch, int32_t frames, int32_t max_channels, void* stream) {
  return kt::stream_advance(windows, n, batch, frames, max_channels, ST(stream));
}
int kt_stream_reset(const KtWindow* windows, int32_t n, int32_t batch, const uint8_t* slots, int32_t max_channels, void* stream) {
  return kt::stream_reset(windows, n, batch, slots, max_channels, ST(stream));
}

int kt_ar_duration_infer(const float* g0c, const float* w1, const float* b1, const float* w2t, const float* b2, const float* wih0t,
                         const float* whh0t, const float* wih1t, const float* whh1t, const float* bias1, const float* fcw, float fcb,
                         float* out, int32_t batch, int32_t length, int32_t hidden, int32_t p1, int32_t p2, void* stream) {
  return kt::ar_duration_infer(g0c, w1, b1, w2t, b2, wih0t, whh0t, wih1t, whh1t, bias1, fcw, fcb, out, batch, length, hidden, p1, p2,
                               ST(stream));
}
int kt_resblock_plan(const KtResblockDesc* d) { return d ? kt::resblock_plan(d) : 0; }
int64_t kt_resblock_image_bytes(const KtResblockDesc* d) { return d ? kt::resblock_image_bytes(d) : 0; }
int kt_resblock_pack(const KtResblockDesc* d, const float* w_fwd, void* img, void* stream) {
  KT_REQUIRE(d, "kt_resblock_pack: null descriptor");
  return kt::resblock_pack(d, w_fwd, img, ST(stream));
}
int kt_resblock_fwd(const KtResblockDesc* d, const float* x, const void* img1, const float* b1, const void* img2,
                    const float* b2, float* h, float* y, void* stream) {
  KT_REQUIRE(d, "kt_resblock_fwd: null descriptor");
  return kt::resblock_fwd(d, x, img1, b1, img2, b2, h, y, ST(stream));
}
int kt_resblock_bwd(const KtConv1dDesc* d1, const KtConv1dDesc* d2, const float* x, const float* h, const float* dy,
                    const void* wimg1_bwd, const void* wimg2_bwd, float* dh, float* dx, void* stream) {
  KT_REQUIRE(d1 && d2 && x && h && dy && wimg1_bwd && wimg2_bwd && dh && dx, "kt_resblock_bwd: null pointer");
  KT_REQUIRE(d1->act_in == KT_ACT_LRELU && d2->act_in == KT_ACT_LRELU && d1->act_out == KT_ACT_NONE && d2->act_out == KT_ACT_NONE &&
                 d1->c_in == d1->c_out && d2->c_in == d2->c_out && d1->c_in == d2->c_in && d1->t_in == d2->t_in && d1->t_out == d1->t_in &&
                 d2->t_out == d2->t_in && d1->batch == d2->batch && d1->nsub == 1 && d2->nsub == 1,
             "kt_resblock_bwd: descriptors are not a (convs1[i], convs2[i]) pair of a ResidualBlock");
  // dh = c2^T(dy) * lrelu'(h);  dx = c1^T(dh) * lrelu'(x) + dy   (the residual path, layers.py:219)
  // (register-staged route: this entry point takes no workspace)
  int rc = kt::conv1d_bwd_data_tc(d2, dy, nullptr, wimg2_bwd, h, dh, nullptr, 0, ST(stream), false);
  if (rc) return rc;
  rc = kt::conv1d_bwd_data_tc(d1, dh, nullptr, wimg1_bwd, x, dx, nullptr, 0, ST(stream), false);
  if (rc) return rc;
  const long long n = (long long)d1->batch * d1->t_in * d1->c_in;
  return kt::add3_scale(dx, dy, nullptr, 1.f, dx, n, ST(stream));
}

int kt_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                     int32_t rows, int32_t c, float eps, void* stream) {
  return kt::layernorm_fwd(x, gamma, beta, y, mean, rstd, rows, c, eps, ST(stream));
}
int64_t kt_layernorm_bwd_workspace(int32_t rows, int32_t c) { return kt::layernorm_bwd_workspace(rows, c); }
int kt_layernorm_bwd(const float* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                     float* dx, float* dgamma, float* dbeta, float* workspace, int64_t workspace_floats,
                     int32_t rows, int32_t c, void* stream) {
  return kt::layernorm_bwd(dy, x, gamma, mean, rstd, dx, dgamma, dbeta, workspace, workspace_floats, rows, c, ST(stream));
}
int kt_attention_fwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const uint8_t* mask,
                     const uint8_t* keep, float* out, float* probs, float* probs_dropped, void* stream) {
  return kt::attention_fwd(d, q, k, v, mask, keep, out, probs, probs_dropped, ST(stream));
}
int kt_attention_bwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const float* probs,
                     const uint8_t* keep, const float* dout, float* dq, float* dk, float* dv, float* delta,
                     int32_t accum_dq, void* stream) {
  return kt::attention_bwd(d, q, k, v, probs, keep, dout, dq, dk, dv, delta, accum_dq, ST(stream));
}
int kt_fsmn_fwd(const float* x, const float* w, const uint8_t* mask, float* y, int32_t batch, int32_t t, int32_t c,
                int32_t k, int32_t pad_left, void* stream) {
  return kt::fsmn_fwd(x, w, mask, y, batch, t, c, k, pad_left, ST(stream));
}
int64_t kt_fsmn_bwd_workspace(int32_t batch, int32_t t, int32_t c, int32_t k) {
  return kt::fsmn_bwd_workspace(batch, t, c, k);
}
int kt_fsmn_bwd(const float* x, const float* dy, const float* w, const uint8_t* mask, float* dx, float* dw,
                float* workspace, int64_t workspace_floats, int32_t batch, int32_t t, int32_t c, int32_t k,
                int32_t pad_left, void* stream) {
  return kt::fsmn_bwd(x, dy, w, mask, dx, dw, workspace, workspace_floats, batch, t, c, k, pad_left, ST(stream));
}
int kt_rows_gather_fwd(const float* in, const int32_t* idx, float* out, int32_t batch, int32_t t_out, int32_t t_in,
                       int32_t c, void* stream) {
  return kt::rows_gather_fwd(in, idx, out, batch, t_out, t_in, c, ST(stream));
}
int kt_rows_gather_bwd(const float* dout, const int32_t* idx, const int32_t* start, const int32_t* count, float* din,
                       int32_t batch, int32_t t_out, int32_t t_in, int32_t c, void* stream) {
  return kt::rows_gather_bwd(dout, idx, start, count, din, batch, t_out, t_in, c, ST(stream));
}
int kt_fp_insert_plan(const void* fp_label, int32_t label_bytes, const float* fp_p, const int32_t* input_lengths,
                      int32_t batch, int32_t length, int32_t t_cap, int32_t* codes, int32_t* rows, int32_t* inter_lengths,
                      void* stream) {
  return kt::fp_insert_plan(fp_label, label_bytes, fp_p, input_lengths, batch, length, t_cap, codes, rows, inter_lengths,
                            ST(stream));
}
int kt_fp_insert_fwd(const float* text_hid, const float* fp_enc, const int32_t* codes, float* out, int32_t batch,
                     int32_t length, int32_t t_cap, int32_t t_ins, int32_t c, void* stream) {
  return kt::fp_insert_fwd(text_hid, fp_enc, codes, out, batch, length, t_cap, t_ins, c, ST(stream));
}
int kt_fp_insert_bwd(const float* dout, const int32_t* codes, const int32_t* rows, float* d_text_hid, float* d_fp_enc,
                     float* partials, int64_t partial_floats, int32_t batch, int32_t length, int32_t t_cap, int32_t t_ins,
                     int32_t c, void* stream) {
  return kt::fp_insert_bwd(dout, codes, rows, d_text_hid, d_fp_enc, partials, partial_floats, batch, length, t_cap, t_ins, c,
                           ST(stream));
}
int kt_fsmn_fwd_stream(const KtStreamWin* w, const float* x, const float* weight, const int32_t* lengths, const float* resid, float* y,
                       int32_t batch, int32_t rows, int32_t c, int32_t k, int32_t pad_left, int32_t row0, void* stream) {
  return kt::fsmn_fwd_stream(w, x, weight, lengths, resid, y, batch, rows, c, k, pad_left, row0, ST(stream));
}
int kt_lstm_stream(const float* gx, const float* whh_t, float* state, float* h, int32_t batch, int32_t rows, int32_t hidden,
                   int32_t gx_pitch, int32_t h_pitch, void* stream) {
  return kt::lstm_stream(gx, whh_t, state, h, batch, rows, hidden, gx_pitch, h_pitch, ST(stream));
}

}  // extern "C"
