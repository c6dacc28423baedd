/*
 * kantts_b200.h -- C ABI of libkantts_b200.so, the sm_90a implementation of the
 * KAN-TTS HiFi-GAN hot path (generator / discriminator convolutions, DWT pooling,
 * mel-spectrogram loss).
 *
 * The reference (modelscope/KAN-TTS) has no FFI layer: the path sits behind Python
 * nn.Modules that dispatch to ATen/cuDNN/cuFFT.  Each entry point below replaces the
 * library dispatch of one reference call site (cited per function, paths relative to
 * the KAN-TTS checkout).  Conventions (SURVEY.md section 8b):
 *   - plain pointers and sizes only, all buffers caller-allocated DEVICE memory,
 *     fp32 unless stated; no hidden allocation, no global mutable state, re-entrant
 *     across the forward and autograd threads;
 *   - every call takes the CUDA stream to launch on (a cudaStream_t passed as void*)
 *     and never synchronises the host;
 *   - return 0 on success, a negative KT_ERR_* code otherwise (the Python wrapper
 *     raises RuntimeError with kt_last_error()).
 *
 * ACTIVATION LAYOUT: channels-last rows.  A logical (B, C, T) tensor of the reference
 * is stored as [B][T][nsub][C] with C contiguous ("row" = one time step of one
 * sub-sequence).  nsub = 1 everywhere except the period discriminator, where the
 * reference's (B, C, T/p, p) view (hifigan.py:258) is stored as [B][T/p][p][C] and the
 * (k,1) Conv2d becomes a Conv1d over the p interleaved sub-sequences.
 */
#ifndef KANTTS_B200_H_
#define KANTTS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KT_OK 0
#define KT_ERR_INVALID -1   /* bad descriptor / unsupported combination */
#define KT_ERR_CUDA -2      /* a CUDA runtime call or launch failed */
#define KT_ERR_WORKSPACE -3 /* workspace too small */

/* activation codes */
#define KT_ACT_NONE 0
#define KT_ACT_LRELU 1 /* leaky relu, slope in the descriptor */
#define KT_ACT_TANH 2  /* output side only */

/* compute paths */
#define KT_PATH_AUTO 0  /* tensor-core where the shape qualifies, FFMA otherwise */
#define KT_PATH_FFMA 1  /* exact-fp32 CUDA-core kernels */
#define KT_PATH_TC 2    /* tensor-core split-bf16 (bf16x3) tensor-core kernels; error if unsupported */

/* One 1-D convolution layer (forward semantics; the backward entry points take the
 * SAME descriptor).  Replaces F.conv1d / F.conv_transpose1d / F.conv2d((k,1)) as
 * dispatched from kantts/models/hifigan/layers.py:44-46,82-88,123,161 and
 * hifigan.py:219-247,328-396 (cuDNN fwd / dgrad / wgrad).
 *
 *   conv       : y[b,to,co] = act_out( bias[co] + sum_{j,ci} w[co,ci,j] * act_in(xu[b, to*stride + j*dilation - pad_left, ci]) ) + resid
 *                xu = x nearest-upsampled by `upsample` (hifigan.py:85: nn.Upsample) ; out-of-range taps read 0
 *   transposed : y[b, ti*stride + j*dilation - pad_left, co] += w[ci,co,j] * act_in(x[b,ti,ci])   (then bias, act_out, resid)
 *   t_out is given explicitly (the causal variants crop: layers.py:87,161).
 */
typedef struct KtConv1dDesc {
  int32_t batch;      /* B */
  int32_t nsub;       /* interleaved sub-sequences per batch item (period p; else 1) */
  int32_t t_in;       /* input time steps per sub-sequence */
  int32_t t_out;      /* output time steps per sub-sequence */
  int32_t c_in;
  int32_t c_out;
  int32_t groups;
  int32_t kernel;
  int32_t stride;
  int32_t dilation;
  int32_t pad_left;
  int32_t transposed; /* 0 conv, 1 ConvTranspose1d */
  int32_t upsample;   /* >=1; nearest-neighbour upsampling of the input (conv only) */
  int32_t act_in;     /* KT_ACT_NONE | KT_ACT_LRELU */
  float act_in_slope;
  int32_t act_out;    /* KT_ACT_NONE | KT_ACT_LRELU | KT_ACT_TANH */
  float act_out_slope;
  int32_t path;       /* KT_PATH_* */
} KtConv1dDesc;

/* Weight layouts consumed by the conv kernels ("kernel layouts"), produced by
 * kt_weight_prepare from the reference parameter layout:
 *   conv       reference (Cout, Cin/g, k):  w_fwd[k][Cin/g][Cout]   w_bwd[k][Cout/g][Cin]
 *   transposed reference (Cin, Cout, k)  :  w_fwd[k][Cin][Cout]     w_bwd[k][Cout][Cin]
 * Both are fp32; kt_weight_pack_tc turns either into the split-bf16 tiles of the tensor-core path. */

/* Weight re-parametrisation + layout (replaces torch._weight_norm at layers.py:29,67,
 * 105,139 and hifigan.py:224,331; plain / spectral-normed weights use mode 0 with an
 * optional device scalar `inv_sigma`).
 *   mode 1 (weight norm, dim 0): w = g[d0] * v / ||v[d0,:,:]||   ; norm_out[d0] = ||v[d0]||
 *   mode 0 (plain)             : w = v * (inv_sigma ? *inv_sigma : 1)
 * v is the reference layout (d0, d1, k); `transposed` says whether d0 is Cin (1) or Cout (0);
 * `groups` as in the conv (d1 = Cin/groups).  w_ref (optional) receives w in reference layout. */
int kt_weight_prepare(const float* v, const float* g, const float* inv_sigma, int32_t mode,
                      int32_t d0, int32_t d1, int32_t k, int32_t transposed, int32_t groups,
                      float* w_fwd, float* w_bwd, float* norm_out, float* w_ref, void* stream);

/* Backward of kt_weight_prepare: dw_fwd is in the layout written by kt_conv1d_bwd_weight
 * (w_fwd layout for a conv, w_bwd layout for a transposed conv).  mode 1: dv, dg (reference layouts);  mode 0: dv = dw * scale. */
int kt_weight_grad(const float* dw_fwd, const float* v, const float* g, const float* norm,
                   const float* inv_sigma, int32_t mode, int32_t d0, int32_t d1, int32_t k,
                   int32_t transposed, int32_t groups, float* dv, float* dg, void* stream);

/* Same, ACCUMULATING into the parameters' gradient buffers: dv += ..., dg += ..., and (optional, both or
 * neither) dbias_dst[0..nbias) += dbias_src.  This is torch's AccumulateGrad (`param.grad += grad`, run once
 * per parameter per backward by the autograd engine under kantts/train/trainer.py:546,580) folded into the
 * kernel that produces the gradient; the caller zeroes the buffers once per backward. */
int kt_weight_grad_accum(const float* dw_fwd, const float* v, const float* g, const float* norm,
                         const float* inv_sigma, int32_t mode, int32_t d0, int32_t d1, int32_t k,
                         int32_t transposed, int32_t groups, float* dv, float* dg, const float* dbias_src,
                         float* dbias_dst, int32_t nbias, void* stream);

/* Forward.  x: [B][t_in][nsub][c_in], y: [B][t_out][nsub][c_out]; bias / resid optional (NULL).
 * resid has y's shape and is added AFTER act_out (layers.py:219 `x = xt + x`; hifigan.py:168). */
int kt_conv1d_fwd(const KtConv1dDesc* d, const float* x, const float* w_fwd, const float* bias,
                  const float* resid, float* y, void* stream);

/* Data gradient.  dy: gradient wrt y; y: the forward output (needed when act_out != NONE,
 * to apply act_out'), x: the forward input (needed when act_in != NONE).  dx is overwritten. */
int kt_conv1d_bwd_data(const KtConv1dDesc* d, const float* dy, const float* y, const float* w_bwd,
                       const float* x, float* dx, void* stream);

/* Weight / bias gradient.  dw (k*Cin/g*Cout floats; w_fwd layout for a conv, w_bwd layout
 * [k][Cout][Cin] for a transposed conv) and dbias (c_out, optional) are overwritten.  */
int kt_conv1d_bwd_weight(const KtConv1dDesc* d, const float* x, const float* dy, const float* y,
                         float* dw, float* dbias, void* stream);

/* ---- tensor-core (wgmma) path: bf16x3 split-precision implicit GEMM, fp32 accumulation in registers ----
 * kt_conv1d_tc_plan: returns the (padded) output-channel tile NT > 0 when direction `dir` (0 forward, 1 data
 * gradient) of the layer can run on the tensor-core kernel, else 0.  Any stride / period / group count /
 * channel count qualifies (channels are zero-padded to 64-wide K chunks and 16-wide N tiles; a grouped
 * conv maps one group to one N tile); only the nearest-upsampled data gradient stays on the FFMA path.
 * kt_conv1d_tc_image_bytes / kt_weight_pack_tc: size of, and packing into, the hi/lo bf16 SWIZZLE_128B
 * weight tiles ([taps][ceil(K/64)][N tiles][hi|lo][NT][64] bf16) from the fp32 kernel-layout weight of
 * that direction (w_fwd for dir 0, w_bwd for dir 1).
 * kt_conv1d_{fwd,bwd_data}_tc: same contract as the fp32 entry points, `wimg` = the packed tiles. */
int kt_conv1d_tc_plan(const KtConv1dDesc* d, int32_t dir);
int64_t kt_conv1d_tc_image_bytes(const KtConv1dDesc* d, int32_t dir);
int kt_weight_pack_tc(const KtConv1dDesc* d, int32_t dir, const float* w, void* out, void* stream);
int kt_conv1d_fwd_tc(const KtConv1dDesc* d, const float* x, const void* wimg, const float* bias, const float* resid,
                     float* y, void* stream);
int kt_conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                          float* dx, void* stream);

/* tensor-core weight gradient (time is the contraction dimension; split-K partial tiles go to `workspace`,
 * a second kernel reduces them -- a single split writes dw / dbias directly).  Plain convs with channel counts % 8 == 0
 * take the TMA-fed variant: `workspace` then also holds the two operands as hi / lo bf16 planes, written by one
 * elementwise pre-pass of the call (the planes are 16-byte aligned inside a 256-byte-aligned workspace).
 * kt_conv1d_bwd_weight_tc_workspace: floats of workspace the layer needs (partials + planes), 0 when the layer is not
 * supported (then use kt_conv1d_bwd_weight).  dw / dbias as above. */
int64_t kt_conv1d_bwd_weight_tc_workspace(const KtConv1dDesc* d);
int kt_conv1d_bwd_weight_tc(const KtConv1dDesc* d, const float* x, const float* dy, const float* y, float* dw,
                            float* dbias, float* workspace, int64_t workspace_floats, void* stream);

/* Elementwise pieces of Generator.forward (hifigan.py:157 `x = sin(x) + x`). */
int kt_sinadd_fwd(const float* x, float* y, int64_t n, void* stream);
int kt_sinadd_bwd(const float* x, const float* dy, float* dx, int64_t n, void* stream);
/* y = scale * (a + b + c)   (hifigan.py:170-176: mean over the resblocks; b, c optional) */
int kt_add3_scale(const float* a, const float* b, const float* c, float scale, float* y, int64_t n, void* stream);

/* Second half of the data gradient of the nearest-upsampled conv (hifigan.py:82-97, `repeat_upsamples`):
 * dx[r][c] = act_in'(x[r][c]) * sum_{u<up} dxu[r*up + u][c], where dxu is the data gradient of the SAME conv
 * taken with upsample = 1 / act_in = NONE over t_in*up input rows (kt_conv1d_bwd_data[_tc]).  rows = B*t_in,
 * c % 4 == 0; x may be NULL when act_in == KT_ACT_NONE. */
int kt_upsample_grad_reduce(const float* dxu, const float* x, int32_t act_in, float act_in_slope, float* dx,
                            int64_t rows, int32_t up, int32_t c, void* stream);

/* db3 single-level analysis DWT, zero padding (pytorch_wavelets.DWT1DForward as used at
 * hifigan.py:445-448,469-471) fused with torch.cat([yl, yh], dim=1): x [B][T] -> y [B][T2][2]
 * with T2 = (T + 5) / 2, channel 0 = low-pass, 1 = high-pass. */
int kt_dwt_db3_fwd(const float* x, float* y, int32_t batch, int32_t t, void* stream);
int kt_dwt_db3_bwd(const float* dy, float* dx, int32_t batch, int32_t t, void* stream);

/* Fused mel-spectrogram (kantts/utils/audio_torch.py:155-186): centre zero-padded framing,
 * periodic-hann window, rFFT, sqrt(clamp(|.|^2, eps)), mel projection, clamp(eps),
 * 20*log10(clamp(.,1e-5)) - 20, clamp(8*(x+100)/100 - 4, -4, 4).
 *   wav  [B][T]            mel [B][n_mels][frames] (reference layout)
 *   melmat [n_bins][n_mels] (n_bins = n_fft/2+1), window [n_fft] (a shorter win_length is centre-padded by the caller).
 * n_fft must be a power of two in [64, 4096] (all shipped configs: 512 / 1024 / 2048). */
typedef struct KtMelDesc {
  int32_t batch, t, n_fft, hop, n_mels, frames; /* frames = t / hop + 1 (center=True) */
  int32_t pad_mode;                              /* 0 zeros (MelSpectrogram), 1 reflect (stft(), librosa.stft) */
  float eps;                                     /* amplitude clamp: 1e-10 (mel) / 1e-7 (stft loss) / 0 (dsp.py) */
  /* dB normalisation: v = clamp(norm_scale * ((20*log10(max(mel, 1e-5)) - ref_db - min_db) / -min_db) - norm_shift,
   * norm_lo, norm_hi).  MelSpectrogram (audio_torch.py:42-63): ref 20, min -100, scale 8, shift 4, [-4, 4];
   * offline dsp.melspectrogram (preprocess/audio_processor/core/dsp.py:66-74,165-201): scale max_norm, shift 0,
   * [0, max_norm]  (symmetric=True: scale 2*max_norm, shift max_norm, [-max_norm, max_norm]). */
  float ref_db, min_db, norm_scale, norm_shift, norm_lo, norm_hi;
} KtMelDesc;
/* Outputs (each optional / NULL): mel [B][n_mels][frames] (needs melmat), amp [B][frames][n_bins]
 * (the clamped magnitude, audio_torch.py:31), spec [B][frames][n_bins][2] (re, im; saved for bwd). */
int kt_stft_mel_fwd(const KtMelDesc* d, const float* wav, const float* window, const float* melmat,
                    float* mel, float* amp, float* spec, void* stream);
/* dwav [B][T] (overwritten) = d/dwav of sum(dmel * mel) + sum(damp * amp); dmel / damp optional. */
int kt_stft_mel_bwd(const KtMelDesc* d, const float* dmel, const float* damp, const float* spec,
                    const float* window, const float* melmat, float* dwav, void* stream);

/* out[0] = scale * sum |a - b|  (F.l1_loss numerator; loss.py:249,309); out[0] is overwritten. */
int kt_l1_sum(const float* a, const float* b, int64_t n, float scale, float* out, void* stream);
/* out[0] += scale * sum |a - b|: one accumulator for a whole feature pyramid (FeatureMatchLoss, loss.py:217-256); the caller
 * zeroes out[0] once. */
int kt_l1_sum_acc(const float* a, const float* b, int64_t n, float scale, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SAM-BERT acoustic model (kantts/models/sambert).  Activations are (B, L, C) rows -- the
 * reference's own layout for this model -- so nn.Linear and the transposed nn.Conv1d pairs
 * (sambert/__init__.py:140-149, fsmn.py:36-43) are kt_conv1d_* calls with nsub = 1 and
 * kernel 1 / 3 / 9; the entry points below cover what is not a convolution.
 * --------------------------------------------------------------------------------------------- */

/* nn.LayerNorm(C, eps) over the last dim (sambert/__init__.py:64,131,197; kantts_sambert.py:58,129).
 * x, y, dx: [rows][C]; mean / rstd: [rows] (saved for backward); 1 <= C <= 1024.
 * Backward needs kt_layernorm_bwd_workspace(rows, C) floats of workspace (partial column sums). */
int kt_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                     int32_t rows, int32_t c, float eps, void* stream);
int64_t kt_layernorm_bwd_workspace(int32_t rows, int32_t c);
int kt_layernorm_bwd(const float* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                     float* dx, float* dgamma, float* dbeta, float* workspace, int64_t workspace_floats,
                     int32_t rows, int32_t c, void* stream);

/* ScaledDotProductAttention over all heads (sambert/__init__.py:17-29 plus the head split / merge of
 * :80-100 and :278-300).  q, k, v and out are row tensors addressed as
 *     q[(b*lq + i)*q_stride + h*d_head + e]      (same for k / v over lk rows, out over lq rows)
 * so the fused QKV projection output is consumed in place (pass base pointers offset to the q / k / v column
 * blocks) and `out` is the merged-heads (B, Lq, H*d_head) tensor.  probs [(h*B + b)][lq][lk] is the
 * reference's returned `attn` (head-major) and is always written (backward reads it).
 * mask: optional uint8, non-zero = masked (-inf before the softmax), element
 *     mask[b*mask_b_stride + i*mask_q_stride + j]   (mask_q_stride 0 = key-padding mask broadcast over queries).
 * d_head in {8, 16, 32, 64}; lk <= 2048. */
typedef struct KtAttnDesc {
  int32_t batch, heads, d_head, lq, lk;
  int32_t q_stride, k_stride, v_stride, o_stride; /* floats between consecutive rows */
  int32_t mask_q_stride;
  int64_t mask_b_stride;
  float scale;                                    /* 1 / temperature = d_head ** -0.5 */
  float keep_scale;                               /* attention dropout: 1 / (1 - p); used only with a keep mask */
} KtAttnDesc;
/* keep: optional attention-dropout keep mask, uint8 [(h*B + b)][lq][lk] (non-zero = kept; nn.Dropout on the
 * probabilities, sambert/__init__.py:26).  `probs` always receives the UNdropped softmax (backward needs it);
 * probs_dropped (optional) receives keep * probs * keep_scale, i.e. the tensor the reference returns as `attn`
 * in training mode. */
int kt_attention_fwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const uint8_t* mask,
                     const uint8_t* keep, float* out, float* probs, float* probs_dropped, void* stream);
/* dq / dk / dv use the strides of q / k / v (so they can be the column blocks of one d(QKV) tensor); dout uses
 * o_stride.  delta: [heads*batch*lq] floats of scratch.  accum_dq != 0: dq += (PNCA: the x- and h-attention
 * share their queries, sambert/__init__.py:283,293). */
int kt_attention_bwd(const KtAttnDesc* d, const float* q, const float* k, const float* v, const float* probs,
                     const uint8_t* keep, const float* dout, float* dq, float* dk, float* dv, float* delta,
                     int32_t accum_dq, void* stream);

/* FSMN MemoryBlockV2 (fsmn.py:46-77): y = keep * (xm + depthwise_conv(pad(xm, lp, K-1-lp))), xm = x * keep,
 * keep = !mask.  x, y [B][T][C]; w [C][K] (the (C,1,K) conv_dw weight); mask optional uint8 [B][T], non-zero = padding.
 * Backward: dx and / or dw (either may be NULL); dw needs kt_fsmn_bwd_workspace floats. */
int kt_fsmn_fwd(const float* x, const float* w, const uint8_t* mask, float* y, int32_t batch, int32_t t, int32_t c,
                int32_t k, int32_t pad_left, void* stream);
int64_t kt_fsmn_bwd_workspace(int32_t batch, int32_t t, int32_t c, int32_t k);
int kt_fsmn_bwd(const float* x, const float* dy, const float* w, const uint8_t* mask, float* dx, float* dw,
                float* workspace, int64_t workspace_floats, int32_t batch, int32_t t, int32_t c, int32_t k,
                int32_t pad_left, void* stream);

/* LengthRegulator (adaptors.py:15-37) as a row gather: out[b][t][:] = idx[b][t] >= 0 ? in[b][idx[b][t]][:] : 0.
 * Backward sums, for every input row (b, i), the output rows of its contiguous span
 * [start[b][i], start[b][i] + count[b][i]) whose idx equals i. */
int kt_rows_gather_fwd(const float* in, const int32_t* idx, float* out, int32_t batch, int32_t t_out, int32_t t_in,
                       int32_t c, void* stream);
int kt_rows_gather_bwd(const float* dout, const int32_t* idx, const int32_t* start, const int32_t* count, float* din,
                       int32_t batch, int32_t t_out, int32_t t_in, int32_t c, void* stream);

/* Autoregressive duration predictor, free-running inference (VarRnnARPredictor.infer, kantts/models/sambert/adaptors.py:67-83):
 * the whole per-symbol recurrence  x -> Prenet(1 -> p1 -> p2, ReLU) -> cat(cond) -> 2-layer LSTM(hidden) -> Linear(hidden, 1) ->
 * ReLU -> next x  in ONE launch (one CTA per batch item) instead of ~10 library launches per symbol from Python.
 *   g0c   [batch][length][4*hidden] = cond . weight_ih_l0[:, p2:]^T + bias_ih_l0 + bias_hh_l0   (precomputed, one GEMM)
 *   w1 [p1] = prenet Linear(1,p1).weight[:,0], b1 [p1]; w2t [p1][p2] = Linear(p1,p2).weight^T, b2 [p2]
 *   wih0t [p2][4h] = weight_ih_l0[:, :p2]^T, whh0t [h][4h] = weight_hh_l0^T; wih1t / whh1t [h][4h]; bias1 [4h] = bias_ih_l1 + bias_hh_l1
 *   fcw [h], fcb: the output Linear; out [batch][length] (before the padding mask). */
int kt_ar_duration_infer(const float* g0c, const float* w1, const float* b1, const float* w2t, const float* b2,
                         const float* wih0t, const float* whh0t, const float* wih1t, const float* whh1t,
                         const float* bias1, const float* fcw, float fcb, float* out, int32_t batch, int32_t length,
                         int32_t hidden, int32_t p1, int32_t p2, void* stream);

/* ---- fused ResidualBlock unit (kantts/models/hifigan/layers.py:213-220, one (convs1[i], convs2[i]) pair) ----------
 *   h = conv(leaky_relu(x); w1, dilation d, pad_left1) + b1
 *   y = conv(leaky_relu(h); w2, dilation 1, pad_left2) + b2 + x
 * x, h, y: [B][T][C] channels-last fp32; C = 32 or 64, odd kernel <= 15; pad_left = (k-1)*dil for the causal variant
 * (layers.py:66), (k-1)*dil/2 otherwise; out-of-range taps read 0.  ONE launch on the tensor-core path (bf16x3): the
 * intermediate stays in shared memory / registers.  kt_resblock_pack turns a conv's fp32 kernel-layout weight
 * ([k][C][C], kt_weight_prepare's w_fwd) into the kernel's weight image (kt_resblock_image_bytes bytes).
 * `h` (optional, may be NULL) receives the first conv's output for the backward pass. */
typedef struct KtResblockDesc {
  int32_t batch, t, channels, kernel, dilation, pad_left1, pad_left2;
  float slope;   /* LeakyReLU negative slope of both pre-activations */
  int32_t path;  /* KT_PATH_* (FFMA: the fused kernel is not available) */
} KtResblockDesc;
int kt_resblock_plan(const KtResblockDesc* d);                 /* 1: the fused kernel supports this shape */
int64_t kt_resblock_image_bytes(const KtResblockDesc* d);      /* per conv; 0 = unsupported */
int kt_resblock_pack(const KtResblockDesc* d, const float* w_fwd, void* img, void* stream);
int kt_resblock_fwd(const KtResblockDesc* d, const float* x, const void* img1, const float* b1, const void* img2,
                    const float* b2, float* h, float* y, void* stream);
/* Backward of the unit from the saved (x, h): the data gradients of both convs (tensor-core kernels, derivative masks and
 * the residual path fused) -- dh = c2^T(dy) * lrelu'(h) is written to `dh` (the weight-gradient kernels of c1 need it),
 * dx = dy + c1^T(dh) * lrelu'(x).  wimg*_bwd: kt_weight_pack_tc(dir = 1) images of the two convs' descriptors d1 / d2
 * (the per-conv descriptors the weight-gradient entry points also take). */
int kt_resblock_bwd(const KtConv1dDesc* d1, const KtConv1dDesc* d2, const float* x, const float* h, const float* dy,
                    const void* wimg1_bwd, const void* wimg2_bwd, float* dh, float* dx, void* stream);

/* Development aid, kept for ABI compatibility: the tensor-core kernels record no per-role timelines; any dev_buf is ignored. */
int kt_debug_set_trace(void* dev_buf);
/* Development aid: ablation switches for timing experiments of the weight-gradient chain: bit 8 no operand split, 9 no MMA
 * kernel, 10 no split-K reduce, 11 no weight-norm backward.  RESULTS ARE WRONG while non-zero. */
int kt_debug_set_flags(int32_t flags);
/* Test aid (no GPU needed): the plan kt_conv1d_bwd_weight_tc would make for this layer on a GPU box.
 * out12 = {supported, TMA variant, time steps per chunk, rows per chunk, padded rows, ring stages, shared-memory bytes,
 * split-K factor, N tile, unit groups, time steps per A box, rows of one A image}. */
int kt_debug_wgrad_plan(const KtConv1dDesc* d, int32_t* out12);

/* library info */
const char* kt_last_error(void);
int kt_version(void);
/* 1 when the library was built with the tensor-core (sm_90a) conv path */
int kt_has_tc(void);

#ifdef __cplusplus
}
#endif
#endif /* KANTTS_B200_H_ */
