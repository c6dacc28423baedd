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
/* opt-in single-pass bf16: each operand rounded once to bf16 (round to nearest), ONE wgmma per K = 16 slice, fp32
 * accumulation; a shape without a tensor-core route runs the FFMA kernels, as KT_PATH_AUTO.  Every tensor-core query and
 * entry point (plans, workspaces, image sizes and packing, forward, data / weight gradient, stream, fused resblock) answers
 * for, and runs, the precision of the descriptor it is given: an image packed for one precision is not valid for the other. */
#define KT_PATH_BF16 3

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
/* Workspace: channel counts % 8 == 0 without nearest-upsampling may take the TMA-fed route, which first writes the
 * gathered operand (forward: act_in(x); data gradient: dy * act_out'(y)) into `workspace` as hi / lo bf16 planes
 * ([plane][B][T][nsub][C], 16-byte aligned).  kt_conv1d_tc_workspace: floats of workspace direction `dir` needs, 0 for
 * the register-staged route (then workspace may be NULL); a smaller workspace returns KT_ERR_WORKSPACE. */
int64_t kt_conv1d_tc_workspace(const KtConv1dDesc* d, int32_t dir);
int kt_conv1d_fwd_tc(const KtConv1dDesc* d, const float* x, const void* wimg, const float* bias, const float* resid,
                     float* y, float* workspace, int64_t workspace_floats, void* stream);
int kt_conv1d_bwd_data_tc(const KtConv1dDesc* d, const float* dy, const float* y, const void* wimg, const float* x,
                          float* dx, float* workspace, int64_t workspace_floats, void* stream);

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

/* accumulate == 0: out[0] = scale * sum |a - b|  (F.l1_loss numerator; loss.py:249,309); out[0] is overwritten.
 * accumulate != 0: out[0] += scale * sum |a - b|: one accumulator for a whole feature pyramid (FeatureMatchLoss,
 * loss.py:217-256); the caller zeroes out[0] once. */
int kt_l1_sum(const float* a, const float* b, int64_t n, float scale, float* out, int32_t accumulate, void* stream);

/* Feature-map columns of the multi-resolution spectrogram discriminator (SpecDiscriminator, hifigan.py:481-582).  Its
 * (k, 1) convs also pad the width-1 frequency axis by p_l per side, so after layer l the map is
 * [class_l x p_l | previous columns | class_l x p_l] around the centre (signal) column, and all columns of one class are
 * the same sequence for every item.  rows [batch + classes][t][c]: the signal rows of the items, then one row block per
 * class in birth order.  reach[k]: how far class k extends from the centre (the sum of the paddings up to its birth layer,
 * strictly increasing from 1); width = 2 * reach[classes - 1] + 1 (1 without classes). */
#define KT_SPEC_MAX_CLASSES 8
typedef struct KtSpecColumnsDesc {
  int32_t batch, t, c, classes;
  int32_t reach[KT_SPEC_MAX_CLASSES];
} KtSpecColumnsDesc;
/* out [batch][t][width][c] (channels-last; the module returns its (batch, c, t, width) view) from rows. */
int kt_spec_columns_fwd(const KtSpecColumnsDesc* d, const float* rows, float* out, void* stream);
/* drows [batch + classes][t][c] (overwritten) = the gradient of rows: each item's centre column, and each class summed over
 * its columns and the items in a fixed order (no atomics: reproducible bits). */
int kt_spec_columns_bwd(const KtSpecColumnsDesc* d, const float* dout, float* drows, void* stream);

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

/* Filled-pause insertion (KanTtsSAMBERT.insert_fp, kantts_sambert.py:766-860).  Row t of utterance b of the output is
 * row t of the stream: for j = 0 .. length-1, the 3 rows of filled pause k_j (when k_j > 0) then text_hid[b][j]; after
 * that text_hid[b][q % length] for q = 0, 1, ...
 * kt_fp_insert_plan: one CTA per utterance.  Either fp_label [batch][length] (label_bytes 4 = int32, 8 = int64;
 * k_j = label when it is 1..3, n_b counts every label > 0 over all positions) or, with label_bytes 0, the softmax output
 * fp_p [batch][length][4] (16-byte aligned): on positions j < input_lengths[b] the flags are (p == max over the 4
 * classes) for classes 1..3, k_j is the first set flag and n_b counts every set flag.  Writes
 *   codes [batch][t_cap]: >= 0 a text_hid row; -(1 + 3 (k-1) + m) row m of filled pause k (rows past t_cap are dropped),
 *   rows [batch][length]: the stream row of text_hid[b][j],
 *   inter_lengths [batch] = input_lengths[b] + 3 n_b.
 * t_ins = length + max(inter_lengths) - max(input_lengths) rows are valid; t_cap >= t_ins is the caller's bound
 * (4 * length for labels, 10 * length for predictions).
 * kt_fp_insert_fwd: out [batch][t_ins][c] from text_hid [batch][length][c] and fp_enc [3][3][c].
 * kt_fp_insert_bwd: d_text_hid [batch][length][c] and / or d_fp_enc [3][3][c] (either may be NULL), each a fixed-order
 * sum (d_fp_enc: per-utterance sums into `partials`, at least 9 * batch * c floats, then a sum over b in order). */
int kt_fp_insert_plan(const void* fp_label, int32_t label_bytes, const float* fp_p, const int32_t* input_lengths,
                      int32_t batch, int32_t length, int32_t t_cap, int32_t* codes, int32_t* rows, int32_t* inter_lengths,
                      void* stream);
int kt_fp_insert_fwd(const float* text_hid, const float* fp_enc, const int32_t* codes, float* out, int32_t batch,
                     int32_t length, int32_t t_cap, int32_t t_ins, int32_t c, void* stream);
int kt_fp_insert_bwd(const float* dout, const int32_t* codes, const int32_t* rows, float* d_text_hid, float* d_fp_enc,
                     float* partials, int64_t partial_floats, int32_t batch, int32_t length, int32_t t_cap, int32_t t_ins,
                     int32_t c, void* stream);

/* Alignment learning (MAS: True, sambert_16k_MAS*.yaml).  Every reduction runs in a fixed order; no float atomics.
 * kt_align_attn_fwd: the distance attention of ConvAttention (kantts/models/sambert/attention.py:85-125) on the (B, L, C)
 * rows the convs produce: q [batch][t_q][c], k [batch][t_k][c], c <= 128,
 *   z[b][i][j] = -0.0005 sum_c (q[b][i][c] - k[b][j][c])^2            (the squares summed directly, exact fp32)
 *   logprob = prior ? z - logsumexp_j(z) + log(prior + 1e-8) : z      (the log_softmax over ALL t_k keys; prior
 *                                                                      [batch][t_q][t_k] or NULL)
 *   soft = softmax over the keys j < key_lengths[b] of logprob, 0 on the other keys.
 * row_lse [batch][t_q] receives logsumexp_j(z) when a prior is given (kept for the backward).
 * kt_align_attn_bwd: dq [batch][t_q][c] and dk [batch][t_k][c] from d_soft and / or d_logprob (either may be NULL), with
 * the softmax backward through soft and, with a prior, the log_softmax backward over all keys; dz [batch][t_q][t_k] is
 * scratch (the gradient of z).  Two launches: per query row, then per key.
 *
 * kt_mas: mas_width1 (kantts/models/sambert/alignment.py:32-71) of every soft[b, :out_lengths[b], :in_lengths[b]], one CTA
 * per utterance: log_p over the rows with log(soft), row 0 restricted to key 0, the step from key j - 1 taken when its log_p
 * is >= (ties and -inf included); the backtrack from (T - 1, N - 1) and the reference's final write hard[b][0][0] = 1.
 * Writes all of hard [batch][t_q][t_k] (0 / 1) and durations [batch][t_k] = sum over the rows of hard.  One decision bit per
 * cell: in shared memory when they fit, else in `workspace` (kt_mas_workspace_bytes, 0 when they fit).
 *
 * kt_attn_ctc_fwd / _bwd: AttentionCTCLoss (kantts/train/loss.py:481-508), one CTA per utterance.  Frame t < T of
 * utterance b is log_softmax([blank_logprob, logprob[b][t][:N]]), N = in_lengths[b], T = out_lengths[b]; the CTC loss of
 * the targets 1..N over those frames, divided by N, 0 when infinite (zero_infinity); loss [1] = their mean over the batch.
 * The backward writes all of d_logprob [batch][t_q][t_k] = d_loss[0] * the gradient of loss.  The alpha / beta recursions
 * run in float64 (their values reach thousands at training lengths and the posteriors cancel them); the frame normalisers,
 * loss and gradient are fp32.  The two float64 state rows live in shared memory: t_k <= 3071.  `workspace` holds the
 * float64 alpha recursion and per-utterance -log p, then the fp32 per-frame normalisers, between the two calls:
 * kt_attn_ctc_workspace_bytes.
 *
 * kt_attn_prior: the alignment prior of a collate batch, beta_binomial_prior_distribution (kantts/datasets/dataset.py:20-31)
 * per utterance as AM_Dataset.collate_fn pads it (dataset.py:816-827).  valid_input_lengths / valid_output_lengths
 * [batch] are the collate's int64 device tensors.  With P = valid_input_lengths[b] + 1 (the symbols with the trailing eos),
 * M = valid_output_lengths[b], n = P, alpha = t + 1, beta = M - t:
 *   prior[b][t][k] = exp(lnC(n, k) + lnB(k + alpha, n - k + beta) - lnB(alpha, beta))   for t < M, k < P
 *                  = 0                                                                  elsewhere
 * with lnB(x, y) = lgamma(x) + lgamma(y) - lgamma(x + y), lnC the log binomial coefficient: the beta-binomial pmf of k
 * (support 0..n; k = P is left out, as in the reference).  The exponent is summed in float64 with the device lgamma, every
 * term that depends on t only, on k only or on t + k only computed once per CTA, and rounded to float32 by
 * __double2float_rn (subnormals kept).  Writes all of prior [batch][t_mel][t_text]; when M > t_mel or P > t_text only the
 * elements inside the pad are written, with the values of the true P and M.  One launch, no host read. */
int kt_attn_prior(const int64_t* valid_input_lengths, const int64_t* valid_output_lengths, float* prior, int32_t batch,
                  int32_t t_mel, int32_t t_text, void* stream);
int kt_align_attn_fwd(const float* q, const float* k, const float* prior, const int32_t* key_lengths, float* logprob,
                      float* soft, float* row_lse, int32_t batch, int32_t t_q, int32_t t_k, int32_t c, void* stream);
int kt_align_attn_bwd(const float* q, const float* k, const float* prior, const float* soft, const float* row_lse,
                      const float* d_soft, const float* d_logprob, float* dz, float* dq, float* dk, int32_t batch,
                      int32_t t_q, int32_t t_k, int32_t c, void* stream);
int64_t kt_mas_workspace_bytes(int32_t batch, int32_t t_q, int32_t t_k);
int kt_mas(const float* soft, const int32_t* in_lengths, const int32_t* out_lengths, float* hard, float* durations,
           uint32_t* workspace, int64_t workspace_bytes, int32_t batch, int32_t t_q, int32_t t_k, void* stream);
int64_t kt_attn_ctc_workspace_bytes(int32_t batch, int32_t t_q, int32_t t_k);
int kt_attn_ctc_fwd(const float* logprob, const int32_t* in_lengths, const int32_t* out_lengths, float* loss,
                    void* workspace, int64_t workspace_bytes, int32_t batch, int32_t t_q, int32_t t_k, float blank_logprob,
                    void* stream);
int kt_attn_ctc_bwd(const float* logprob, const int32_t* in_lengths, const int32_t* out_lengths, const float* d_loss,
                    const void* workspace, int64_t workspace_bytes, float* d_logprob, int32_t batch, int32_t t_q,
                    int32_t t_k, float blank_logprob, void* stream);

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
/* kt_blstm_ragged: inference of a 1-layer bidirectional nn.LSTM (hidden <= 256) over a padded batch of ragged sequences,
 * both directions in ONE launch (one CTA per (item, direction), one thread per gate): pack_padded_sequence -> nn.LSTM
 * (bidirectional=True) -> pad_packed_sequence(total_length = length).  lengths: device int32 [batch], never read on the host.
 *   gx     [batch][length][8 * hidden]: x . [weight_ih_l0; weight_ih_l0_reverse]^T + the two directions' bias_ih + bias_hh
 *          (one k = 1 conv over the concatenated weights)
 *   whh_t  [2][hidden][4 * hidden]: weight_hh_l0^T, weight_hh_l0_reverse^T
 *   h      [batch][length][2 * hidden]: forward | backward outputs.  The forward direction runs rows [0, len_b), the
 *          backward one starts from zeros at row len_b - 1 and runs down to row 0; rows >= len_b are zero.
 * An item's rows depend on its own gx rows, its length and the weights only (the same sums in the same order for any batch
 * or length).  PyTorch gate order (i, f, g, o); exact fp32. */
int kt_blstm_ragged(const float* gx, const float* whh_t, const int32_t* lengths, float* h, int32_t batch, int32_t length,
                    int32_t hidden, void* stream);
/* kt_lstm_train_fwd / kt_lstm_train_bwd: one layer of a uni- (dirs = 1) or bidirectional (dirs = 2) nn.LSTM (hidden <= 256)
 * in training, one CTA per (item, direction).  lengths: device int32 [batch] or NULL.  With lengths, the packed semantics
 * of pack_padded_sequence: the forward direction runs rows [0, len_b), the backward one from row len_b - 1 down to row 0,
 * both from zeros, and rows >= len_b of h are zero.  Without, every row runs (nn.LSTM over the padded rows).
 *   gx      [batch][length][dirs * 4 * hidden]: x . weight_ih^T + bias_ih + bias_hh of each direction (one k = 1 conv)
 *   whh_t   [dirs][hidden][4 * hidden]: weight_hh^T of each direction (forward)
 *   whh     [dirs][4 * hidden][hidden]: weight_hh of each direction (backward)
 *   init    [batch][dirs][2][hidden] or NULL: the initial h then c of each (item, direction), zeros when NULL
 *   h       [batch][length][dirs * hidden]: the output;  c [batch][length][dirs * hidden]: the cell states, zero on rows >=
 *           len_b (optional in the forward);  acts [batch][length][dirs * 4 * hidden]: the gate activations sigmoid(i), sigmoid(f), tanh(g),
 *           sigmoid(o) (optional in the forward).  The backward reads the h, c and acts of a forward with the same lengths.
 *   dh, dc  [batch][length][dirs * hidden]: the gradients of h and c (dc may be NULL: zero)
 *   dgates  [batch][length][dirs * 4 * hidden]: the gradient of gx (zero on rows >= len_b)
 *   h_prev  [batch][length][dirs * hidden]: each row's recurrent input (h of the row before it in its direction's order, zero
 *           at the direction's first row (init's h when given) and on rows >= len_b): dW_hh = sum over rows of
 *           dgates^T h_prev, per direction.
 *   dstate  init's layout or NULL: the gradient of the initial (h, c).
 * Both recurrences are exact fp32 with a fixed summation order: an item's rows depend on its own rows, its length and the
 * weights only.  PyTorch gate order (i, f, g, o). */
int kt_lstm_train_fwd(const float* gx, const float* whh_t, const int32_t* lengths, const float* init, float* h, float* c,
                      float* acts, int32_t batch, int32_t length, int32_t dirs, int32_t hidden, void* stream);
int kt_lstm_train_bwd(const float* dh, const float* dc, const float* whh, const int32_t* lengths, const float* init,
                      const float* h, const float* c, const float* acts, float* dgates, float* h_prev, float* dstate,
                      int32_t batch, int32_t length, int32_t dirs, int32_t hidden, void* stream);

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
/* 1: the fused kernel supports this shape (no GPU needed).  The x tile arrives as one TMA box of
 * ceil8(128 + (k-1)*dilation) rows (+ dilation when C = 32), at most 256: e.g. C = 32, k = 15, dilation 11 is not fused. */
int kt_resblock_plan(const KtResblockDesc* d);
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

/* ---- streaming inference of causal layers (Generator.streamer: the waveform chunk by chunk) -------------------------
 * A stream keeps each layer input of batch item b in a WINDOW of `pitch` rows x C channels, channels-last:
 *   window row first + t  =  time step t of the current chunk (t >= 0),
 *   rows [0, first)       =  the last `first` time steps of the earlier chunks (zeros at the start of an utterance).
 * KtStreamWin places the three row tensors of one conv call: element (b, t, c) of x is
 * x[((b * in_pitch + in_first + t) * c_in + c], likewise y (out_*) and resid (res_*; ignored when resid is NULL). */
typedef struct KtStreamWin {
  int32_t in_pitch, in_first;
  int32_t out_pitch, out_first;
  int32_t res_pitch, res_first;
} KtStreamWin;
/* Streams of a NON-CAUSAL generator and of the post-net: each window trails the pushed frames by `lag` rows (its chunk row t
 * of item b is utterance row u = frames_done[b] * rows_per_frame - lag + t), and each batch slot holds an utterance of
 * lengths[b] frames.  KtStreamMask describes the input window of one conv call: pass it as `m` to the stream forward, which
 * then reads a tap of item b as zero unless 0 <= u < lengths[b] * rows_per_frame -- the whole-utterance forward's zero
 * padding, applied per slot.  lengths and frames_done are device int32 [batch]; the conv calls only read frames_done. */
typedef struct KtStreamMask {
  const int32_t* lengths;
  int32_t* frames_done;
  int32_t rows_per_frame, lag;
} KtStreamMask;
/* Forward of one chunk.  The descriptor is the layer's with t_in / t_out = the chunk's rows (nsub == 1): a tap before the
 * chunk reads the window's earlier rows, down to -in_first, where the whole-sequence forward reads its zero padding; a
 * nearest-upsampled conv reads input row floor(t / upsample) of the same window.  The output goes to rows
 * out_first + [0, t_out) of each item's output window.  `m`: the input window's utterance bounds (KtStreamMask), or NULL
 * for none.  _tc_stream: the register-staged tensor-core kernel (kt_conv1d_tc_plan(d, KT_PLAN_STREAM) != 0; no
 * workspace), `wimg` = the forward image of that N tile. */
int kt_conv1d_fwd_stream(const KtConv1dDesc* d, const KtStreamWin* w, const KtStreamMask* m, const float* x,
                         const float* w_fwd, const float* bias, const float* resid, float* y, void* stream);
int kt_conv1d_fwd_tc_stream(const KtConv1dDesc* d, const KtStreamWin* w, const KtStreamMask* m, const float* x,
                            const void* wimg, const float* bias, const float* resid, float* y, void* stream);
/* kt_conv1d_tc_plan / kt_conv1d_tc_workspace / kt_debug_conv_tc_plan: direction flag of the stream forward (OR'd into dir 0):
 * the plan of kt_conv1d_fwd_tc_stream, which always takes the register-staged route. */
#define KT_PLAN_STREAM 16
/* Elementwise stages into a window: row t of item b of x, a, b, c at x[((b * x_pitch + t) * ch], of y at
 * y[((b * y_pitch + y_first + t) * ch], t < rows.  y = sin(x) + x;  y = scale * (a + b + c) (b, c optional). */
int kt_sinadd_fwd_win(const float* x, float* y, int32_t batch, int32_t rows, int32_t ch, int32_t x_pitch, int32_t y_pitch,
                      int32_t y_first, void* stream);
int kt_add3_scale_win(const float* a, const float* b, const float* c, float scale, float* y, int32_t batch, int32_t rows,
                      int32_t ch, int32_t x_pitch, int32_t y_pitch, int32_t y_first, void* stream);
/* One window of a stream: [batch][pitch][channels] fp32 at `base`, keeping `history` rows between chunks; a chunk of f
 * frames writes f * rows_per_frame rows at row `history`. */
typedef struct KtWindow {
  float* base;
  int32_t pitch, channels, history, rows_per_frame;
} KtWindow;
/* ONE launch over the device table `windows` [n]: after a chunk of `frames` frames, rows [0, history) of every window take
 * the last `history` rows of (history | chunk), i.e. rows [r, r + history) with r = frames * rows_per_frame -- also when
 * r < history and the two ranges overlap.  max_channels >= every window's channels. */
int kt_stream_advance(const KtWindow* windows, int32_t n, int32_t batch, int32_t frames, int32_t max_channels, void* stream);
/* ONE launch: rows [0, history) of every window are zeroed for the batch items b with slots[b] != 0 (device uint8 [batch]). */
int kt_stream_reset(const KtWindow* windows, int32_t n, int32_t batch, const uint8_t* slots, int32_t max_channels, void* stream);
/* ONE launch at the end of a chunk of `frames` frames: rows [first, first + rows) of each item's window y (`ch` channels,
 * `pitch` rows per item), described by m, are zeroed where their utterance row lies outside the utterance; then
 * frames_done[b] += frames for every item. */
int kt_stream_mask_advance(const KtStreamMask* m, float* y, int32_t batch, int32_t rows, int32_t ch, int32_t pitch,
                           int32_t first, int32_t frames, void* stream);

/* ---- ragged batches through the whole-utterance forward (Generator.forward(..., lengths=)) ---------------------------------
 * A whole-utterance mask is a KtStreamMask with frames_done = NULL and lag = 0: item b's rows [0, lengths[b] *
 * rows_per_frame) of the layer's input are data, and the masked forward reads every later row as zero -- the zero padding the
 * item meets run alone.  rows_per_frame counts the input tensor's rows (before a nearest-upsampled conv's up-sampling).
 * kt_conv1d_fwd_masked / kt_conv1d_fwd_tc_masked / kt_resblock_fwd_masked: the forwards above (nsub == 1), same routes, N
 * tiles, images and workspaces, masked; the fused ResBlock masks both its input and its intermediate.
 * kt_rows_mask: rows t >= lengths[b] * rows_per_frame of item b of y [batch][rows][ch] are set to zero. */
int kt_conv1d_fwd_masked(const KtConv1dDesc* d, const KtStreamMask* m, const float* x, const float* w_fwd, const float* bias,
                         const float* resid, float* y, void* stream);
int kt_conv1d_fwd_tc_masked(const KtConv1dDesc* d, const KtStreamMask* m, const float* x, const void* wimg, const float* bias,
                            const float* resid, float* y, float* workspace, int64_t workspace_floats, void* stream);
int kt_resblock_fwd_masked(const KtResblockDesc* d, const KtStreamMask* m, const float* x, const void* img1, const float* b1,
                           const void* img2, const float* b2, float* h, float* y, void* stream);
int kt_rows_mask(const KtStreamMask* m, float* y, int32_t batch, int32_t rows, int32_t ch, void* stream);

/* ---- streaming SAM-BERT post-net (PostNet.streamer: decoder rows in, final post-net rows out, chunk by chunk) ---------------
 * `m` (KtStreamMask, one row per frame) describes a window: chunk row u of item b lies inside its utterance iff lo <= u < hi,
 * lo = lag - frames_done[b] and hi = lo + lengths[b].  So each slot can be anywhere in its own utterance and no chunk reads
 * device data on the host.
 *
 * kt_fsmn_fwd_stream_slots: one chunk of MemoryBlockV2 with FsmnEncoderV2's residual fused, seen as a causal depthwise FIR
 * whose output lags its input by rp = k - 1 - pad_left rows.  x, y and resid are windows placed by `w` (KtStreamWin, c
 * channels): input rows [-(k-1), rows) of the chunk are read (in_first >= k - 1), output rows [0, rows) are written.  `m`
 * describes the input window; output row t is the frame of input row t - rp, and its tap j reads input row t + j - (k-1).
 * With keep(u) = (lo <= u < hi) and xm = keep * x:
 *   y[t] = keep(t - rp) * (xm[t - rp] + sum_j weight[c][j] * xm[t + j - (k-1)]) + resid[t]      (resid optional)
 * xm is a selection, not a product: rows outside the utterance read as zeros whatever the window holds there.
 * The skip term first, then the taps in order, each an fma: kt_fsmn_fwd's sum, so a streamed row equals the whole-sequence
 * row bit for bit.  weight [c][k] as in kt_fsmn_fwd.
 * kt_lstm_stream_slots: `rows` steps of a 1-layer unidirectional nn.LSTM (hidden <= 256), one CTA per batch item.  `m`
 * describes gx: row t of item b is frame t - lo.
 *   gx     row t of item b at gx[(b * gx_pitch + t) * 4 * hidden]: x . weight_ih^T + bias_ih + bias_hh (one k = 1 conv)
 *   whh_t  [hidden][4 * hidden] = weight_hh^T
 *   state  [batch][2][hidden]: (h, c) carried from the previous chunk, overwritten with (h, c) after the last row.  A chunk
 *          whose first row is frame 0 or earlier ignores it and starts from (h, c) = 0; a row before frame 0 leaves (h, c)
 *          as they are (zero) and outputs that zero h, so frame 0 starts from (h, c) = 0.
 *   h      row t of item b at h[(b * h_pitch + t) * hidden]: the LSTM output.
 * PyTorch gate order (i, f, g, o); exact fp32. */
int kt_fsmn_fwd_stream_slots(const KtStreamWin* w, const KtStreamMask* m, const float* x, const float* weight,
                             const float* resid, float* y, int32_t batch, int32_t rows, int32_t c, int32_t k, int32_t pad_left,
                             void* stream);
int kt_lstm_stream_slots(const float* gx, const float* whh_t, float* state, float* h, const KtStreamMask* m, int32_t batch,
                         int32_t rows, int32_t hidden, int32_t gx_pitch, int32_t h_pitch, void* stream);
/* kt_pnca_step_slots: one free-running decoder step of a PNCA layer's two attentions for `batch` slots, each at its own
 * step s = step[b] (device int32 [batch], as mem_len, x_bw, h_bw; active: device uint8 [batch]).
 *   q_row  [batch][3 * heads * d_head]: the step's fused Q | K | V projection
 *   x_kv   [batch][max_steps][2 * heads * d_head]: the self K | V cache; the call writes row s from q_row's K | V (key s
 *          of this call's attention is read from q_row, rows < s from the cache)
 *   h_kv   [batch][max_steps][2 * heads * d_head]: the memory K | V rows
 *   out_x  [batch][heads * d_head]: softmax(q k^T / sqrt(d_head)) v over self keys [max(0, s - x_bw[b]), s]
 *   out_h  likewise over memory keys [s, min(s + h_bw[b], mem_len[b] - 1)]
 * Only the band's keys are read; no mask tensor.  A slot with active[b] == 0 (or s outside [0, min(mem_len[b], max_steps)))
 * gets zero outputs and its cache is not written.  d_head 8, 16 or 32; fp32 (exp from expf). */
int kt_pnca_step_slots(const float* q_row, float* x_kv, const float* h_kv, const int32_t* step, const int32_t* mem_len,
                       const int32_t* x_bw, const int32_t* h_bw, const uint8_t* active, float* out_x, float* out_h,
                       int32_t batch, int32_t heads, int32_t d_head, int32_t max_steps, void* stream);

/* ---- seeded NSF excitation (SourceModule, kantts/models/hifigan/layers.py:229-290) ---------------------------------------
 * kt_nsf_excitation: the sine-plus-noise excitation of `frames` frames of `batch` slots as a deterministic function of each
 * slot's seed, its f0 / voiced flag and the sample index -- a chunk's rows equal the matching rows of the whole utterance's.
 *   f0uv  row j of item b at f0uv[(b * f0uv_pitch + f0uv_first + j) * 2]: (f0 in Hz, voiced flag)
 *   e     row r of item b at e[(b * e_pitch + e_first + r) * (H + 1)], r = j * hop + i, 0 <= i < hop: the H + 1 harmonics
 *   state seeds [batch] (device int64), phase [batch][H + 1] (device float64), samples_done [batch] (device int64);
 *         phase and samples_done are advanced by the call (zeros start an utterance), seeds are only read.
 * With h = 0..H the harmonic, n = samples_done[b] + r the sample index since the slot's reset, seed = (k0 low word, k1 high):
 *   c_{h,j} = f0_j * (h + 1) / sr                       float64
 *   P_{h,j+1} = frac(P_{h,j} + hop * c_{h,j})           float64, P_{h,0} = phase[b][h] (the only order-dependent sum)
 *   theta = (float) 2 pi frac(P_{h,j} + (i + 1) c_{h,j})   (the reference's inclusive cumsum)
 *   phi_h = (float)(-pi + 2 pi w0 2^-32), (w0..w3) = Philox4x32-10(counter (0, 0, h, 1), key (k0, k1));  phi_0 = 0
 *   z = (float)(sqrt(-2 log u1) cos(2 pi u2)), u_k = (w_{k-1} + 0.5) 2^-32 in float64, (w0..w3) = Philox4x32-10((n low,
 *       n high, h, 0), (k0, k1))
 *   e = (alpha sin(theta + phi) + sigma z) uv + (k (sigma z)) (1 - uv),  k = (float)((double)alpha / 3 / (double)sigma)
 * in float32, every operation rounded as written (no contraction, no fast-math); sr = sampling_rate.  The reference uses
 * alpha 0.1, sigma 0.003.  nb_harmonics H < 32.  Two launches (the rows, then the state). */
typedef struct KtNsfState {
  const int64_t* seeds;
  double* phase;
  int64_t* samples_done;
} KtNsfState;
int kt_nsf_excitation(const float* f0uv, int32_t f0uv_pitch, int32_t f0uv_first, const KtNsfState* s, float* e,
                      int32_t e_pitch, int32_t e_first, int32_t batch, int32_t frames, int32_t hop, int32_t nb_harmonics,
                      int32_t sampling_rate, float alpha, float sigma, void* stream);

/* Speaker-embedding extractor (kantts/preprocess/se_processor, csrc/speaker.cu): inference only, exact fp32, fixed-order
 * reductions.  Item b of a batch owns rows [0, lengths[b]) of its tensors; every kernel writes the rows at or past that as
 * zeros and reduces over the valid rows only, so an item's results do not depend on the rest of its batch.
 *
 * kt_kaldi_fbank: torchaudio.compliance.kaldi.fbank(wav[b, :lengths[b]], num_mel_bins=n_mels) at its other defaults
 * (400-sample frames every 160 samples, snip_edges, no dither, DC removal, pre-emphasis 0.97, povey window, 512-point power
 * spectrum, Kaldi mel triangles from low_hz to Nyquist, log(max(e, FLT_EPSILON))), minus each channel's mean over the
 * utterance's frames.  out [batch][frames][n_mels], frames = 1 + (n_samples - 400) / 160; item b has
 * 1 + (lengths[b] - 400) / 160 frames (lengths[b] in [400, n_samples]).  Two launches.
 * kt_se_tap_gather: y[b][fo][t][k][c] (rows of y_pitch floats) = x[b * sb + fi * sf + t * st + c] with
 * fi = stride * fo + k - pad (zero outside [0, f_in)): the frequency taps of a 2-D conv as the channels of a 1-D one.
 * kt_se_affine_rows: y[b][r][c] (row pitch y_pitch) = act(scale[c] * x[b][r][c] + shift[c]) (row pitch x_pitch); scale and
 * shift both NULL for a copy; act = ReLU when relu != 0.
 * kt_se_gate_stats: per item and `seg`-row segment (the last one partial), the sum and the max of each channel of h
 * [batch][t][c] over the segment's valid rows into stats [batch][ceil(t / seg)][2][c]; zeroes h's rows past each item.
 * kt_se_gate_apply: per segment, s = sigmoid(w2 relu(w1 (mean(h) + segmax(h)) + b1) + b2) from those stats (w1 [c_mid][c],
 * w2 [c_out][c_mid]), then out[b][r][o] (row pitch out_pitch) = y[b][r][o] * s[o], y [batch][t][c_out].
 * kt_se_stats_pool: out [batch][2c] = the mean and the unbiased std of each channel of x [batch][t][c] over the valid rows. */
int kt_kaldi_fbank(const float* wav, const int32_t* lengths, float* out, int32_t batch, int32_t n_samples, int32_t frames,
                   int32_t n_mels, float sample_rate, float low_hz, void* stream);
int kt_se_tap_gather(const float* x, int64_t sb, int64_t sf, int64_t st, const int32_t* lengths, float* y, int32_t y_pitch,
                     int32_t batch, int32_t f_in, int32_t t, int32_t c, int32_t f_out, int32_t taps, int32_t stride,
                     int32_t pad, void* stream);
int kt_se_affine_rows(const float* x, int32_t x_pitch, const float* scale, const float* shift, int32_t relu,
                      const int32_t* lengths, float* y, int32_t y_pitch, int32_t batch, int32_t t, int32_t c, void* stream);
int kt_se_gate_stats(float* h, const int32_t* lengths, float* stats, int32_t batch, int32_t t, int32_t c, int32_t seg,
                     void* stream);
int kt_se_gate_apply(const float* y, const float* stats, const float* w1, const float* b1, const float* w2, const float* b2,
                     const int32_t* lengths, float* out, int32_t out_pitch, int32_t batch, int32_t t, int32_t c,
                     int32_t c_mid, int32_t c_out, int32_t seg, void* stream);
int kt_se_stats_pool(const float* x, const int32_t* lengths, float* out, int32_t batch, int32_t t, int32_t c, void* stream);

/* Masked-symbol pretraining of the text encoder (KanTtsTextsyBERT, sybert.yaml; csrc/bert.cu).
 * kt_seq_ce_fwd: SeqCELoss (kantts/train/loss.py:444-460) of logits [rows][v] (any v >= 1), int64 targets [rows] and float
 * masks [rows], one warp per row:
 *   lse[r]  = log sum_j exp(logits[r][j])                       (online max / sum in fp32, written for the backward)
 *   arg[r]  = the first j with the row's largest logit          (torch.argmax's rule on ties)
 *   loss[0] = sum_r (lse[r] - logits[r][t_r]) m_r / M,  err[0] = sum_r [arg[r] != t_r] m_r / M,  mask_sum[0] = M = sum_r m_r
 *                                                               (float32; device scalars)
 * The sums run in float64: per-CTA partials in `workspace` (kt_seq_ce_workspace_bytes(rows)), then one reducing warp; the
 * grid depends on `rows` only, so two calls give bit-identical scalars.  M == 0 gives NaN loss and error, as the reference
 * does; a target outside [0, v) gives a NaN loss.  Two launches, no host read.
 * kt_seq_ce_bwd: dlogits[r][j] = (d_loss[0] / M) m_r (exp(logits[r][j] - lse[r]) - [j == t_r]), with d_loss (device [1])
 * and M = mask_sum[0] read on the device.
 *
 * kt_bert_mask: BERT_Text_Dataset.bert_masking (kantts/datasets/dataset.py:873-920, 1022-1040) of a batch, one CTA per
 * utterance.  lings [batch][length][n_feat] int64 with the symbol id in feature 0; valid_lengths [batch] int32 (the
 * collate's valid_input_lengths: positions from valid_lengths[b] on, the trailing eos and the padding, are never selected).
 * With key (k0, k1) = (seed low word, seed high word), (c2, c3) = (call low word, call high word) and
 * (w0..w3) = Philox4x32-10(counter (i, b, c2, c3), key) for position i of utterance b:
 *   selected    i < valid_lengths[b] and w0 < threshold;  threshold = ceil(mask_ratio 2^32) makes this w0 2^-32 < mask_ratio
 *               exactly, the float64 compare of the reference's uniform draw
 *   rank        the position of (w1 2^32 + w2, i) in ascending order among the n selected positions of the utterance
 *   n_mask = floor(n * 0.8), n_rand = floor(n * 0.1)                     (float64, as math.floor in Python)
 *   out symbol  mask_id when rank < n_mask; the utterance's replacement id when n_mask <= rank < n_mask + n_rand;
 *               otherwise the symbol itself
 *   replacement (w0' n_sy) >> 32 (an id in [0, n_sy - 1]), (w0'..w3') = Philox4x32-10(counter (0xFFFFFFFF, b, c2, c3), key)
 * Writes out_lings (lings with feature 0 masked), targets [batch][length] (feature 0 unmasked) and bert_masks
 * [batch][length] (1.0 at the selected positions, else 0.0).  length * 9 bytes of shared memory (length <= 22755).  One
 * launch. */
int64_t kt_seq_ce_workspace_bytes(int32_t rows);
int kt_seq_ce_fwd(const float* logits, const int64_t* targets, const float* masks, float* lse, float* loss, float* err,
                  float* mask_sum, void* workspace, int64_t workspace_bytes, int32_t rows, int32_t v, void* stream);
int kt_seq_ce_bwd(const float* logits, const int64_t* targets, const float* masks, const float* lse, const float* mask_sum,
                  const float* d_loss, float* dlogits, int32_t rows, int32_t v, void* stream);
int kt_bert_mask(const int64_t* lings, const int32_t* valid_lengths, int64_t* out_lings, int64_t* targets, float* bert_masks,
                 int32_t batch, int32_t length, int32_t n_feat, int64_t seed, int64_t call, int64_t threshold, int32_t n_sy,
                 int32_t mask_id, void* stream);

/* Test aid (no GPU needed): the plan kt_conv1d_bwd_weight_tc would make for this layer on a GPU box.
 * out12 = {supported, TMA variant, time steps per chunk, rows per chunk, padded rows, ring stages, shared-memory bytes,
 * split-K factor, N tile, unit groups, time steps per A box, rows of one A image}. */
int kt_debug_wgrad_plan(const KtConv1dDesc* d, int32_t* out12);
/* Test aid (no GPU needed): the plan kt_conv1d_{fwd,bwd_data}_tc would make for direction `dir` on a GPU box.
 * out9 = {N tile (0: not on the tensor cores), TMA route, time steps per M tile, rows per M tile, time steps per image box,
 * image stages, weight stages, shared-memory bytes, workspace floats}; tile and stage entries describe the first launch. */
int kt_debug_conv_tc_plan(const KtConv1dDesc* d, int32_t dir, int64_t* out9);
/* Test aid (no GPU needed): 1 when those launches take the shared-memory staged epilogue (given 16-byte aligned operands),
 * 0 for the register epilogue (stream chunks, produced channels or channels per N tile % 4 != 0) or a layer off the
 * tensor cores. */
int kt_debug_conv_tc_epilogue(const KtConv1dDesc* d, int32_t dir);
/* Test aid (no GPU needed): how those launches pack the items of a batch into M tiles when an item has few output rows.
 * out5 = {items per M tile (1: not packed), image rows of one item's block, MMA rows issued per N tile over all launches,
 * the same with one item per tile, output rows produced per N tile}. */
int kt_debug_conv_tc_pack(const KtConv1dDesc* d, int32_t dir, int64_t* out5);

/* library info */
const char* kt_last_error(void);
int kt_version(void);
/* 1 when the library was built with the tensor-core (sm_90a) conv path */
int kt_has_tc(void);

#ifdef __cplusplus
}
#endif
#endif /* KANTTS_B200_H_ */
