/*
 * qdiff_b200 -- C ABI of the H100-native (sm_90a) quantized-diffusion UNet engine (libqdiff_b200.so).
 *
 * The reference (Xiuyu-Li/q-diffusion) has no FFI layer: its boundary is the Python class API of
 * `qdiff` (QuantModel.forward, qdiff/quant_model.py:68-69) and every op underneath is a PyTorch
 * library call.  This header is the boundary a maintainer binds (ctypes stub in INTEGRATION.md):
 * each entry point names the reference code it replaces.  Plain pointers and sizes only; all
 * pointers are DEVICE pointers unless stated; every call is asynchronous on the given stream;
 * every function returns 0 on success or a negative qd_status.  No CPU fallback exists.
 */
#ifndef QDIFF_B200_H
#define QDIFF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* qd_stream_t; /* cudaStream_t */

enum qd_status {
  QD_OK = 0,
  QD_ERR_BAD_ARG = -1,
  QD_ERR_UNSUPPORTED = -2,
  QD_ERR_CUDA = -3,
  QD_ERR_NOT_FINALIZED = -4
};

/* Activation quantizer parameters (UniformAffineQuantizer.forward, qdiff/quant_layer.py:82-88):
 * code = clamp(rne(x / delta) + zero_point, qmin, qmax).  Symmetric 8 bit: [-128,127], zp = 0;
 * asymmetric n bit: [0, 2^n-1].  Codes are stored as raw bytes (s8 if qmin < 0, else u8). */
typedef struct qd_qparams {
  float delta;
  int32_t zero_point;
  int32_t qmin;
  int32_t qmax;
} qd_qparams;

/* ------------------------------------------------------------------------------------------
 * qd_qgemm_i8 -- QuantModule.forward (qdiff/quant_layer.py:248-279) for Conv2d 3x3 (stride 1,
 * pad 1), Conv2d 1x1, Conv1d k=1 and Linear, as INT8 wgmma GEMM with the de-quantisation fused
 * into the epilogue:
 *   y[m,n] = scale[n] * (sum_k a[m,k] * w[n,k] - corr[cls(m)][n]) + bias[n]
 *            (+ rowvec[m / rows_per_batch][n]) (+ residual[m,n])
 * a: activation codes, NHWC / token-major.  taps==1: [M, lda] bytes; taps==9: [B,H,W,C] dense.
 * w: weight codes minus zero point (s8), [n_rows][taps*C], tap-major then channel (OHWI).
 * corr: zx * sum_k w[n,k]; for taps==9 one row per border class (3x3 classes, row-major:
 *       top/mid/bottom x left/mid/right) because the reference zero-pads after de-quantisation.
 * geglu: GEGLU projection fused with its consumer's quantizer: N counts x AND gate columns, interleaved in
 *       groups of 4 (w row 8b+i = x-feature 4b+i, row 8b+4+i = gate-feature 4b+i); out_q is [M, N/2].
 * w_int4_packed: the 4-bit weight codes stay packed in HBM (K3 of the survey): w is [n_rows][taps*C/2] bytes; the 8 codes
 *       8g .. 8g+7 of a row occupy bytes 4g .. 4g+3, byte 4g+j = wq[8g+j] | wq[8g+4+j] << 4 (a masked 32-bit word is four
 *       consecutive codes) with UNSIGNED codes wq in [0,15]; w_zero[n] in [0,15] is the row's zero point.  The
 *       kernel unpacks to wq - w_zero (s8) in shared memory between the TMA load and the MMA; everything else
 *       (scale, corr, epilogue) is unchanged.  Halves the weight bytes in HBM and through L2.
 * Output: fp32 `out` and/or re-quantised codes `out_q` with the consumer's quantizer `oq`
 *       (out_q_transposed: [M/rows_per_batch][N][ldq], ldq >= rows_per_batch, 16-token groups permuted as
 *       qd_qattention expects its V^T operand).
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_gemm_desc {
  const void* a;
  const void* w;
  long long lda;        /* bytes between rows of a (taps==1) */
  int32_t M, N, C, taps;
  int32_t w_rows;       /* rows present in w (>= N; padded rows must be zero) */
  int32_t B, H, W;      /* conv geometry (taps==9): M == B*H*W */
  int32_t a_signed;     /* activation codes are s8 (symmetric) or u8 */
  const float* scale;   /* [N] delta_x * delta_w[n] */
  const float* bias;    /* [N] or NULL */
  const int32_t* corr;  /* [9][N] (taps==9) / [N] (taps==1) or NULL when zx == 0 */
  const float* rowvec;  /* [M/rows_per_batch][ld_rowvec] or NULL (timestep-embedding add) */
  long long ld_rowvec;
  int32_t rows_per_batch;
  int32_t out_q_transposed;
  const float* residual; /* [M, ldr] or NULL; may alias out */
  long long ldr;
  float* out;            /* [M, ldo] or NULL */
  long long ldo;
  void* out_q;           /* codes or NULL */
  long long ldq;
  qd_qparams oq;
  int32_t bn_hint;       /* 0 = auto N-tile; else the N tile: a multiple of 16 up to 128 (geglu: of 32) */
  int32_t out_q_head_dim;   /* > 0: row-major out_q is written per head with padding: column n -> */
  int32_t out_q_head_pitch; /*      (n / head_dim) * head_pitch + n % head_dim   (attention Q / K operands) */
  int32_t geglu;         /* 1: rows of w (and scale/bias/corr) are interleaved [4 x-features, 4 gate-features]...;
                            out_q receives Q(x * gelu_erf(gate)) with N/2 columns (ldm/modules/attention.py:42-44) */
  int32_t w_int4_packed; /* 1: w holds packed unsigned 4-bit codes, see above */
  int32_t k_dup;         /* 0 / 1: plain.  2: the reduction runs TWICE over the activation against two weight segments, w is
                          * [n_rows][2][taps*C]: y = scale * sum_k x_k (wa_k + wb_k).  8-bit weights: wq - zw spans [-255, 255] and
                          * does not fit one s8 operand; wa = floor(ws/2), wb = ws - wa do (unless ws = 255), and ONE launch with
                          * a doubled K replaces two accumulating GEMMs.  corr / scale refer to the sum wa + wb. */
  const int8_t* w_zero;  /* [n_rows] zero points of the packed codes (w_int4_packed only) */
  /* Optional, for requantising GEMMs (out_q set, out NULL, geglu 0): the epilogue constants pre-divided by the consumer's
   * step, scale_q[n] = scale[n] / oq.delta and bias_q[n] = bias[n] / oq.delta + oq.zero_point (computed in double by the
   * caller).  With them the epilogue emits  code = clamp(rne(acc * scale_q + bias_q [+ residual / oq.delta]), qmin, qmax)
   * with ONE fused multiply-add per element (the quotient differs from the two-step y / delta by <= 1 ulp, i.e. a code can
   * differ from quant_layer.py:82-87 applied to the fp32 y only where y / delta sits within an ulp of a rounding
   * boundary - the same class as the fused GroupNorm / SiLU / GELU quantizers).  NULL: the exact two-step form. */
  const float* scale_q;
  const float* bias_q;
  /* Optional (fp32 output only): per-column partial sums for a GroupNorm that consumes `out`.  gn_stats[(m / 32) * ld_stats
   * + n] = (sum, sum of squares) of out[m0 .. m0+31, n] over the 32-row slab of row m (only rows < M), written by the
   * epilogue warp that owns the slab: no atomics, deterministic.  gn_stats points at the column of out's first column;
   * ld_stats is the row pitch in float2 units.  qd_groupnorm_quant turns the slabs into per-(image, group) mean / rstd
   * (stats_in), replacing its own pass over the fp32 tensor (GroupNorm32: ldm util.py:214-216). */
  float* gn_stats;
  long long ld_stats;
  /* Weight-only layers (set_quant_state(True, False): quantised weights, fp32 activations; BASELINE configs[0]):
   * a_bf16 = 1: `a` holds the activation as THREE bfloat16 planes per pixel, [M][3][Cp] (hi, mid, lo with
   * x = hi + mid + lo to 2^-24 relative, written by qd_split_bf16x3), `w` the zero-point-free weight codes as bfloat16
   * [n_rows][taps][3][Cp] (the codes repeated for the three planes: |code| <= 255 is exact in bfloat16), C = BYTES per
   * tap = 6 * Cp, lda in bytes.  The contraction runs on wgmma bf16 x bf16 with fp32 accumulation, so
   * y = scale[n] * sum_k x[m,k] * ws[n,k] + bias (+ rowvec, + residual) carries fp32-level rounding only
   * (qdiff/quant_layer.py:263-279 with use_act_quant False).  No corr, no out_q, no geglu. */
  int32_t a_bf16;
  /* out_q_f16 = 1 (row-major out_q only): out_q receives fp16 values (code - zero_point) instead of 8-bit codes; ldq and
   * out_q_head_pitch then count fp16 elements.  Operand format of qd_attention_desc.qk_f16 (the attention's QK^T
   * on f16 MMAs: the same integers, no zero-point correction pass).  The centred code is an integer of
   * magnitude <= 255, exact in fp16. */
  int32_t out_q_f16;
} qd_gemm_desc;

int qd_qgemm_i8(const qd_gemm_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_quantize -- standalone activation fake-quant input side (qdiff/quant_layer.py:256-264)
 * with the elementwise producer fused: dst = Q(f(src)).
 *   act: 0 none, 1 SiLU (x*sigmoid(x): nonlinearity / nn.SiLU), 2 GEGLU (src has 2*C columns,
 *        value = src[:, c] * gelu_erf(src[:, C + c]); ldm/modules/attention.py:42-44)
 *   split > 0: columns [0,split) use q0, columns [split,C) use q1 (split-shortcut,
 *        qdiff/quant_layer.py:257-261)
 *   upsample2x: src is [B,H,W,C], dst [B,2H,2W,C] nearest (F.interpolate, openaimodel.py:116)
 * Codes: +-inf and values whose quotient x / delta overflows take the rail of their sign; NaN takes qmin.
 * Vector kernel when C, ld_src, ld_dst and split are multiples of 4, src is 16-byte and dst 4-byte aligned; otherwise a
 * scalar kernel with the same results.  upsample2x needs the vector kernel: refused (QD_ERR_UNSUPPORTED) otherwise.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_quantize_desc {
  const float* src;
  long long ld_src;
  void* dst;
  long long ld_dst;
  int32_t M, C;
  int32_t act;
  int32_t split;
  qd_qparams q0, q1;
  int32_t upsample2x, B, H, W;
} qd_quantize_desc;

int qd_quantize(const qd_quantize_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_groupnorm_quant -- GroupNorm32 / Normalize (32 groups; ldm util.py:214-216 eps 1e-5,
 * ddim diffusion.py:32-33 eps 1e-6) [+ scale-shift] [+ SiLU] + up to 3 consumer quantizers.
 * x: fp32 NHWC [B, HW, C] (row pitch ld_x).  ws: 8-byte aligned workspace of at least
 * qd_groupnorm_workspace_floats(B, HW, C, groups) floats (small feature maps take a single-kernel path that
 * does not touch it).  Alignment (else QD_ERR_UNSUPPORTED): the single-kernel path moves channel pairs, so x and out_f
 * need 8-byte alignment and ld_f, ld_q even, out_q / raw_q 2-byte alignment; the other paths move channel quads, so x and
 * out_f need 16-byte alignment, ld_f and ld_q multiples of 4, out_q / raw_q 4-byte alignment.  stats_in: 8-byte aligned.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_groupnorm_desc {
  const float* x;
  long long ld_x;
  int32_t B, HW, C, groups;
  float eps;
  int32_t silu;
  const float* gamma;
  const float* beta;
  const float* ss_scale; /* [B, ld_ss] per-image (1+scale) operand or NULL (use_scale_shift_norm) */
  const float* ss_shift;
  long long ld_ss;
  int32_t n_out;         /* number of quantized outputs (0..3) */
  int32_t reserved;
  void* out_q[3];
  long long ld_q[3];
  qd_qparams q[3];
  float* out_f;          /* optional fp32 output (NULL if unused) */
  long long ld_f;
  float* ws;
  /* optional codes of the UN-normalised input (the block's skip_connection reads the same tensor through its own
   * act quantizer, split in two channel ranges when --split is on: quant_layer.py:253-262).  Channels < raw_split
   * use q_raw[0], the others q_raw[1]; raw_split % 4 == 0. */
  void* raw_q;
  long long ld_raw;
  int32_t raw_split;
  int32_t reserved2;
  qd_qparams q_raw[2];
  /* optional: 32-row slab sums written by the producing GEMM(s) (qd_gemm_desc.gn_stats), float2 [B*HW/32][ld_stats_in],
   * pointing at x's first column; needs HW % 32 == 0.  When set, the statistics pass over x is skipped. */
  const float* stats_in;
  long long ld_stats_in;
} qd_groupnorm_desc;

int qd_groupnorm_quant(const qd_groupnorm_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Weight-only mode (quant_act False): activations stay fp32.
 * qd_split_bf16x3 -- dst[m][p][c] = plane p of f(src[m][c]) as bfloat16 (p = 0 hi, 1 mid, 2 lo), c < C; columns C..Cp-1 of
 *   every plane must be zero (allocate dst zeroed).  f: act 0 none, 1 SiLU; upsample2x as in qd_quantize.  ld_dst = 3*Cp.
 *   Vector kernel when C and ld_src are multiples of 4, src is 16-byte and dst 8-byte aligned; otherwise a scalar kernel
 *   with the same results.  upsample2x needs the vector kernel: refused (QD_ERR_UNSUPPORTED) otherwise.
 *   fp32 attention: d + Tk > 12288 is refused (QD_ERR_UNSUPPORTED) unless the 8-row kernel takes the call (not causal,
 *   Tq >= 256, d, ld_q, ld_k, offsets and head strides multiples of 4, q and k 16-byte aligned).
 * qd_attention_fp32 -- softmax(scale * q k^T) v per (batch, head) in fp32: QuantAttnBlock.forward with use_act_quant
 *   False (qdiff/quant_block.py:360-386) and QKVAttentionLegacy (openaimodel.py:384-406; scale = 1/sqrt(ch) applied to
 *   the product).  q: [B*Tq, ld_q], head h at columns q_off + h*head_stride_q (k, v likewise); out [B*Tq, ld_out].
 *   causal = 1: query row r attends to keys 0..r only (the CLIP text encoder's self-attention, CLIPAttention.forward of
 *   transformers' modeling_clip.py with the causal mask of CLIPTextTransformer: FrozenCLIPEmbedder.forward,
 *   ldm/modules/encoders/modules.py:150-155).  Masked keys take no probability whatever their values.  Needs Tq == Tk;
 *   always runs the one-row-per-block kernel.  0 (what a zero-initialised descriptor holds): every key.
 * ------------------------------------------------------------------------------------------ */
/* qd_split_desc.act: 0 none, 1 SiLU, 2 GEGLU (src has 2*C columns: value = src[:, c] * gelu_erf(src[:, C + c])),
 * 3 quick-GELU x * sigmoid(1.702 x) in fp32 with the accurate exponential (CLIPMLP with hidden_act "quick_gelu", the
 * activation between fc1 and fc2 of the text encoder that FrozenCLIPEmbedder runs, modules.py:150-155) */
typedef struct qd_split_desc {
  const float* src;
  long long ld_src;
  void* dst;             /* bfloat16 */
  long long ld_dst;      /* elements: 3 * Cp */
  int32_t M, C, Cp;
  int32_t act;
  int32_t upsample2x, B, H, W;
} qd_split_desc;

typedef struct qd_attention_fp_desc {
  const float* q;
  const float* k;
  const float* v;
  long long ld_q, ld_k, ld_v;
  int32_t B, heads, d, Tq, Tk;
  int32_t q_off, k_off, v_off;
  int32_t head_stride_q, head_stride_k, head_stride_v;
  float scale;
  float* out;
  long long ld_out;
  int32_t causal;        /* 0: all Tk keys; 1: key j <= query row r only (Tq == Tk) */
} qd_attention_fp_desc;

/* qd_embed_tokens -- the text encoder's input embedding (CLIPTextEmbeddings.forward of transformers' modeling_clip.py,
 *   called by FrozenCLIPEmbedder.forward, ldm/modules/encoders/modules.py:150-155):
 *   out[(b*T + t) * ld_out + c] = tok[ids[b*T + t] * C + c] + pos[t * C + c]   (fp32, one rounding: torch's add)
 *   ids int32 [B*T]; tok [vocab][C], pos [>= T][C] fp32.  An id outside [0, vocab) writes NaN across its row (the host
 *   refuses such ids before they are uploaded). */
typedef struct qd_embed_desc {
  const int32_t* ids;
  const float* tok;
  const float* pos;
  float* out;
  long long ld_out;
  int32_t B, T, C, vocab;
} qd_embed_desc;

int qd_embed_tokens(const qd_embed_desc* d, qd_stream_t stream);

/* out[i] = a*x[i] + b*y[i] + c*z[i] (y / z may be NULL): the DPM-Solver++ multistep update
 * x_t = (sigma_t/sigma_s) x - alpha_t (e^-h - 1) m0 - 0.5 alpha_t (e^-h - 1) D1   (dpm_solver.py:504-527, 755-795). */
int qd_lincomb3(float* out, float a, const float* x, float b, const float* y, float c, const float* z, long long n,
                qd_stream_t stream);
int qd_split_bf16x3(const qd_split_desc* d, qd_stream_t stream);
int qd_attention_fp32(const qd_attention_fp_desc* d, qd_stream_t stream);
long long qd_groupnorm_workspace_floats(int B, int HW, int C, int groups);

/* ------------------------------------------------------------------------------------------
 * qd_layernorm_quant -- nn.LayerNorm(C) (eps 1e-5) followed by the act quantizers of its
 * consumers (to_q/to_k/to_v or ff.net.0.proj; qdiff/quant_block.py:268-270).
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_layernorm_desc {
  const float* x;
  long long ld_x;
  int32_t M, C;
  float eps;
  int32_t n_out;
  const float* gamma;
  const float* beta;
  void* out_q[3];
  long long ld_q[3];
  qd_qparams q[3];
  float* out_f;          /* optional fp32 output (weight-only state: the consumers take fp32); n_out may then be 0 */
  long long ld_f;
} qd_layernorm_desc;
/* Refused (QD_ERR_UNSUPPORTED): C > 2048 or C % 4; x, gamma, beta, out_f not 16-byte aligned; ld_x, ld_f, ld_q not
 * multiples of 4; out_q not 4-byte aligned. */

int qd_layernorm_quant(const qd_layernorm_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_im2col_i8 -- explicit patch gather for the convs the implicit-GEMM path does not take
 * (stride-2 downsample convs: openaimodel.py:134-160 pad 1, ddim diffusion.py:55-74 pad (0,1,0,1);
 * conv_in with C_in 3/4).  src: codes NHWC [B,H,W,C]; dst: [B*Ho*Wo, ld_dst], k = (ky*3+kx)*C + c,
 * out-of-image taps = pad_code (the activation zero point == real 0), columns >= 9C zero.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_im2col_desc {
  const void* src;
  void* dst;
  long long ld_dst;
  int32_t B, H, W, C;
  int32_t Ho, Wo, stride, pad_top, pad_left;
  int32_t pad_code;
} qd_im2col_desc;

int qd_im2col_i8(const qd_im2col_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_qattention -- quantised attention core:
 *   CIFAR  QuantAttnBlock.forward            qdiff/quant_block.py:354-386
 *   LDM    QuantQKMatMul/QuantSMVMatMul      qdiff/quant_block.py:123-157 (+ openaimodel.py:384-406)
 *   SD     cross_attn_forward                qdiff/quant_block.py:190-221
 * q,k: codes [B, Tq|Tk, *] with head h at columns q_off + h*head_stride (d codes each);
 * vt: V codes TRANSPOSED [B, n_rows_v, Tk_pad] with head h at rows v_off + h*head_stride; inside every
 *     group of 16 keys, key 8a+2b+c is stored at byte 4b+2a+c (what qd_qgemm_i8 out_q_transposed writes).
 * ws: int32 workspace, B*heads*roundup(Tk,128) entries (zero-point row sums of K; unused when zq == 0).
 * S = sum_d (q-zq)(k-zk) * sim_scale (sim_scale = dq*dk*softmax scale), P = softmax_j(S) in fp32,
 * Pq = clamp(rne(P/dw)+zw, 0.., 2^sm_bits-1) (sm_bits 8 or 16), out = dw*dv * sum_j (Pq-zw)(v-zv).
 * out: fp32 [B, Tq, ld_out] at columns h*d, and/or out_q: the same values re-quantised with `oq`.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_attention_desc {
  const void* q;
  const void* k;
  const void* vt;
  long long ld_q, ld_k;      /* bytes per token row */
  long long ld_vt;           /* bytes per V^T row (>= Tk, multiple of 16) */
  long long v_batch_stride;  /* bytes between batches of V^T */
  int32_t B, heads, d, Tq, Tk;
  int32_t q_off, k_off, v_off, head_stride_q, head_stride_k, head_stride_v;
  int32_t q_signed, k_signed, v_signed, p_signed;
  int32_t zq, zk, zv, zw;
  int32_t p_qmin, p_qmax, sm_bits;
  float sim_scale;
  float delta_w;             /* softmax quantizer step */
  float out_scale;           /* delta_w * delta_v */
  float* out;            /* fp32 output or NULL */
  long long ld_out;
  void* ws;
  void* out_q;           /* optional: codes of the consumer's activation quantizer `oq` (to_out / proj_out input) */
  long long ld_out_q;
  qd_qparams oq;
  /* qk_f16 = 1: q and k hold fp16 values (code - zero_point) in the per-head padded layout (head_stride_q, head_stride_k
   * >= 2 d BYTES, d <= 64; ld_q / ld_k / offsets in bytes as always); zq / zk / q_signed / k_signed / ws are ignored.
   * Same result as the code path (exact integer arithmetic in fp32); d in {16, 24, 32, 40, 48, 64}. */
  int32_t qk_f16;
  int32_t reserved5;
} qd_attention_desc;

int qd_qattention(const qd_attention_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Small fp32 helpers on the path.
 *  qd_timestep_embedding: out[b] = trig(t[b] * freqs[k]); freqs[dim/2] is the host-computed frequency
 *      table (same fp32 expression as the reference, so the angles are bit-identical).
 *      mode 0 = ldm timestep_embedding order [cos,sin] (ldm/modules/diffusionmodules/util.py:151-171);
 *      mode 1 = ddim get_timestep_embedding order [sin,cos] (ddim/models/diffusion.py:6-24).
 *  qd_copy2d: strided fp32 copy (torch.cat along channels, openaimodel.py:776).
 *  qd_nchw_to_nhwc / qd_nhwc_to_nchw: UNet boundary layout change (latents are NCHW fp32).
 *  qd_avgpool2x / qd_upsample2x_f32: Downsample(use_conv=False) / Upsample for resblock_updown.
 *  copy2d, avgpool and upsample move float4: C (and ld) multiples of 4 and 16-byte aligned src / dst, else
 *  QD_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------ */
int qd_timestep_embedding(const float* t, const float* freqs, int32_t B, int32_t dim, int32_t mode, float* out,
                          qd_stream_t s);
int qd_copy2d(const float* src, long long ld_src, float* dst, long long ld_dst, int32_t M, int32_t C, qd_stream_t s);
int qd_nchw_to_nhwc(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, qd_stream_t s);
int qd_nhwc_to_nchw(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, qd_stream_t s);
int qd_avgpool2x(const float* src, float* dst, int32_t B, int32_t H, int32_t W, int32_t C, qd_stream_t s);
int qd_upsample2x_f32(const float* src, float* dst, int32_t B, int32_t H, int32_t W, int32_t C, qd_stream_t s);
/* qd_vq_lookup: the codebook step of VQModelInterface.decode (ldm/models/autoencoder.py:274-283 -> taming's
 *      VectorQuantizer2.forward): for each of `rows` latent pixels z[r, 0..C) (NHWC fp32, row pitch ld_z) the nearest of
 *      the n_e codebook rows by d = sum(z^2) + sum(e^2) - 2 z.e (fp32, lowest index on ties); out = z + (e - z).  C <= 16.
 *      torch.argmin's order: a NaN distance wins (the first one), so a NaN latent row comes out NaN in its NaN channels;
 *      a row whose distances are all +inf takes entry 0. */
/* qd_softmax_rows: in-place softmax over each row of an fp32 [rows, cols] matrix with row pitch ld (the softmax of the
 *      first-stage AttnBlock, model.py:190-192, between its two tensor-core products). */
int qd_softmax_rows(float* x, long long ld, int32_t rows, int32_t cols, qd_stream_t s);
int qd_vq_lookup(const float* z, long long ld_z, const float* codebook, float* out, long long ld_out, int32_t rows, int32_t C,
                 int32_t n_e, qd_stream_t s);

/* ------------------------------------------------------------------------------------------
 * qd_sampler_step -- closed-form latent update of the denoising loop, fused with the
 * classifier-free-guidance combine (e_t = e_uc + s (e_c - e_uc), plms.py:185-190):
 *   DDIM / generalized_steps (ddim/functions/denoising.py:23-29, ldm ddim.py:205-219) and the PLMS
 *   Adams-Bashforth combine (plms.py:203-238).  All tensors fp32 NCHW, n = elements per tensor.
 *   e_t' = c_e0*e + c_e1*old1 + c_e2*old2 + c_e3*old3   (PLMS order weights; DDIM: c_e0 = 1)
 *   pred_x0 = (x - sqrt_one_minus_at * e_t') / sqrt(a_t)
 *   x_prev = sqrt(a_prev) * pred_x0 + dir_coef * e_t' + sigma * noise
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_sampler_desc {
  const float* x;
  const float* eps;       /* [n] or, with cfg_scale != 0, [2n]: uncond half then cond half */
  const float* old1;
  const float* old2;
  const float* old3;
  const float* noise;     /* NULL when sigma == 0 */
  float* x_prev;
  float* pred_x0;         /* optional */
  float* eps_out;         /* optional: guided (combined) eps e_t before multistep weights */
  long long n;
  float cfg_scale;        /* 0 = no guidance (eps has n elements) */
  float c_e0, c_e1, c_e2, c_e3;
  float sqrt_at, sqrt_one_minus_at, sqrt_a_prev, dir_coef, sigma;
} qd_sampler_desc;

int qd_sampler_step(const qd_sampler_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_ancestral_step -- the ancestral DDPM update: posterior mean of (x0, x_t) plus scaled noise.
 *   ddpm_steps of the CIFAR script        ddim/functions/denoising.py:53-65  (x0 clamped, sigma = sqrt(beta_t))
 *   LatentDiffusion p_sample (-v)         ldm/models/diffusion/ddpm.py:220-233, 1052-1112
 *                                         (predict_start_from_noise + q_posterior, no clamp, sigma = exp(0.5 logvar))
 *   x0 = c_x * x - c_e * eps;  if (clamp) x0 = clamp(x0, -1, 1)
 *   x_prev = m_x0 * x0 + m_x * x + sigma * noise          (no noise term when noise == NULL, e.g. t == 0)
 * All tensors fp32, n elements each.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_ancestral_desc {
  const float* x;
  const float* eps;
  const float* noise;     /* NULL: no noise term */
  float* x_prev;
  float* pred_x0;         /* optional: the (clamped) x0 */
  long long n;
  float c_x, c_e;
  float m_x0, m_x;
  float sigma;
  int32_t clamp;
} qd_ancestral_desc;

int qd_ancestral_step(const qd_ancestral_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * qd_weight_scale_search -- the channel-wise 'mse' initialisation of an asymmetric n-bit weight quantizer
 * (UniformAffineQuantizer.init_quantization_scale, qdiff/quant_layer.py:112-190), one row = one output channel.
 *   Row r is w[r * ld + k] for k in [k0, k1) (one split-shortcut half, or the whole row).  With x_max, x_min its extremes
 *   (no clamp to 0), candidate i = 0..79 in fp32 as the reference computes it:
 *     s_i = (float)(1.0 - 0.01 * i)  (double, then rounded)     new_max = x_max * s_i, new_min = x_min * s_i
 *     delta_i = (new_max - new_min) / (2^n - 1)                 zp_i = rne(-new_min / delta_i)
 *     xq = (clamp(rne(x / delta_i) + zp_i, 0, 2^n - 1) - zp_i) * delta_i       (IEEE division, fp32)
 *   score_i = sum over the row of |x - xq|^2.4, summed in float64 in a fixed order (the reference's 1/K factor, which
 *   cannot change the choice, is left out).  The chosen candidate is the first one with a strictly smaller score.
 *   Each |x - xq|^2.4 term is double pow() of the exact fp32 error: the float64 value to pow's last-bit accuracy.
 * Outputs per row: delta[r], zero_point[r] (fp32), index[r] (0..79); score[r] (optional, NULL: not written).
 * n_bits in [2, 8].  A row that is constant or holds a non-finite value has no candidate with a usable step (the reference
 * leaves delta at None): the call is refused with QD_ERR_UNSUPPORTED, naming the first such row.
 * The call synchronises `stream` to read that verdict back, so it cannot be captured into a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_wsearch_desc {
  const float* w;         /* [N, ld] fp32, row-major (OIHW flattened) */
  long long ld;           /* row pitch in elements */
  int32_t N;
  int32_t k0, k1;         /* column range [k0, k1) of every row, 0 <= k0 < k1 <= ld */
  int32_t n_bits;
  float* delta;           /* [N] */
  float* zero_point;      /* [N] */
  int32_t* index;         /* [N] chosen candidate */
  double* score;          /* [N] optional: the chosen candidate's score */
} qd_wsearch_desc;

int qd_weight_scale_search(const qd_wsearch_desc* d, qd_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Engine: a recorded program of the ops above for one UNet (QuantModel.forward,
 * qdiff/quant_model.py:68-69 -> UNetModel.forward openaimodel.py:745-782 / Model.forward
 * ddim/models/diffusion.py:308-360).  The host graph builder (qdiff_b200/graph.py) records ops
 * once; qd_engine_run replays them on a stream (optionally as one CUDA graph).  The engine owns
 * only the recorded descriptors and TMA maps; buffers belong to the caller.
 * ------------------------------------------------------------------------------------------ */
typedef struct qd_engine qd_engine;

enum qd_op_kind {
  QD_OP_GEMM = 1,
  QD_OP_QUANTIZE = 2,
  QD_OP_GROUPNORM = 3,
  QD_OP_LAYERNORM = 4,
  QD_OP_IM2COL = 5,
  QD_OP_ATTENTION = 6,
  QD_OP_TIMESTEP_EMB = 7,
  QD_OP_COPY2D = 8,
  QD_OP_NCHW_TO_NHWC = 9,
  QD_OP_NHWC_TO_NCHW = 10,
  QD_OP_AVGPOOL2X = 11,
  QD_OP_UPSAMPLE2X = 12,
  QD_OP_SPLIT3 = 13,
  QD_OP_ATTENTION_FP = 14,
  QD_OP_VQ_LOOKUP = 15,
  QD_OP_SOFTMAX_ROWS = 16,
  QD_OP_EMBED = 17        /* desc: qd_embed_desc */
};

/* generic argument block for the small helpers when recorded into an engine */
typedef struct qd_misc_desc {
  const float* src;
  float* dst;
  long long ld_src, ld_dst;
  int32_t a, b, c, d;   /* meaning per op: see qd_engine_add_op */
  const float* aux;     /* QD_OP_TIMESTEP_EMB: frequency table; QD_OP_VQ_LOOKUP: codebook [c][b] (a = rows, b = C, c = n_e);
                           QD_OP_SOFTMAX_ROWS: src == dst, a = rows, b = cols, ld_src = row pitch */
} qd_misc_desc;

int qd_engine_create(int device, qd_engine** out);
/* desc points at the matching qd_*_desc (qd_misc_desc for kinds 7..12, 15, 16; qd_embed_desc for QD_OP_EMBED); copied.
 * Every descriptor is checked here with the same rules its qd_* entry point applies (argument ranges, leading dimensions,
 * alignment of the base pointers), so a descriptor the kernels cannot take is refused when it is added, not at replay. */
int qd_engine_add_op(qd_engine* e, int kind, const void* desc);
int qd_engine_num_ops(const qd_engine* e);
int qd_engine_finalize(qd_engine* e);
int qd_engine_run(qd_engine* e, qd_stream_t stream);
/* run ops [first, last) only (debug / per-layer parity) */
int qd_engine_run_range(qd_engine* e, int first, int last, qd_stream_t stream);
void qd_engine_destroy(qd_engine* e);

const char* qd_last_error(void);
int qd_num_sms(void);
/* number of kernels this library launched since load (bench.py "gpu_launches") */
long long qd_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* QDIFF_B200_H */
