/*
 * dwm_b200 — C ABI of the H100-native (sm_90a) kernels behind OpenDWM's CTSD
 * denoising hot path.
 *
 * The reference (SenseTime-FVG/OpenDWM) has no C/FFI interface of its own: its
 * plug point is the JSON `_class_name` factory (src/dwm/common.py:133-172) that
 * instantiates `dwm.models.crossview_temporal_dit.DiTCrossviewTemporalConditionModel`
 * etc.  The Python mirror of those classes (src/dwm in this repo) calls the
 * entry points below through ctypes.  Each entry point cites the reference
 * code whose arithmetic it replaces.
 *
 * Conventions
 *  - every function returns 0 on success, <0 on error; the message is available
 *    from dwm_b200_last_error() (thread local).
 *  - all pointers are DEVICE pointers owned by the caller (PyTorch); nothing is
 *    allocated here.  Launches are asynchronous on `stream`.
 *  - 16-bit activations/weights are bf16 (DWM_BF16) or fp16 (DWM_F16);
 *    opt-in 8-bit GEMM operands are E4M3 (DWM_E4M3) with one fp32 scale per row;
 *    biases, norm weights, modulation vectors, residual streams are fp32.
 *  - there is NO CPU fallback: calling these without a Hopper (sm_90a) GPU fails.
 *  - alignment (dwm_b200_linear, dwm_b200_conv): A / W / x / weight / out, bias, resid, gate,
 *    blend_x and every peer_out are 16-byte aligned; the fp32 row pitches ldr, gate_ld and
 *    ldx are multiples of 4 elements (16-byte rows), the 16-bit pitches multiples of 8.  The
 *    epilogue reads these rows as float2 / float4 and the RESID rows are also prefetched by
 *    bulk copies; a call that breaks a rule returns < 0 before anything is launched.
 */
#ifndef DWM_B200_H_
#define DWM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dwm_stream_t; /* cudaStream_t */

enum dwm_dtype { DWM_BF16 = 0, DWM_F16 = 1, DWM_F32 = 2, DWM_E4M3 = 3 };
/* DWM_ACT_QUICK_GELU: x * sigmoid(1.702 x) (CLIP-L's quick_gelu); DWM_EPI_STORE with
 * 16-bit operands only. */
enum dwm_act { DWM_ACT_NONE = 0, DWM_ACT_GELU_TANH = 1, DWM_ACT_GELU_ERF = 2, DWM_ACT_SILU = 3, DWM_ACT_RELU = 4,
               DWM_ACT_QUICK_GELU = 5 };

/* Epilogues of dwm_b200_linear (all fused into the wgmma GEMM kernel). */
enum dwm_epilogue {
  /* out16[r(m), n] = act(acc + bias[n]) */
  DWM_EPI_STORE = 0,
  /* GEGLU (diffusers FeedForward activation_fn="geglu", used by
   * VTSelfAttentionBlock.ff_in / .ff, crossview_temporal.py:548,559):
   * weight rows are pre-packed in blocks of 256 = [128 value rows | 128 gate rows];
   * out16[m, j] = (acc_v + b_v) * gelu_erf(acc_g + b_g), out width N/2. */
  DWM_EPI_GEGLU = 1,
  /* fused q/k/v projection + per-head RMSNorm(q), RMSNorm(k) (head_dim 64;
   * diffusers Attention qk_norm="rms_norm", crossview_temporal.py:552-555):
   * columns [0,D) are q, [D,2D) k, [2D,3D) v with D = qk_region. */
  DWM_EPI_QKNORM = 2,
  /* fp32 residual stream update, optionally gated and alpha-blended:
   *   v = acc + bias[n];  v *= gate[item(m), n];  v += resid[rr(m), n];
   *   if blend_x: v = alpha[b(m)] * blend_x[m, n] + (1 - alpha[b(m)]) * v
   *   out32[m, n] = v
   * (JointTransformerBlock gated residuals; AlphaBlender crossview_temporal.py:53-72) */
  DWM_EPI_RESID = 3,
  /* out32[m, n] = act(acc + bias[n]) */
  DWM_EPI_F32 = 4,
  /* gated tanh-GELU (T5 v1.1 DenseGatedActDense, feed_forward_proj="gated-gelu"):
   * the weight packed as for DWM_EPI_GEGLU with value rows wi_1 and gate rows wi_0;
   * out16[m, j] = (acc_v + b_v) * gelu_tanh(acc_g + b_g), out width N/2.  16-bit operands. */
  DWM_EPI_GEGLU_TANH = 5
};

typedef struct dwm_linear_args {
  int64_t M, N, K;
  const void* A;   /* [M, K] 16-bit, row pitch lda elements */
  int64_t lda;
  const void* W;   /* [N, K] 16-bit (torch.nn.Linear weight layout), row pitch ldw */
  int64_t ldw;
  const float* bias; /* [N] or NULL */
  int dtype;       /* dwm_dtype of A, W and of 16-bit outputs */
  int epilogue;    /* dwm_epilogue */
  int act;         /* dwm_act (STORE / F32 epilogues) */
  void* out;
  int64_t ldo;     /* row pitch of out, elements */
  /* item structure of the M rows: item(m) = m / rows_per_item (0 => one item).
   * 16-bit outputs go to row  item * out_item_stride + m % rows_per_item + out_row_offset
   * (lets sample and context tokens of one view-frame land in one joint buffer).
   * With rows_per_item > 0, 16-bit epilogues need out_item_stride >= rows_per_item (so that
   * items never share output rows); fp32 outputs (RESID, F32) are never remapped. */
  int64_t rows_per_item;
  int64_t out_item_stride;
  int64_t out_row_offset;
  /* QKNORM */
  const float* q_norm_weight; /* [64] */
  const float* k_norm_weight; /* [64] */
  int64_t qk_region;          /* D */
  float eps;
  int qk_norm_regions;        /* regions [0, n) are normalised (0 => default 2: q and k);
                                 region 0 uses q_norm_weight, region 1 k_norm_weight */
  /* RESID */
  const float* resid;   /* fp32 [*, ldr] or NULL */
  int64_t ldr;
  int64_t resid_row_mod; /* rr(m) = m % resid_row_mod if > 0; m if 0; item(m) if < 0 */
  const float* gate;    /* fp32 [items, gate_ld] or NULL */
  int64_t gate_ld;
  const float* blend_x; /* fp32 [M, ldx] or NULL */
  int64_t ldx;
  const float* alpha;   /* fp32 [batches]; b(m) = m / rows_per_batch */
  int64_t rows_per_batch;
  /* fused compute + collective (16-bit epilogues): every output tile is ALSO stored to
   * the same element offset of n_peer_out peer buffers (device pointers into other GPUs'
   * memory, NVLink P2P / symmetric memory).  Used to scatter the K,V projection of a
   * frame shard straight into every peer's gathered K,V buffer, replacing GEMM +
   * all-gather by one kernel. */
  void* peer_out[8];
  int n_peer_out;
  /* FP8 (dtype == DWM_E4M3): A and W are E4M3 with row scales, a_scale fp32 [M] and
   * w_scale fp32 [N] (one per weight row = output channel, in packed row order).  The fp32
   * accumulator of A8 . W8^T is multiplied by a_scale[m] * w_scale[n] before the bias; the
   * epilogue then runs as for 16-bit operands, with out_dtype (DWM_BF16 / DWM_F16) the type
   * of its 16-bit outputs.  K, lda and ldw must be multiples of 16. */
  const float* a_scale;
  const float* w_scale;
  int out_dtype;
} dwm_linear_args;

const char* dwm_b200_version(void);
const char* dwm_b200_last_error(void);
/* Runtime switches (no reference counterpart; they select between kernels that must agree,
 * which tests/ use for kernel-variant parity): "gemm_2cta" = 1 routes dwm_b200_linear (M >= 512)
 * to the kernel for clusters of two CTAs that share each weight tile by TMA multicast, 0 to the
 * 1-CTA kernel (default: env DWM_GEMM_2CTA, else 1);
 * "attn_tc" routes eligible head_dim-64 attention (contiguous sequences; gathered sequences of
 * whole `inner`-token units with an optional unit mask): >= 1 = wgmma kernel (default), 0 =
 * mma.sync kernel, -1 = re-read env DWM_ATTN_TC / DWM_ATTN_LEGACY;
 * "ln_staged" = 1 (default) runs large LayerNorms through the bulk-copy staged kernel, 0
 * keeps the register-resident kernel;
 * "resid_tma" = 1 (default) has the TMA unit prefetch the residual / blend rows of a
 * DWM_EPI_RESID tile into L2 while its MMAs run, 0 leaves them to the epilogue's loads;
 * "gemm_bn" = 0 (default) picks the GEMM tile width (128 or 256 columns) by wave
 * efficiency, 128 / 256 force it (GEGLU always uses 256);
 * "conv_2cta" = 1 (default) runs convolutions with >= 2 pixel tiles per SM on clusters of two
 * CTAs sharing each weight slice, 0 on the 1-CTA kernel; "conv_halo" = 1 (default) routes kw = 3,
 * W >= 128, C_out-tile <= 128 convolutions to the halo-row kernel (one load of a 130-pixel
 * row segment serves the three dw taps), 0 to the per-tap kernels. */
int dwm_b200_set_option(const char* name, int value);

/* y = epilogue(A @ W^T): replaces every torch.nn.Linear / 1x1 / patchify conv on the
 * path (diffusers Attention.to_q/k/v/to_out, FeedForward, AdaLayerNormZero.linear,
 * PatchEmbed.proj, SD3Transformer2DModel.proj_out; call sites
 * crossview_temporal_dit.py:421-431,517-521,599-600, crossview_temporal.py:562-582). */
int dwm_b200_linear(const dwm_linear_args* args, dwm_stream_t stream);

/* ---- attention -------------------------------------------------------------------- */
/* Multi-head softmax attention over GATHERED token groups of the fused q|k|v buffer
 * produced by DWM_EPI_QKNORM (no permuted copy).  Position j of group (g0,g1,g2) is row
 *   g0*group_strides[0] + g1*group_strides[1] + g2*group_strides[2]
 *     + (j / inner) * stride_outer + (j % inner) * stride_inner
 * q = cols [h*64, h*64+64), k = D + ..., v = 2D + ....  Output rows use the out_* strides;
 * with split > 0, positions j >= split go to out2 row g*(seq-split) + (j-split)
 * (context tokens of the joint attention).  mask: uint8 [batches, n_outer, n_outer],
 * entry [g0 / mask_div, jq / inner, jk / inner] != 0 means "attend".  A query whose every
 * key is masked gets an output of 0 (F.scaled_dot_product_attention gives NaN there; a NaN
 * would spread through the whole residual stream).  Rows of qkv that no sequence position
 * maps to (padding between groups) are never used and may hold anything, NaN included.
 * Replaces F.scaled_dot_product_attention inside diffusers AttnProcessor2_0 /
 * JointAttnProcessor2_0 and the einops regroupings of
 * crossview_temporal_dit.py:300-315 (cross-view rowwise + mask expansion) and :335-361
 * (temporal full / rowwise / pointwise). */
typedef struct dwm_attention_args {
  const void* qkv;
  int64_t ld;
  int64_t D;
  int heads;
  int head_dim; /* must be 64 */
  int dtype;
  int64_t group_dims[3];
  int64_t group_strides[3];
  int seq;
  int inner;
  int64_t stride_outer, stride_inner;
  void* out;
  int64_t ldo;
  int64_t out_group_strides[3];
  int64_t out_stride_outer, out_stride_inner;
  int split;
  void* out2;
  int64_t ldo2;
  const unsigned char* mask;
  int mask_div;
  int n_outer;
  float scale;
  /* Optional separate key/value source (kv != NULL): keys at column k_col + h*64, values
   * at v_col + h*64 of `kv`, with their own row formula.  Used when the frame axis is
   * sharded across GPUs: queries are the local frames, keys/values the all-gathered
   * frames of every rank (position j = rank*T_local + t_local). */
  const void* kv;
  int64_t ld_kv;
  int64_t k_col, v_col;
  int64_t kv_group_strides[3];
  int seq_kv;
  int inner_kv;
  int64_t kv_stride_outer, kv_stride_inner;
  /* Mask row of query unit 0 (>= 0; 0 = the unsharded meaning): query unit u = jq / inner reads
   * mask row mask_q_offset + u, while key units index the mask over all n_outer units.  Used
   * when the view axis is sharded: queries are the V_local views from v_offset, keys / values
   * (kv) the gathered views of every rank, and mask_q_offset = v_offset.  With a mask and
   * mask_q_offset > 0, mask_q_offset + (seq - 1) / inner must be < n_outer (the last query unit
   * reads a mask row).  Separate K,V with a unit mask and whole
   * units (seq_kv = n_outer * inner_kv, inner_kv = inner <= 128, n_outer <= 32, seq_kv > 64,
   * unit strides 1) runs on the wgmma kernel that also runs the unsharded call over all units,
   * and every local query row is bit-identical to its row of that call; separate K,V without a
   * mask runs on the mma.sync kernel. */
  int mask_q_offset;
} dwm_attention_args;

int dwm_b200_attention(const dwm_attention_args* args, dwm_stream_t stream);

/* Text-encoder attention (CLIP / T5 self-attention over 77-token prompts): dwm_b200_attention
 * with causal != 0 masking key j > query i (CLIP), or with bias (fp32 [heads, seq, seq], shared
 * by every group) added to the scaled scores before the softmax (T5's relative-position bias);
 * one of the two.  Contiguous sequences only (group_dims[1] = group_dims[2] = 1, inner = seq =
 * group_strides[0], unit strides, no mask / kv / split), any seq >= 1.  They run on the wgmma
 * kernel whatever "attn_tc" says; a call it cannot serve returns < 0. */
int dwm_b200_attention_text(const dwm_attention_args* args, int causal, const float* bias,
                            dwm_stream_t stream);

/* ---- row ops ---------------------------------------------------------------------- */
/* LayerNorm over the last dim of an fp32 residual stream, emitting the 16-bit GEMM operand.
 *   t = x[m] (+ add_item[m / rows_per_item]) (+ add_full[m]);  if sum_out: sum_out[m] = t
 *   n = (t - mean) * rsqrt(var + eps) (* weight + bias)
 *   out[m]  = n * (1 + scale[item]) + shift[item]      (modulation optional)
 *   out2[m] = n * (1 + scale2[item]) + shift2[item]    (SD35AdaLayerNormZeroX, optional)
 * Replaces torch.nn.LayerNorm (crossview_temporal.py:545,550,558), AdaLayerNormZero /
 * AdaLayerNormContinuous modulation and the `hidden_states + view_emb` adds
 * (crossview_temporal_dit.py:229-230,334,491-494). */
typedef struct dwm_layernorm_args {
  int64_t M, D;
  const float* x;
  int64_t ldx;
  const float* add_item; /* [items, add_item_ld] or NULL */
  int64_t add_item_ld;
  const float* add_full; /* [M, add_full_ld] or NULL */
  int64_t add_full_ld;
  int64_t rows_per_item; /* item(m) = m / rows_per_item (0 => single item) */
  float* sum_out;        /* optional fp32 [M, ld_sum] */
  int64_t ld_sum;
  const float* weight;   /* [D] or NULL */
  const float* bias;     /* [D] or NULL */
  float eps;
  const float* shift;    /* [items, mod_ld] or NULL */
  const float* scale;
  const float* shift2;
  const float* scale2;
  int64_t mod_ld;
  void* out;
  int64_t ldo;
  void* out2;
  int64_t ldo2;
  int dtype;
  /* dtype == DWM_E4M3: out (and out2) are E4M3; each row is quantized from its fp32
   * modulated value with scale amax(|row|) / 448, written to out_scale[m] (out2_scale[m]). */
  float* out_scale;
  float* out2_scale;
} dwm_layernorm_args;

int dwm_b200_layernorm(const dwm_layernorm_args* args, dwm_stream_t stream);

/* RMSNorm of an fp32 stream (T5LayerNorm): out[m] = weight * x[m] * rsqrt(mean(x[m]^2) + eps),
 * statistics in fp32, out of dtype DWM_BF16 / DWM_F16 (the GEMM operand) or DWM_F32.  D and the
 * pitches ldx / ldo are multiples of 4; x, weight 16-byte and out 8-byte (fp32: 16-byte) aligned. */
int dwm_b200_rmsnorm(const float* x, int64_t M, int64_t D, int64_t ldx, const float* weight, float eps,
                     void* out, int64_t ldo, int dtype, dwm_stream_t stream);

/* Token (and absolute position) embedding gather into the fp32 residual stream of a text encoder:
 *   out[m, :] = tok[ids[m], :] (+ pos[m % seq, :])
 * ids int64 [M] (each < vocab; a bad id traps), tok fp32 [vocab, D], pos fp32 [>= seq, D] or NULL,
 * out fp32 [M, ldo].  One fp32 add: bit-exact against torch's embedding + add. */
int dwm_b200_embed(const int64_t* ids, int64_t M, int64_t seq, const float* tok, int64_t vocab,
                   const float* pos, int64_t D, float* out, int64_t ldo, dwm_stream_t stream);

/* Row-wise E4M3 quantization of a GEMM operand: x [M, K] (dtype DWM_BF16 / DWM_F16 / DWM_F32,
 * row pitch ld) -> out E4M3 [M, K] (pitch ldo bytes) and scale fp32 [M].  Per row:
 * amax = max |x|; amax == 0 -> scale 1, q = 0; otherwise inv = 448 / amax,
 * q = cvt.rn.satfinite.e4m3(x * inv), scale = amax / 448 (IEEE fp32 divisions).
 * K must be a multiple of 16.  Feeds the FP8 down / out projections (GELU, GEGLU and
 * attention outputs) and packs FP8 weights (one scale per output channel). */
int dwm_b200_quantize_rows(const void* x, int64_t M, int64_t K, int64_t ld, int dtype, void* out,
                           int64_t ldo, float* scale, dwm_stream_t stream);

/* out16[i] = act(in32[i]) over n elements: SiLU(temb) feeding the AdaLayerNormZero linears of
 * the joint blocks (called at crossview_temporal_dit.py:517-521) and the UNet ResBlock
 * time_emb_proj (crossview_temporal.py:104-113); plain 16-bit casts of GEMM / conv operands. */
int dwm_b200_act_cast(const float* in, void* out, int64_t n, int act, int dtype, dwm_stream_t stream);

/* diffusers Timesteps(num_channels, flip_sin_to_cos, downscale_freq_shift): sinusoidal
 * embedding of n fp32 scalars -> 16-bit [n, channels] (crossview_temporal_dit.py:153-154,
 * 163-164, 431-439, 528-532, 559-563). */
int dwm_b200_sinusoid(const float* t, int64_t n, int channels, int flip_sin_to_cos,
                      float downscale_freq_shift, void* out, int64_t ldo, int dtype,
                      dwm_stream_t stream);

/* PatchEmbed im2col: latents [items, C, H, W] (fp32) -> 16-bit [items*(H/p)*(W/p), C*p*p],
 * column = c*p*p + py*p + px (Conv2d weight flattening), crossview_temporal_dit.py:421. */
int dwm_b200_patchify(const float* x, int64_t items, int C, int H, int W, int patch, void* out,
                      int64_t ldo, int dtype, dwm_stream_t stream);

/* Fused tail of one denoising step (ctsd.py:2071-2090 + crossview_temporal_dit.py:603-621 +
 * temporal_independent.py:176-197): un-patchify the proj_out tokens, classifier-free
 * guidance combine, per-frame Euler update with INT32 sigma indices, round to the model
 * dtype like the reference, keep frames outside the schedule range unchanged.
 *   tokens: fp32 [cfg*B*T*V*S, p*p*C], column = (py*p+px)*C + c, uncond half first
 *   idx:    int32 [B, T, V];  sigmas: fp32 [n_sigmas];  in_range: uint8 [T]
 *   latents (in/out): fp32 [B, T, V, C, H, W];  noise_pred (optional out): same shape
 *   round_dtype: DWM_BF16 / DWM_F16 rounds the updated latent like
 *   `prev_sample.to(model_output.dtype)`; DWM_F32 keeps fp32. */
int dwm_b200_cfg_euler_step(const float* tokens, int64_t ld_tok, int cfg, float guidance_scale,
                            int64_t B, int64_t T, int64_t V, int C, int H, int W, int patch,
                            const int32_t* idx, const float* sigmas, int n_sigmas,
                            const unsigned char* in_range, float* latents, float* noise_pred,
                            int round_dtype, dwm_stream_t stream);

/* FlowMatchEulerDiscreteScheduler.step_by_indices (temporal_independent.py:176-197) on a
 * latent-layout model output: sample[e] += (sigmas[idx[e/inner]+1] - sigmas[idx[e/inner]]) *
 * model_output[e], rounded to round_dtype; idx int32 [n/inner]. */
int dwm_b200_euler_step_by_indices(const float* model_output, float* sample, int64_t n,
                                   int64_t inner, const int32_t* idx, const float* sigmas,
                                   int n_sigmas, int round_dtype, dwm_stream_t stream);

/* ---- convolution -------------------------------------------------------------------- */
/* im2col-free convolution (implicit GEMM on wgmma) over channels-last activations:
 *   x      16-bit [nb, tp, h, w, c_in]   (tp includes the KT-1 leading causal frames)
 *   weight 16-bit [kt*kh*kw, c_out, c_in] (tap-major: tap = (dt*kh + dh)*kw + dw)
 *   out    rows = nb*(tp-kt+1)*h*w pixels, c_out columns (channels-last), pitch ldo
 * spatial zero padding kh/2, kw/2; no implicit temporal padding.  c_out must be a multiple
 * of 32 (pad the weight rows); tiles of 256 / 128 / 64 / 32 output channels.  Epilogues: DWM_EPI_STORE (16-bit,
 * bias + act), DWM_EPI_F32, DWM_EPI_RESID (fp32: acc + bias + resid).  Opt-in E4M3 x and
 * weight with per-volume / per-channel scales (a_scale, w_scale below): RESID, and F32 when
 * c_out is a multiple of 128 (the VAE ResNet conv1).
 * Replaces diffusers CogVideoXCausalConv3d / CogVideoXUpsample3D.conv inside
 * AutoencoderKLCogVideoX.decode (called at ctsd.py:1634-1640, 1615-1617) and the
 * AdapterResnetBlock 3x3 convs (adapters.py:20). */
typedef struct dwm_conv_args {
  const void* x;
  int64_t nb, tp, h, w, c_in;
  const void* weight;
  int kt, kh, kw;
  int64_t c_out;
  const float* bias;
  int dtype;
  int epilogue;
  int act;
  void* out;
  int64_t ldo;
  const float* resid;
  int64_t ldr;
  /* resid_per_item != 0: `resid` holds ONE row per item of rows_per_item consecutive output
   * pixels (ResnetBlock2D's `+ time_emb_proj(silu(temb))[:, :, None, None]`).  resid,
   * resid_per_item and blend_x need DWM_EPI_RESID; output rows are never remapped. */
  int resid_per_item;
  int64_t rows_per_item;
  /* optional AlphaBlender after the residual (DWM_EPI_RESID):
   * out = alpha[b] * blend_x + (1 - alpha[b]) * (acc + bias + resid), b = row / rows_per_batch */
  const float* blend_x;
  int64_t ldx;
  const float* alpha;
  int64_t rows_per_batch;
  /* FP8 (dtype == DWM_E4M3; epilogue DWM_EPI_RESID, or DWM_EPI_F32 with c_out % 128 == 0):
   * x and weight are E4M3, with
   * a_scale fp32 [nb] (one scale per VOLUME: every tap of an output pixel reads the same
   * volume) and w_scale fp32 [c_out] (one per output channel, over all taps and input
   * channels; 8-byte aligned).  The fp32 accumulator is multiplied by a_scale[nb] *
   * w_scale[n] before the bias / residual / blend.  c_in must be a multiple of 16; a ragged
   * last 128-channel block is zero-filled.  Channel blocks are 128 E4M3 elements. */
  const float* a_scale;
  const float* w_scale;
} dwm_conv_args;

int dwm_b200_conv(const dwm_conv_args* args, dwm_stream_t stream);

/* ---- GroupNorm / SpatialNorm3D / upsampling pixel kernels (channels-last fp32 activations) of
 * the VAE decoders the reference calls at src/dwm/pipelines/ctsd.py:1609-1643, 2095-2098 and of
 * the UNet ResBlocks / TransformerModel (src/dwm/models/crossview_temporal.py:75-164, 288-289) -- */
/* GroupNorm statistics: sums[n][g] = (sum, sum of squares) over the C/groups channels of
 * group g and all `pixels` (= T*H*W) of volume n; `sums` (double [nb, groups, 2]) is zeroed
 * here.  (torch.nn.GroupNorm in ResnetBlock2D / TemporalResnetBlock, crossview_temporal.py:104-113;
 * diffusers CogVideoXSpatialNorm3D.norm_layer, where statistics are per decode chunk.) */
int dwm_b200_groupnorm_stats(const float* x, int64_t nb, int64_t pixels, int C, int groups,
                             double* sums, dwm_stream_t stream);
/* out16[n, out_t0 + t, h, w, c] = act( GN(x)*gamma+beta [ * zy[nearest] + zb[nearest] ] )
 * with zy = conv_y(zq), zb = conv_b(zq) given at the latent resolution [nb, Tz, hz, wz, C]
 * (nearest-neighbour lookup, first frame mapped separately when T is odd > 1).  Writes
 * into a 16-bit channels-last buffer of out_T frames at frame offset out_t0 (the leading
 * frames hold the causal-conv cache).  zy = zb = NULL gives plain GroupNorm (+SiLU), the
 * `norm -> nonlinearity` prefix of every ResBlock convolution (crossview_temporal.py:126-158)
 * and of `conv_norm_out -> conv_act` (crossview_temporal_unet.py:815-817). */
int dwm_b200_spatialnorm_silu(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                              int groups, const double* sums, float eps, const float* gamma,
                              const float* beta, const float* zy, const float* zb, int Tz, int hz,
                              int wz, int apply_silu, void* out, int64_t out_T, int64_t out_t0,
                              int dtype, dwm_stream_t stream);
/* GroupNorm(+SiLU) with an E4M3 output, the operand of an FP8 dwm_b200_conv: the values of
 * dwm_b200_spatialnorm_silu with zy = zb = NULL (the fp32 y the 16-bit path would round),
 * quantized with ONE scale per volume n: amax = max |y| over the volume's T frames;
 * amax == 0 -> out_scale[n] = 1, q = 0; otherwise q = cvt.rn.satfinite.e4m3(y * (448 / amax)),
 * out_scale[n] = amax / 448 (IEEE fp32).  out is E4M3 [nb, out_T, H, W, C]; only frames
 * [out_t0, out_t0 + T) are written (the leading cache frames stay as they are).  Two passes
 * over x (amax, then quantize); out_scale (fp32 [nb]) is the amax scratch in between, so the
 * call allocates nothing.  C must be a multiple of 16. */
int dwm_b200_groupnorm_silu_e4m3(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                 int groups, const double* sums, float eps, const float* gamma,
                                 const float* beta, int apply_silu, void* out, int64_t out_T,
                                 int64_t out_t0, float* out_scale, dwm_stream_t stream);
/* SpatialNorm3D(+SiLU) with an E4M3 output, the operand of an FP8 causal dwm_b200_conv of the
 * CogVideoX decoder: the values y of dwm_b200_spatialnorm_silu (zy / zb and the latent frame map
 * included), quantized with ONE scale per volume n by the rule of dwm_b200_groupnorm_silu_e4m3,
 * into frames [out_t0, out_t0 + T) of out E4M3 [nb, out_T, H, W, C].  The causal-conv cache:
 * tail_in (16-bit [nb, 2, H, W, C] of type tail_dtype, or NULL) is the previous chunk's cached
 * tail; the volume's amax covers it and y, and it is quantized with that scale into frames
 * out_t0 - 2, out_t0 - 1 (out_t0 >= 2).  Without tail_in those frames are left as they are (the
 * caller copies frame out_t0's bytes there: they share the scale).  tail_out (same layout, may
 * be tail_in) receives the next chunk's cache: the operand's last two frames in 16 bit, y
 * rounded to tail_dtype or, for T = 1, tail_in's frame 1 (else y's replica) and y.  Passes:
 * amax, quantize, scale; out_scale (fp32 [nb]) is the amax scratch, so nothing is allocated.
 * C must be a multiple of 16. */
int dwm_b200_spatialnorm_silu_e4m3(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                   int groups, const double* sums, float eps, const float* gamma,
                                   const float* beta, const float* zy, const float* zb, int Tz, int hz,
                                   int wz, int apply_silu, void* out, int64_t out_T, int64_t out_t0,
                                   float* out_scale, const void* tail_in, void* tail_out, int tail_dtype,
                                   dwm_stream_t stream);
/* Frame-shard GroupNorm(+SiLU) of the temporal ResBlock convolutions: x holds T of a window's
 * frames and `sums` (double [nb, groups, 2]) the statistics already summed over the window's
 * `stat_frames` frames, so mean and variance use stat_frames*H*W*C/groups samples.  out is the
 * shard's temporal-conv operand [nb, T + 2, H, W, C] with the local frames at 1 ... T.  Local
 * frame 0 is also stored at frame prev_out_T - 1 of prev_out (the previous shard's operand
 * [nb, prev_out_T, H, W, C]) and local frame T - 1 at frame 0 of next_out ([nb, next_out_T, ...]);
 * the neighbours store their boundary frames into out the same way.  A NULL neighbour (first /
 * last shard of the window) stores the own halo frame as zero, the conv's time padding.  The
 * values are those of dwm_b200_spatialnorm_silu with zy = zb = NULL for the same sums. */
int dwm_b200_groupnorm_silu_halo(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                 int groups, const double* sums, int64_t stat_frames, float eps,
                                 const float* gamma, const float* beta, int apply_silu, void* out,
                                 void* prev_out, int64_t prev_out_T, void* next_out,
                                 int64_t next_out_T, int dtype, dwm_stream_t stream);
/* E4M3 frame-shard variant, pass 1: amax[n] (fp32 [nb]) = max |y| over the shard's frames of
 * volume n, y as in dwm_b200_groupnorm_silu_halo.  Reduce it with MAX over the window's shards. */
int dwm_b200_groupnorm_silu_e4m3_amax(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W,
                                      int C, int groups, const double* sums, int64_t stat_frames,
                                      float eps, const float* gamma, const float* beta,
                                      int apply_silu, float* amax, dwm_stream_t stream);
/* Pass 2: quantizes with the given (window-wide) amax exactly as dwm_b200_groupnorm_silu_e4m3
 * does for that amax, writes out_scale[n] (may alias amax), and stores the frames and halo
 * frames as dwm_b200_groupnorm_silu_halo does. */
int dwm_b200_groupnorm_silu_e4m3_halo(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W,
                                      int C, int groups, const double* sums, int64_t stat_frames,
                                      float eps, const float* gamma, const float* beta,
                                      int apply_silu, const float* amax, void* out, void* prev_out,
                                      int64_t prev_out_T, void* next_out, int64_t next_out_T,
                                      float* out_scale, dwm_stream_t stream);
/* CogVideoXUpsample3D interpolation: nearest x2 in H, W and (compress_time) in T, where an
 * odd T > 1 keeps its first frame un-doubled in time; fp32 in, 16-bit out
 * [nb, T', 2H, 2W, C].  Also the F.interpolate(nearest, x2) of the UNet / AutoencoderKL
 * up-samplers (crossview_temporal_unet.py:263-266, 347-350). */
int dwm_b200_upsample_nearest(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                              int compress_time, void* out, int dtype, dwm_stream_t stream);

/* out[i] = s0[i / inner] * x[i] + s1[i / inner] * y[i]: DDPMScheduler.add_noise /
 * get_velocity with per-(b,t,v) coefficients (temporal_independent.py:8-45). */
int dwm_b200_lincomb2(const float* x, const float* y, const float* s0, const float* s1, int64_t n,
                      int64_t inner, float* out, dwm_stream_t stream);

/* Fused CFG combine + DPM-Solver++ step (midpoint, order <= 2) of
 * src/dwm/schedulers/dpm_solver.py, in place over n fp32 elements:
 *   m  = w_uncond * u + w_cond * c      (cfg 2: pred = [u ; c], 2n; cfg 1: m = pred, n)
 *   x0 = c_x * latents + c_m * m
 *   p  = k_s * latents + k_0 * x0 (+ k_1 * x0_prev when order == 2)
 *   x0_prev <- x0;  latents <- p
 * row: fp32 [6] in device memory, (c_x, c_m, k_s, k_0, k_1, order) with order 1 or 2, so that
 * a captured CUDA graph replays whichever step was loaded into it.  Every line is rounded to
 * fp32 as dwm_b200_lincomb2 rounds it; a first-order step does not read x0_prev.  latents and
 * x0_prev must not overlap each other, pred or row. */
int dwm_b200_cfg_dpmpp_step(const float* pred, int cfg, float w_uncond, float w_cond, int64_t n,
                            const float* row, float* latents, float* x0_prev, dwm_stream_t stream);

/* y += a * x over n fp32 elements (adapter residual adds of the UNet,
 * crossview_temporal_unet.py:729-731, 759-761). */
int dwm_b200_axpy(const float* x, float* y, int64_t n, float a, dwm_stream_t stream);

/* out[r, :] = softmax(scale * x[r, :]) for fp32 scores -> 16-bit probabilities.  Replaces
 * the softmax inside F.scaled_dot_product_attention of the single-head (head_dim 512)
 * mid-block Attention of diffusers AutoencoderKL (called by the reference at
 * src/dwm/pipelines/ctsd.py:1633-1640, 2095-2098); Q K^T and P V run through dwm_b200_linear. */
int dwm_b200_softmax_rows(const float* x, int64_t rows, int64_t cols, int64_t ld, float scale,
                          void* out, int64_t ldo, int dtype, dwm_stream_t stream);

/* Fused CFG combine + DDIM update (eta = 0) with per-(b,t,v) INT32 timesteps
 * (reference src/dwm/schedulers/temporal_independent.py:67-170 + ctsd.py:1548-1575):
 *   pred     fp32 [cfg * n_items * inner] (uncond half first), latent layout
 *   latents  fp32 [n_items * inner] in/out;  timesteps int32 [n_items]
 *   prev_t = t - step_ratio; alpha_prev = alphas_cumprod[prev_t] or final_alpha_cumprod (< 0)
 *   prediction_type: 0 epsilon, 1 sample, 2 v_prediction. */
int dwm_b200_cfg_ddim_step(const float* pred, int cfg, float guidance_scale, int64_t n_items,
                           int64_t inner, const int32_t* timesteps, int step_ratio,
                           const float* alphas_cumprod, int n_alphas, float final_alpha_cumprod,
                           int prediction_type, float* latents, int round_dtype,
                           dwm_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DWM_B200_H_ */
