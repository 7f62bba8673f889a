/* libddpo_b200 -- C ABI of the H100 (sm_90a) DDPO hot path.
 *
 * The reference (jannerm/ddpo) has no FFI layer: its seam is a set of Python call
 * signatures between pipeline/*.py and ddpo.* whose arithmetic runs inside XLA.  This
 * header is what a binding for that path binds to; each entry point names the
 * reference code it replaces (file:line relative to the reference repo; "3P" marks
 * un-vendored diffusers 0.12.1 / optax 0.1.5 / jax 0.4.8 code reached from that line).
 *
 * Conventions
 *   - every pointer is CALLER-OWNED DEVICE memory (16-byte aligned, contiguous unless a
 *     leading dimension is given); the library never allocates tensors;
 *   - activations are NHWC ([B, H, W, C] == [M, C] row major); GEMM weights are bf16
 *     [N, K] with K contiguous (for a conv K = (tap, c_in), tap = ky*3+kx);
 *   - all calls are asynchronous on `stream` (a cudaStream_t passed as void*), issue no
 *     host synchronisation and are re-entrant across streams;
 *   - return value: DDPO_OK (0) or a negative ddpo_status; ddpo_last_error() returns a
 *     thread-local message.  No exception crosses the ABI.
 *   - reductions use fixed orders (no float atomics): results are bit-reproducible and
 *     independent of the batch size.
 */
#ifndef DDPO_B200_H_
#define DDPO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  DDPO_OK = 0,
  DDPO_ERR_INVALID = -1, /* bad argument */
  DDPO_ERR_CUDA = -2,    /* CUDA runtime / driver error */
  DDPO_ERR_UNSUPPORTED = -3
} ddpo_status;

const char* ddpo_last_error(void);
/* library / device sanity: returns the SM count of the current device (>0) or <0 */
int ddpo_device_sm_count(void);
int ddpo_abi_version(void);

/* ---------------------------------------------------------------- PRNG -------------
 * jax.random (threefry2x32), 3P jax==0.4.8; reference call sites
 * pipeline/policy_gradient.py:51,201,244-245; pipeline_flax_stable_diffusion.py:196-197,232,252 */
/* host: split(key) -> num keys (out: [num][2]) */
int ddpo_threefry_split_host(const uint32_t key[2], int num, uint32_t* out);
/* host: PRNGKey(seed) */
int ddpo_prng_key_host(uint64_t seed, uint32_t out[2]);
/* device: jax.random.normal(key, shape with n elements) -> out[n] fp32; key is a DEVICE pointer to 2 words */
int ddpo_threefry_normal(const uint32_t* key_dev, float* out, int64_t n, void* stream);

/* ------------------------------------------------------------ DDIM scheduler -------
 * FlaxDDIMScheduler.step  (ddpo/diffusers_patch/scheduling_ddim_flax.py:229-361) fused with the
 * classifier-free-guidance combine (pipeline_flax_stable_diffusion.py:226-229,
 * training/policy_gradient.py:103-105). */
typedef struct {
  const float* eps_uncond;     /* [B, n] model output, unconditional branch */
  const float* eps_cond;       /* [B, n] model output, text branch (== eps_uncond & guidance 1 for no CFG) */
  const float* sample;         /* [B, n] x_t */
  const float* alphas_cumprod; /* [num_train_timesteps] */
  const int32_t* timesteps;    /* [B] (timestep_stride 1) or [1] (timestep_stride 0) */
  int timestep_stride;
  float final_alpha_cumprod;
  int step_ratio;              /* num_train_timesteps // num_inference_steps */
  float guidance_scale;
  float eta;
  int batch;
  int n;                       /* C*H*W elements per sample */
  float* workspace;            /* >= batch*DDPO_DDIM_CHUNKS floats + batch uint32 counters, zero-initialised once */
  int prediction_type;         /* scheduling_ddim_flax.py:303-321: DDPO_PRED_EPSILON / _SAMPLE / _V_PREDICTION */
} ddpo_ddim_common;
#define DDPO_PRED_EPSILON 0
#define DDPO_PRED_SAMPLE 1
#define DDPO_PRED_V 2
#define DDPO_DDIM_CHUNKS 8

/* sample mode (scheduling_ddim_flax.py:346-348): prev = mean + sigma * normal(key) ; log_prob */
int ddpo_ddim_step_sample(const ddpo_ddim_common* c, const uint32_t* key_dev, float* prev_sample /*[B,n]*/,
                          float* log_prob /*[B]*/, void* stream);
/* score mode (:351-359 with prev_sample given): log_prob of prev_sample */
int ddpo_ddim_logprob_fwd(const ddpo_ddim_common* c, const float* prev_sample, float* log_prob, void* stream);
/* backward of score mode + CFG: d_eps_uncond, d_eps_cond given dL/dlog_prob [B] */
int ddpo_ddim_logprob_bwd(const ddpo_ddim_common* c, const float* prev_sample, const float* dlogp,
                          float* d_eps_uncond, float* d_eps_cond, void* stream);

/* ------------------------------------------------------------------ PPO ------------
 * ddpo/training/policy_gradient.py:121-134 (clipped surrogate, info) and its gradient.
 * info = {approx_kl, clipfrac, loss} averaged over `batch`.  `batch` may stack several reference-sized
 * micro-batches (the reference's train_batch_size = micro_batch) evaluated at the same parameters: the gradient
 * is d(sum over micro-batches of the micro-batch mean loss) = (dL_i/dlogp_i) / micro_batch, i.e. exactly what the
 * reference accumulates over that many train_step calls. */
int ddpo_ppo_loss(const float* log_prob, const float* old_log_prob, const float* advantages, int batch,
                  int micro_batch, float clip_range, float* info3, float* dlogp, void* stream);

/* --------------------------------------------------------- dense contractions ------
 * nn.Conv / nn.Dense of 3P diffusers FlaxUNet2DConditionModel (reached from
 * pipeline_flax_stable_diffusion.py:219-224 and training/policy_gradient.py:87-102). */
typedef struct {
  /* A operand: bf16 NHWC activations.  conv: [batch, h*stride, w*stride, c] per source (two sources =
   * channel concat [a0 | a1]); linear: a0 is [m, c0].  lda = elements between consecutive pixels/rows. */
  const void* a0;
  const void* a1;
  int c0, c1, lda0, lda1;
  int is_conv, batch, h, w; /* h, w: OUTPUT grid */
  int conv_stride;          /* 1, or 2 (3x3, symmetric pad 1: Flax padding ((1,1),(1,1))) */
  int taps;                 /* 9 (3x3, pad 1) or 1 (1x1 / linear) */
  int m;                    /* linear: rows */
  int n;                    /* output channels */
  const void* wt;           /* bf16 [n, taps*(c0+c1)] */
  const float* bias;        /* [n] or NULL */
  const float* rowvec;      /* [batch, rowvec_ld] or NULL: per-sample vector added to every row of the sample */
  int rows_per_sample, rowvec_ld;
  const float* residual;    /* fp32 [M, ld_res] or NULL */
  int ld_res;
  float* out_f32;           /* [M, ld_out] or NULL */
  void* out_bf16;           /* [M, ld_out] or NULL */
  int ld_out;
  int geglu;                /* out_bf16[M, n/2] = lin * gelu_tanh(gate); weight rows tile-interleaved */
  int accumulate_out;       /* out_f32 += */
  int bn_override;          /* 0 = planned; else the tile width (tests): 32, 64, 96, 128, 160, 192, 256 */
  void* aux_bf16;           /* GEGLU only, optional: bf16 [M, n] pre-activation (tile-interleaved, bias included) */
  int conv_pad;             /* 0 = the 3x3 default (symmetric pad 1); 1 = NO low-side padding: out[y,x] = sum in[s y + dy, s x + dx],
                               reads past the high edge are zero -- the VAE encoder's down-sample (pad ((0,1),(0,1)) + VALID) */
  float* gn_stats;          /* optional, with out_f32: fp32 [ceil(M/32), n, 2] = per 32-row slab and output column the (sum, sum
                               of squares) of the values written to out_f32.  The GroupNorm that consumes out_f32 takes its
                               statistics from these (ddpo_groupnorm_args.stats0/1) instead of reading the tensor twice. */
  int bm_override;          /* 0 = planned; else the tile height (tests): 64 or 128 */
} ddpo_igemm_args;
int ddpo_igemm(const ddpo_igemm_args* a, void* stream);
/* The output tile ddpo_igemm runs for an [m, k] x [k, n] product (k = taps * (c0 + c1)): plan = {BM, BN, CTAs per SM,
 * operand stages}.  A function of the shape alone; the overrides are those of ddpo_igemm_args.  No GPU needed. */
int ddpo_igemm_plan(int m, int n, int k, int geglu, int bm_override, int bn_override, int* plan);

/* ------------------------------------------------------------ normalisation --------
 * flax.linen.GroupNorm(32, eps 1e-5)(+nn.swish) / LayerNorm(eps 1e-5) of the 3P Flax U-Net
 * (FlaxResnetBlock2D norm1/2, FlaxTransformer2DModel.norm, conv_norm_out, BasicTransformerBlock norm1-3). */
typedef struct {
  const float* x0;      /* fp32 [batch, hw, c0] (pixel pitch ld0) */
  const float* x1;      /* optional second tensor: channel concat [x0 | x1] */
  int c0, c1, ld0, ld1;
  int batch, hw;
  const float* scale;   /* [c0+c1] */
  const float* bias;
  float eps;
  int silu;
  void* y_bf16;         /* bf16 [batch, hw, c] or NULL */
  float* y_f32;         /* fp32 [batch, hw, c] or NULL */
  void* raw_bf16;       /* bf16 copy of the un-normalised input or NULL */
  float* workspace;     /* ddpo_groupnorm_workspace_floats(); the first batch*chunks*64 floats (forward
                           statistics) must be kept until the backward call */
  int stats_only_skip;  /* 1: statistics already in workspace, only apply */
  const float* stats0;  /* optional: slab statistics [batch*hw/32, c0, 2] of x0 written by the GEMM that produced it
                           (ddpo_igemm_args.gn_stats); needs hw % 32 == 0.  With stats for every source the forward is ONE pass
                           over x (no statistics pass). */
  const float* stats1;  /* same for x1 [batch*hw/32, c1, 2] */
  int dy_bf16;          /* backward only: `dy` points to bf16 (the dgrad GEMM that produced it wrote its bf16 output) */
} ddpo_groupnorm_args;
int64_t ddpo_groupnorm_workspace_floats(int batch, int hw, int channels);
int ddpo_groupnorm_fwd(const ddpo_groupnorm_args* a, void* stream);
/* dx0/dx1 (+)= d/dx ; dscale/dbias += (parameter gradients always accumulate) */
int ddpo_groupnorm_bwd(const ddpo_groupnorm_args* a, const void* dy, float* dx0, float* dx1, int ldd0, int ldd1,
                       int accumulate, float* dscale, float* dbias, void* stream);
int ddpo_layernorm_fwd(const float* x, const float* scale, const float* bias, void* y_bf16, float* stats /*[m,2] or NULL*/,
                       int m, int c, float eps, void* stream);
int64_t ddpo_layernorm_bwd_workspace_floats(int m, int c);
/* dy: fp32, or bf16 when dy_bf16 != 0 (the output of the dgrad GEMM that feeds this norm) */
int ddpo_layernorm_bwd(const float* x, const float* scale, const float* stats, const void* dy, float* dx,
                       int accumulate, float* dscale, float* dbias, float* workspace, int m, int c, int dy_bf16,
                       void* stream);

/* --------------------------------------------------- layout / small layers ---------
 * weight re-layout: fp32 Flax params ([in,out] Dense, HWIO Conv == [(tap,cin), cout]) -> bf16 GEMM operands */
int ddpo_prep_weight(const float* src, void* dst_bf16, int k, int n, int ldk, int row_offset, int col_offset,
                     int geglu_bn, void* stream);
/* ld_dst (0 = taps*n): row pitch of dst; col_offset: first column written -- lets several weights share one K-concatenated
 * dgrad operand (the q/k/v input gradients of self-attention are ONE GEMM over K = 3C) */
int ddpo_prep_weight_dgrad(const float* src, void* dst_bf16, int taps, int k, int n, int ld_dst, int col_offset, void* stream);
int ddpo_permute_geglu_bias(const float* src, float* dst, int n, int bn, void* stream);
int ddpo_cast_bf16(const float* x, void* y_bf16, int64_t n, void* stream);
/* FlaxUpsample2D's jax.image.resize(nearest): out[i] = in[i/2] */
int ddpo_upsample2x_bf16(const float* x, void* y_bf16, int batch, int h, int w, int c, void* stream);
int ddpo_upsample2x_bwd(const float* dy, float* dx, int batch, int h, int w, int c, int accumulate, void* stream);
/* conv_in: NCHW fp32 latents -> NHWC fp32; conv_out: NHWC fp32 -> NCHW fp32 (N = 4).
 * gn_stats: optional [ceil(batch*h*w/32), cout, 2] slab statistics of y for the consuming GroupNorm (see ddpo_igemm_args) */
int ddpo_conv_in(const float* x_nchw, const float* w_hwio, const float* bias, float* y_nhwc, int batch, int cin,
                 int h, int w, int cout, float* gn_stats, void* stream);
int ddpo_conv_out(const float* x_nhwc, const float* w_hwio, const float* bias, float* y_nchw, int batch, int h,
                  int w, int cin, int cout, void* stream);
/* FlaxTimesteps(flip_sin_to_cos=True, freq_shift=0) and the M=batch Dense layers of the time embedding */
int ddpo_timestep_sincos(const int32_t* t, int t_stride, float* out, int batch, int dim, void* stream);
int ddpo_dense_small(const float* x, const float* w_in_out, const float* bias, float* y, int batch, int k, int n,
                     int silu_in, int silu_out, void* stream);
/* Grouped ddpo_dense_small for layers sharing the input x [batch, k] (the ResNet blocks' time_emb_proj Dense layers,
 * 3P FlaxResnetBlock2D): one launch; `groups_dev` is a DEVICE array of n_groups records
 * { int64 w_off, bias_off, y_off (floats, relative to params_base / y_base); int32 n, cta0 } sorted by cta0
 * (cta0 = running sum of ceil(n/32)); layer g's output is y_base + y_off[g], shape [batch, n].  Bit-identical to the
 * separate ddpo_dense_small calls (no activation on either side). */
int ddpo_dense_small_grouped(const float* x, const float* params_base, float* y_base, const void* groups_dev, int n_groups,
                             int total_ctas, int batch, int k, void* stream);

/* ---------------------------------------------------------------- attention --------
 * FlaxAttention core (3P diffusers attention_flax.py): softmax(Q K^T d^-0.5) V with d = head_dim, which must be 40,
 * 64, 80 or 160 (SD2: 64 everywhere; SD1.x: 40, 80, 160); any other value is DDPO_ERR_INVALID.
 * Head h of q, k, v and out sits at columns [h*d, h*d + d).  Every bf16 pointer must be 16-byte aligned and every
 * row pitch a multiple of 8 elements (16 bytes) and at least heads*d; otherwise DDPO_ERR_INVALID and nothing is
 * written.  Only the d real columns of each head are written. */
typedef struct {
  const void* q;  /* bf16 [batch, nq, ldq], head h at columns [h*d, h*d + d) */
  const void* k;  /* bf16 [batch, nk, ldk] */
  const void* v;  /* bf16 [batch, nk, ldv] */
  void* out;      /* bf16 [batch, nq, ldo] */
  float* lse;     /* fp32 [batch, heads, nq] log-sum-exp of the scaled scores, or NULL */
  int batch, heads, nq, nk, head_dim;
  int ldq, ldk, ldv, ldo;
  int causal;     /* 1: query i sees keys j <= i (3P transformers FlaxCLIPTextModel's causal mask); needs nq == nk */
} ddpo_attention_args;
int ddpo_attention_fwd(const ddpo_attention_args* a, void* stream);

/* ------------------------------------------------------- weight gradients ----------
 * dW[(tap, c_in), c_out] += sum_pixels X[pixel+tap, c_in] * dY[pixel, c_out], written in the Flax
 * parameter layout and accumulated (jax.grad at ddpo/training/policy_gradient.py:138 fused with
 * AccumulatingTrainState's grad_acc += g, :44-47). */
typedef struct {
  const void* dy;  /* bf16 [M, ldy] output gradient */
  int ldy, n;
  const void* x0;  /* bf16 NHWC forward input(s) of the layer (same geometry as ddpo_igemm_args) */
  const void* x1;
  int c0, c1, ldx0, ldx1;
  int is_conv, batch, h, w, conv_stride, taps, m;
  float* dw;       /* fp32 [taps*(c0+c1), n], accumulated */
  float* workspace;
  int64_t workspace_floats;
} ddpo_wgrad_args;
int64_t ddpo_wgrad_workspace_floats(const ddpo_wgrad_args* a);
int ddpo_wgrad(const ddpo_wgrad_args* a, void* stream);

/* attention backward (dQ, dK, dV; deterministic two-kernel scheme), see csrc/attention_bwd.cu.  Head dims, column
 * layout and alignment rules as for ddpo_attention_fwd (they apply to out, dout, dq, dk and dv too); the scale is
 * head_dim^-0.5. */
typedef struct {
  const void* q; const void* k; const void* v; const void* out; const void* dout; /* bf16 */
  const float* lse;  /* [batch, heads, nq] from the forward */
  float* delta;      /* [batch, heads, nq] scratch */
  void* dq; void* dk; void* dv; /* bf16 outputs */
  int batch, heads, nq, nk, head_dim;
  int ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;
} ddpo_attention_bwd_args;
int ddpo_attention_bwd(const ddpo_attention_bwd_args* a, void* stream);

/* ------------------------------------------------ memory-bound backward pieces ----- */
int64_t ddpo_colsum_workspace_floats(int m, int n, int rows_per_group);
/* out[g][n] (+)= sum of the rows of group g of dy (fp32 [m, ld]); optional bf16 copy of dy (GEMM operand).
 * rows_per_group == m: bias gradient; rows_per_group == H*W: per-sample sums (time-embedding projection). */
int ddpo_colsum_cast(const float* dy, int ld, void* y_bf16, float* out, int rows_per_group, int accumulate,
                     float* workspace, int m, int n, void* stream);
int ddpo_colsum_bf16(const void* x_bf16, int ld, float* out, int accumulate, float* workspace, int m, int n, void* stream);
/* dff: fp32 [m, n/2], or bf16 when dff_bf16 != 0 */
int ddpo_geglu_bwd(const void* pre_bf16, const void* dff, void* dpre_bf16, int64_t m, int n, int bn, int dff_bf16,
                   void* stream);
int64_t ddpo_conv_out_bwd_workspace_floats(int cin);
int ddpo_conv_out_bwd(const float* x_nhwc, const float* w_hwio, const float* dy_nchw, float* dx_nhwc, float* dw,
                      float* dbias, float* workspace, int batch, int h, int w, int cin, void* stream);
int64_t ddpo_conv_in_wgrad_workspace_floats(int cin, int cout);
int ddpo_conv_in_wgrad(const float* lat_nchw, const float* dx_nhwc, float* dw, float* workspace, int batch, int cin,
                       int h, int w, int cout, void* stream);
int ddpo_dense_small_bwd(const float* x, const float* w, const float* bias, const float* dy, float* dpre_ws, float* dw,
                         float* db, float* dx, int dx_accumulate, int batch, int k, int n, int silu_in, int silu_out,
                         void* stream);
int ddpo_dilate2x_bf16(const float* x, void* y_bf16, int batch, int h, int w, int c, void* stream);
int ddpo_copy2d(const float* src, int lds, float* dst, int ldd, int64_t rows, int cols, int accumulate, void* stream);
/* dst[r, :] = src[index[r], :] (fp32 rows of row_floats, a multiple of 4; index is a DEVICE int64 array): the
 * per-minibatch gather of (sample, timestep) rows out of the on-device trajectory buffer that replaces the
 * reference's host-side shuffles + per-step H2D (pipeline/policy_gradient.py:385-404,415-423) */
int ddpo_gather_rows(const float* src, const int64_t* index_dev, float* dst, int rows, int64_t row_floats, void* stream);

/* ---------------------------------------------------------------- VAE decode --------
 * vae_decode (pipeline/policy_gradient.py:174-182, ddpo/training/diffusion.py:105-112): latents / 0.18215 ->
 * 3P diffusers FlaxAutoencoderKL.decode -> (x/2 + 0.5).clip(0,1), NHWC.  The decoder's 3x3 / 1x1 convolutions,
 * GroupNorm(32, eps 1e-6)+swish and Dense layers run on ddpo_igemm / ddpo_groupnorm_fwd (pixel rows up to 1024 wide);
 * these three entry points are the pieces that are not GEMM shaped. */
/* out = post_quant_conv(latents / scaling): 1x1 conv on NCHW fp32, w_in_out [channels, channels] (HWIO 1x1) */
int ddpo_vae_post_quant(const float* latents_nchw, const float* w_in_out, const float* bias, float scaling, int batch,
                        int channels, int h, int w, float* out_nchw, void* stream);
/* probs[r, :] = softmax(scale * scores[r, :]) (bf16): FlaxAttentionBlock's single-head attention weights */
int ddpo_softmax_rows(const float* scores, int64_t ld_scores, float scale, void* probs_bf16, int64_t ld_probs, int rows,
                      int n, void* stream);
/* decoder conv_out (3x3, cin -> 3) on the normalised fp32 NHWC input; raw_nchw [B,3,H,W] (decoder .sample, optional)
 * and img_nhwc [B,H,W,3] = (raw/2 + 0.5).clip(0,1) (optional) */
/* VAE encoder pieces (reference ddpo/training/callbacks.py:37-57 `vae_fn`; 3P FlaxAutoencoderKL.encode):
 * images NHWC in [0,1] -> NCHW (x - 0.5) / 0.5 */
int ddpo_vae_image_to_nchw(const float* img_nhwc, float* out_nchw, int batch, int h, int w, void* stream);
/* 3x3 conv (pad 1) to 8 channels in fp32 (encoder conv_out: precision-critical, N = 8 is not tensor-core shaped),
 * then quant_conv (1x1, 8 -> 8) and the posterior's logvar clip to [-30, 20]: moments NHWC [batch, h, w, 8] = mean | logvar */
int ddpo_vae_encoder_head(const float* x_nhwc, const float* w_hwio, const float* bias, const float* wq_in_out,
                          const float* bq, float* moments_nhwc, int batch, int h, int w, int cin, void* stream);
/* decoded images [0,1] fp32 -> uint8 with the reference's truncating cast `(image * 255).astype(np.uint8)`
 * (ddpo/training/callbacks.py:181, ddpo/utils/hdf5.py:31), on the device so that the rewards' images leave as bytes */
int ddpo_image_to_uint8(const float* img, unsigned char* out, long long n, void* stream);
int ddpo_vae_conv_out(const float* x_nhwc, const float* w_hwio, const float* bias, float* raw_nchw, float* img_nhwc,
                      int batch, int h, int w, int cin, void* stream);

/* -------------------------------------------------------------- text encoder --------
 * CLIP text model the reference runs on the host CPU (pipeline/policy_gradient.py:185-187; inside the RWR step at
 * ddpo/training/diffusion.py:45-51,62-68; 3P transformers==4.28.1 FlaxCLIPTextModel).  Linears run on ddpo_igemm,
 * the causal self-attention on ddpo_attention_fwd (causal = 1), the pre-LayerNorms on ddpo_layernorm_fwd. */
/* out[m, :] = token_embedding[ids[m], :] + position_embedding[m % seq_len, :]  (fp32) */
int ddpo_embed_tokens(const int32_t* ids, const float* token_embedding, const float* position_embedding, float* out,
                      int rows, int seq_len, int dim, int vocab, void* stream);
/* y = act(x) as bf16; act 0 = gelu (erf form), 1 = quick_gelu (x * sigmoid(1.702 x)) */
int ddpo_act_bf16(const float* x, void* y_bf16, int64_t n, int act, void* stream);
/* LayerNorm with fp32 output (final_layer_norm: the conditioning tensor is fp32) */
int ddpo_layernorm_f32(const float* x, const float* scale, const float* bias, float* y, int m, int c, float eps,
                       void* stream);

/* ------------------------------------------------------------ aesthetic reward ------
 * CLIP ViT image tower + LAION aesthetic head (ddpo/training/callbacks.py:60-95, ddpo/models/laion.py:7-18; 3P transformers
 * FlaxCLIPModel.get_image_features).  Transformer layers run on the text tower's building blocks (non-causal attention,
 * quick_gelu); the small Dense layers of the head on ddpo_dense_small.  EXPERIMENTAL: written after the round's GPU
 * budget was spent, validated on the CPU only (oracle pinned against transformers, host assembly dry run). */
/* non-overlapping patches: out bf16 [batch*(size/patch)^2, ldk], column (ky*patch + kx)*3 + c, zero padded to ldk */
int ddpo_patchify_bf16(const float* img_nhwc, void* out_bf16, int batch, int size, int patch, int ldk, void* stream);
/* out[b, 0] = class_embedding + pos[0]; out[b, 1+p] = patches[b, p] + pos[1+p]   (fp32 [batch, n_patches+1, dim]) */
int ddpo_vit_tokens(const float* patches, const float* class_embedding, const float* position_embedding, float* out,
                    int batch, int n_patches, int dim, void* stream);
/* y[r] = x[r] / ||x[r]||_2 */
int ddpo_l2norm_rows(const float* x, float* y, int m, int c, void* stream);

/* ------------------------------------------------------------------ RWR ------------
 * Reward-weighted regression step around the U-Net (ddpo/training/diffusion.py:6-102).
 * ddpo_rwr_noisy_latents: latents = (mean + exp(0.5 clip(logvar,-30,20)) * normal(key_sample, NHWC shape)) * scaling
 * (3P FlaxDiagonalGaussianDistribution.sample, :16-23), noise = normal(key_noise, NCHW shape) (:27),
 * noisy = sqrt(a_t) latents + sqrt(1 - a_t) noise (3P add_noise_common, :36-41).
 *   moments_nhwc [B, h, w, 2*channels] fp32 (mean | logvar); outputs NCHW [B, channels, h, w]; latents_out optional.
 * ddpo_rwr_mse_loss: pred = e_u + g (e_c - e_u) (:77-79); per-sample mean squared error against `noise` (:83);
 * loss = mean over the batch, or sum_b weights[b] * mse_b when weights != NULL (:84-90); d_eps_* = dloss/d eps
 * (either may be NULL).  workspace: ddpo_rwr_workspace_floats(batch) floats, zero-initialised once. */
/* host: jax.random.randint(key, (n,), minval, maxval) int32 -- the per-sample training timesteps (:27-32) */
int ddpo_threefry_randint_host(const uint32_t key[2], int n, int32_t minval, int32_t maxval, int32_t* out);
int64_t ddpo_rwr_workspace_floats(int batch);
int ddpo_rwr_noisy_latents(const float* moments_nhwc, const uint32_t* key_sample_dev, const uint32_t* key_noise_dev,
                           const int32_t* timesteps /*[B]*/, const float* alphas_cumprod, float scaling, int batch,
                           int channels, int h, int w, float* noise_out, float* noisy_out, float* latents_out,
                           void* stream);
int ddpo_rwr_mse_loss(const float* eps_uncond, const float* eps_cond, const float* noise, const float* weights,
                      float guidance_scale, int batch, int n, float* loss_out /*[1]*/, float* per_sample_out /*[B] or NULL*/,
                      float* d_eps_uncond, float* d_eps_cond, float* workspace, void* stream);

/* ---------------------------------------------------------------- optimizer --------
 * optax.chain(clip_by_global_norm, adamw(mu_dtype=bf16)) + AccumulatingTrainState.apply_gradients(do_update=True)
 * (pipeline/policy_gradient.py:130-150, ddpo/training/policy_gradient.py:32-43). */
int64_t ddpo_optim_workspace_bytes(void);
int ddpo_grad_sumsq(const float* g, int64_t n, void* workspace, float* sumsq_out, void* stream);
int ddpo_clip_adamw(float* params, float* grad_acc, void* mu_bf16, float* nu, int64_t n, const float* sumsq_dev,
                    float grad_scale, float max_norm, float lr, float b1, float b2, float eps, float weight_decay,
                    int step, float* norm_out, void* stream);

/* optax.chain(clip_by_global_norm, adafactor(lr, weight_decay_rate=wd)) at optax's other defaults (momentum None,
 * decay_rate 0.8, eps 1e-30, clipping_threshold 1, multiply_by_parameter_scale) + the same apply_gradients
 * (pipeline/policy_gradient.py:132-150).
 * ddpo_adafactor_plan (host only, no device needed): tensor t has ndims[t] dims (taken in order from `dims`) and
 * starts at offsets[t] of the flat n-float buffer; offsets ascend and tensors do not overlap.  A tensor is factored as
 * optax decides (ndim >= 2 and second-largest dim >= min_dim_size_to_factor); its two largest dims must then be its
 * last two, its last dim a multiple of 4 and its offset a multiple of 4, else DDPO_ERR_INVALID.  sizes[3] receives the
 * plan's int64 words, the state floats and the workspace floats; tensor_info[ntensors][3] (may be NULL) receives per
 * tensor the kind (0 unfactored, 1 factored with v_row over the second-last dim, 2 factored with v_row over the last
 * dim) and the state offsets of v_row and v_col, or of v and -1.  State is optax's v_row, v_col / v, leaf by leaf, in
 * tensor order.  With plan == NULL only the sizes are computed.  On error nothing is written.
 * ddpo_clip_adafactor: plan_host and plan_dev are the same plan in host and device memory; params and grad_acc
 * 16-byte aligned; state zero-initialised before step 1; step = 1 + number of earlier updates.  The workspace starts
 * with [ntensors][2] floats: each tensor's clip denominator max(1, rms(u)) and parameter scale.  On an argument error
 * nothing is written. */
int ddpo_adafactor_plan(int ntensors, const int64_t* offsets, const int32_t* ndims, const int64_t* dims, int64_t n,
                        int min_dim_size_to_factor, int64_t* plan, int64_t plan_words, int64_t* sizes,
                        int64_t* tensor_info);
int ddpo_clip_adafactor(float* params, float* grad_acc, float* state, int64_t state_floats, int64_t n,
                        const int64_t* plan_host, const int64_t* plan_dev, float* workspace, int64_t workspace_floats,
                        const float* sumsq_dev, float grad_scale, float max_norm, float lr, float weight_decay, int step,
                        float* norm_out, void* stream);

/* ------------------------------------------------ image-symmetry / consistency rewards -----
 * Reference ddpo/training/callbacks.py:122-140 (consistency), 166-213 (rotational), 216-241 (rotational_corr),
 * 244-260 (mirror), 268-292 (mirror_corr), 295-344 (thumbnail).  Images are uint8 NHWC RGB [batch, h, w, 3].
 * Transforms, read in place by the first pass: ImageOps.mirror, and Pillow's rotate(90 / 180 / 270) fast paths
 * (transposes; 90 and 270 only for square images -- Pillow rotates other shapes through its affine path). */
enum { DDPO_IMAGE_IDENTITY = 0, DDPO_IMAGE_MIRROR = 1, DDPO_IMAGE_ROT90 = 2, DDPO_IMAGE_ROT180 = 3, DDPO_IMAGE_ROT270 = 4 };
/* One pass of Image.resize(BICUBIC, reducing_gap=None): axis 0 resamples the columns of the transformed image
 * (dst [batch, th, n_out, 3]), axis 1 its rows (dst [batch, n_out, tw, 3]); (th, tw) = (h, w), swapped for 90 / 270.
 * table [n_out][2 + ksize] int32 (xmin, n, then n of ksize 22-bit fixed-point weights), once in host and once in
 * device memory; every entry must lie inside the input.  acc = 2^21 + sum(pixel * k), dst = clamp(acc >> 22, 0, 255). */
int ddpo_resample_u8(const uint8_t* src, int batch, int h, int w, int transform, int axis, int n_out,
                     const int32_t* table_host, const int32_t* table_dev, int ksize, uint8_t* dst, void* stream);
/* out fp32 [batch, size, size, 3] = (double(float32(x) / 255) - CLIP mean) / CLIP std of the crop at (top, left) */
int ddpo_clip_normalize_u8(const uint8_t* src, int batch, int h, int w, int top, int left, int size, float* out,
                           void* stream);
/* out [batch][4]: sum(((a - T a) mod 256)^2 mod 256), sum a, sum a^2, sum a * T(a) over all h * w * 3 bytes of each
 * image; T is DDPO_IMAGE_MIRROR or DDPO_IMAGE_ROT180 */
int ddpo_pair_stats_u8(const uint8_t* src, int batch, int h, int w, int transform, uint64_t* out, void* stream);
/* feats fp32 [variants * n, dim] (row v * n + i: variant v of image i, variant 0 the original) -> out[n] fp32 = mean
 * over v >= 1 of degrees(arccos(clip(cos(f_0, f_v), 0, 1))), in double */
int ddpo_feature_angles(const float* feats, int variants, int n, int dim, float* out, void* stream);
/* out[i] = exp(logit_scale) * cos(img[i], txt[i]) for fp32 [n, dim] rows, in double */
int ddpo_scaled_cosine(const float* img, const float* txt, int n, int dim, float logit_scale, float* out, void* stream);

/* ------------------------------------------------------------------ low-rank adapters (LoRA) --------
 * diffusers' LoRALinearLayer in the Flax layout: y = x W + b + scale (x D) U with W fp32 [k, n], D fp32 [k, rank]
 * (down.weight^T) and U fp32 [rank, n] (up.weight^T).
 * lora_merge: bf16(W + scale D U), the rank-sum in fp32 and one rounding, into the forward operand layout of
 * ddpo_prep_weight (fwd_bf16 [.., ldk], row n + row_offset) and / or the dgrad layout of ddpo_prep_weight_dgrad with
 * taps = 1 (dgrad_bf16 [k, ld_dst], column col_offset + n) and / or the fp32 sum itself (merged_f32 [k, n]); any
 * output may be NULL.  ldk <= 0: k, ld_dst <= 0: n.
 * lora_grad: for g <= 3 adapters that share x bf16 [m, k] (row pitch ldx), with dy[i] bf16 [m, n] (row pitch lddy),
 * down[i] / up[i] fp32 as above:  d_up[i] += scale (x down[i])^T dy[i],  d_down[i] += scale x^T (dy[i] up[i]^T).
 * dy, down, up, d_down, d_up are host arrays of g device pointers.  rank is 4, 8 or 16; ldx, lddy multiples of 8 and
 * x / dy 16-byte aligned.  Deterministic (fixed-order two-stage reduction over m); the workspace (fp32, at least
 * ddpo_lora_grad_workspace_floats, which is -1 for an unsupported shape) holds one partial per CTA cluster. */
int ddpo_lora_merge(const float* w, int k, int n, const float* down, const float* up, int rank, float scale,
                    void* fwd_bf16, int ldk, int row_offset, void* dgrad_bf16, int ld_dst, int col_offset,
                    float* merged_f32, void* stream);
int64_t ddpo_lora_grad_workspace_floats(int rank, int g, int m, int k, int n);
int ddpo_lora_grad(const void* x, int ldx, const void* const* dy, int lddy, const float* const* down,
                   const float* const* up, float* const* d_down, float* const* d_up, int g, int m, int k, int n,
                   int rank, float scale, float* workspace, int64_t workspace_floats, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DDPO_B200_H_ */
