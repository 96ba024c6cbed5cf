/* rf_b200.h — C ABI of librf_b200.so: the H100-native (sm_90a) FLUX.1-dev DiT hot path of
 * Diffusion-CoT/ReflectionFlow.
 *
 * The reference has no FFI layer (it is pure Python over diffusers); its de-facto operator
 * boundaries are Python callables.  Each entry point below names the reference interface it
 * replaces (file:line under the reference tree).  Conventions:
 *   - all tensor arguments are DEVICE pointers to contiguous bf16 unless stated otherwise;
 *     token-major [tokens, channels] with an explicit row pitch in ELEMENTS where one is given
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); every call only
 *     enqueues work on it — no hidden synchronisation, no allocation of caller-visible memory
 *   - return value 0 = OK, negative = error; rf_last_error() returns a thread-local message
 *   - a handle (rf_dit*) is bound to the CUDA device current at rf_dit_create and is not
 *     thread-safe; weights are COPIED into handle-owned, kernel-friendly packed storage
 *   - there is no CPU fallback: without a CUDA device every compute call fails with an error
 */
#ifndef RF_B200_H_
#define RF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RF_B200_ABI_VERSION 2

/* error / version ------------------------------------------------------------------------- */
const char* rf_last_error(void);
int rf_abi_version(void);

/* ------------------------------------------------------------------------------------------
 * Operator level (what nn.Linear / SDPA / LayerNorm calls on the path dispatch to today).
 * These are the units the parity tests exercise one by one.
 * ---------------------------------------------------------------------------------------- */

/* epilogue kinds of rf_op_linear */
#define RF_EPI_BIAS 0     /* y = bf16(xW^T + b)                      nn.Linear                */
#define RF_EPI_GELU 1     /* y = bf16(gelu_tanh(bf16(xW^T + b)))     FeedForward net[0], act_mlp
                             (train_flux/flux/block.py:252,296)                               */
#define RF_EPI_GATE_RES 2 /* y = bf16(res + bf16(gate * bf16(xW^T+b)))  gated residual
                             (block.py:218-228,253-264,320-328)                               */
#define RF_EPI_QKV 3      /* fused to_q|to_k|to_v: per-head RMSNorm(q,k) * w, interleaved RoPE
                             (block.py:27-41,74-78,81-99)                                     */

/* y[M,N] = epilogue(x[M,K] @ W[N,K]^T).  Replaces torch.nn.Linear.forward at every call site of
 * train_flux/flux/block.py and transformer.py:92-93,115,244.  K % 64 == 0, N % 64 == 0.
 * addend (nullable): [M,N] bf16 added after the bias rounding (peft LoRA B(A(x)) term,
 * lora_controller.py:5-42).  RF_EPI_QKV: N = 3*heads*128, rope_cos/rope_sin are fp32 [M,64]
 * pair-compact tables (diffusers FluxPosEmbed values at even channels), norm_q/norm_k bf16 [128]. */
int rf_op_linear(int epilogue, int M, int N, int K, const void* x, int ldx, const void* W,
                 const void* bias, void* y, int ldy, const void* addend, int ld_addend,
                 const void* res, int ld_res, const void* gate, const float* rope_cos,
                 const float* rope_sin, const void* norm_q, const void* norm_k, void* stream);

/* rf_op_linear with peft's unfused LoRA arithmetic fused in (condition-token call sites under
 * enable_lora, train_flux/flux/lora_controller.py:5-42; targets train_flux/config.yaml:53):
 *   y = epilogue( bf16( bf16(x W^T + b) + bf16( bf16(x lora_A^T) lora_B^T ) ) )
 * lora_A: [t_cols, K] with t_cols = 64 (one target, rank zero-padded to 64) or 192 (stacked q|k|v A
 * factors, RF_EPI_QKV); lora_B: [N, 64] (rank zero-padded).  M >= 128, N % 128 == 0, K % 64 == 0;
 * epilogues GELU / GATE_RES / QKV.  workspace: rf_op_linear_lora_workspace_bytes(M) bytes of device
 * memory (the bf16 down-projection lives there).  The down-projection runs as one GEMM launch with one
 * CTA per 128 x 64-column output tile (8-24 CTAs at M = 1024), full K per tile; the product GEMM is one
 * launch whose tiles each carry one extra 64-deep k-block for the low-rank term. */
size_t rf_op_linear_lora_workspace_bytes(int M);
int rf_op_linear_lora(int epilogue, int M, int N, int K, const void* x, int ldx, const void* W,
                      const void* bias, void* y, int ldy, const void* lora_A, int t_cols,
                      const void* lora_B, const void* res, int ld_res, const void* gate,
                      const float* rope_cos, const float* rope_sin, const void* norm_q,
                      const void* norm_k, void* workspace, void* stream);

/* O = softmax(Q K^T / sqrt(128)) V, non-causal, head_dim 128, token-major operands
 * [batch*n_tok, heads*128] with row pitch ld_qkv / ld_out.  Replaces
 * F.scaled_dot_product_attention at train_flux/flux/block.py:123-125 (plus the cat/transpose
 * around it).  cond_mode: 0 = plain; 1 = additive bias `cond_bias` between tokens [0,n_main)
 * and [n_main,n_tok) (attn.c_factor, block.py:115-122); 2 = those cross blocks masked out
 * (union_cond_attn = False, block.py:106-114).  With cond_mode != 0, 0 < n_main < n_tok (any split).
 * cond_mode 1 with cond_bias = -inf (condition_scale 0: log 0) is computed as cond_mode 2, which it equals. */
int rf_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out,
                    int n_tok, int heads, int batch, int n_main, int cond_mode, float cond_bias,
                    void* stream);

/* out = LayerNorm(x; no affine, eps 1e-6) * (1 + scale) + shift with the reference's bf16
 * rounding after every op.  diffusers AdaLayerNormZero/ZeroSingle/Continuous body and
 * block.py:232-247.  dim % 256 == 0, dim <= 3072.  Row r uses scale/shift + (r / rows_per_batch)
 * * mod_stride. */
int rf_op_ln_modulate(const void* x, int ldx, void* out, int ld_out, int rows, int dim,
                      const void* scale, const void* shift, int rows_per_batch, int mod_stride,
                      void* stream);

/* y[b,n] = bf16(sum_k act(x[b,k]) W[n,k] + bias[n]); act 0 = identity, 1 = bf16(silu(x)).
 * The adaLN `linear(silu(temb))` of every block and the timestep/guidance/text embedder MLPs
 * (transformer.py:102-114).  K % 8 == 0, K <= 4096. */
int rf_op_gemv(const void* x, int ldx, int batch, const void* W, const void* bias, void* y, int ldy,
               int N, int K, int act, void* stream);

/* diffusers Timesteps(256, flip_sin_to_cos=True, shift 0) of bf16(t * pre_scale) -> bf16 [batch,256]
 * (transformer.py:95,98,102-114). */
int rf_op_timestep_embed(const void* t, float pre_scale, void* out, int batch, void* stream);

/* FlowMatchEulerDiscreteScheduler.step: x = bf16(float(x) + (sigmas[i+1]-sigmas[i]) * float(v))
 * (generate.py:276).  sigmas: device fp32; step: device int32 index i. */
int rf_op_euler_step(void* x, const void* v, const float* sigmas, const int* step, int n,
                     void* stream);

/* Pillow-compatible BICUBIC resize of a uint8 HWC image (Image.resize default filter): the
 * parent -> condition resize of tts/tts_reflectionflow.py:276-277.  Integer resampling tables
 * (bounds [out,2] = (first, count), coef [out, ksize], 22 fractional bits) come from the host
 * (reflectionflow_b200/resize.py::precompute_coeffs); tmp = uint8 [H, out_w, 3] scratch. */
int rf_op_resize_u8(const uint8_t* in_hwc, int H, int W, uint8_t* tmp, uint8_t* out_hwc, int out_h,
                    int out_w, const int* bounds_x, const int* coef_x, int ksize_x, const int* bounds_y,
                    const int* coef_y, int ksize_y, void* stream);

/* ------------------------------------------------------------------------------------------
 * Model level: the FLUX DiT forward and the denoise loop.
 * ---------------------------------------------------------------------------------------- */
typedef struct rf_dit rf_dit;

typedef struct rf_dit_config {
  int num_layers;          /* double-stream blocks (FLUX.1-dev: 19) */
  int num_single_layers;   /* single-stream blocks (38)             */
  int num_heads;           /* 24; head_dim is fixed at 128          */
  int in_channels;         /* 64                                    */
  int joint_attention_dim; /* 4096 (T5 width)                       */
  int pooled_projection_dim; /* 768 (CLIP pooled width)             */
  int guidance_embeds;     /* 1 for FLUX.1-dev                      */
  int lora_rank;           /* 0 = no LoRA storage; else max rank (<= 128) of the LoRA (cond tokens, + latent_lora).
                              Ranks <= 64 are stored zero-padded to 64, ranks 65..128 to 128 (one resp. two 64-deep
                              low-rank k-blocks per fused GEMM tile) */
} rf_dit_config;

int rf_dit_create(const rf_dit_config* cfg, rf_dit** out);
void rf_dit_destroy(rf_dit* h);

/* Copy one parameter into the handle.  `key` is the diffusers state-dict key of
 * FluxTransformer2DModel (e.g. "transformer_blocks.3.attn.to_q.weight"); src is a DEVICE
 * pointer to contiguous bf16 of `numel` elements.  Stands in for
 * DiffusionPipeline.from_pretrained(...).to("cuda") (tts/tts_reflectionflow.py:498-501). */
int rf_dit_load_weight(rf_dit* h, const char* key, const void* src, int64_t numel);

/* peft LoRA factors of one target Linear (pipe.load_lora_weights, tts_reflectionflow.py:503-505).  Any Linear of
 * FluxTransformer2DModel is a target (train/model.py:73-80 "all-linear"); other parameters (norm_q, biases, ...) are
 * refused.  module = diffusers module path without ".weight" (e.g. "single_transformer_blocks.0.proj_out");
 * A: [r, in_features] bf16, B: [out_features, r] bf16 (device); in_/out_features are checked against the target
 * Linear (a mismatched adapter file is an error, not an out-of-bounds read); r <= lora_rank; scale = that target's
 * lora_alpha / r, any finite value (NaN / inf are refused).  Setting a target again replaces its factors; targets
 * stay set until rf_dit_clear_lora.
 * Which rows carry the term follows lora_controller.py:5-42 (enable_lora zeroes the scaling of the modules it
 * names, inside its block only):
 *   x_embedder, and per block norm1.linear, attn.to_q/to_k/to_v, attn.to_out.0, ff.net.2 (double) and norm.linear,
 *   attn.to_q/to_k/to_v, proj_mlp, proj_out (single): the condition tokens (and cond_temb's modulation); with
 *   latent_lora (rf_dit_prepare) also the image stream of the double blocks, the txt + img rows of the single
 *   blocks and the image / main-row modulation of temb;
 *   context_embedder: the text rows, always;
 *   time_text_embed.{timestep,guidance,text}_embedder.linear_{1,2}: temb and cond_temb, always (every modulation
 *   vector downstream changes);
 *   norm_out.linear: the final modulation, always;  proj_out (top level): the image rows, always;
 *   per double block norm1_context.linear, attn.add_q_proj/add_k_proj/add_v_proj (before norm_added_q/k and RoPE),
 *   attn.to_add_out, ff_context.net.0.proj (before the GELU), ff_context.net.2: the text stream, always;
 *   per double block ff.net.0.proj (before the GELU): the image rows always and the condition rows.
 * The factors of the Linears outside train_flux/config.yaml:53 are allocated on their first rf_dit_set_lora.
 * Arithmetic (peft): y = bf16( bf16(x W^T + b) + bf16( bf16(T B^T) * s ) ), T = bf16(x A^T), with s the
 * target's effective scaling float(scale * call_scale) (product in double, as peft's `scaling *= scale`;
 * call_scale from rf_dit_set_lora_scale).  A target whose s is 0 adds nothing and runs no launch. */
int rf_dit_set_lora(rf_dit* h, const char* module, const void* A, const void* B, int r,
                    int in_features, int out_features, float scale);

/* Unset every LoRA target (diffusers' unload_lora_weights): the handle computes the adapter-free model until
 * rf_dit_set_lora is called again.  The factor storage stays allocated (zeroed); merged copies are re-made and the
 * captured denoise step is re-captured at the next call. */
int rf_dit_clear_lora(rf_dit* h);

/* The call-level LoRA multiplier (diffusers' joint_attention_kwargs["scale"], scale_lora_layers): every
 * target's scaling is multiplied by `scale` from the next rf_dit_forward / rf_dit_denoise on; 1 by default,
 * any finite value.  It stays until changed.  A denoise call whose scale differs from the one its captured
 * step was built with re-captures the step (one capture + instantiate); in merged mode (rf_dit_prepare flag
 * bit3) the merged weights are re-merged at the new scale (one pass over the LoRA target weights). */
int rf_dit_set_lora_scale(rf_dit* h, double scale);

/* Number of parameters still missing (0 = ready); names via rf_last_error(). */
int rf_dit_missing_weights(rf_dit* h);

/* Fix the problem geometry: token counts, position ids (bf16 [n,3], device), model_config flags.
 * Builds the RoPE tables once (the reference rebuilds them every step, transformer.py:130-134)
 * and sizes the workspace.  n_cond = 0 selects entry A (stock FluxTransformer2DModel.forward);
 * n_cond > 0 selects entry B (train_flux/flux/transformer.py:47 tranformer_forward).
 * flags: bit0 latent_lora (LoRA on the image and text tokens too; entry A included), bit1
 * add_cond_attn (not implemented: fails), bit2 union_cond_attn==False, bit3 = apply the LoRA as merged
 * weights W + B A for the LoRA'd tokens (peft fuse_lora semantics: one rounding of the merged weight
 * instead of three roundings of the low-rank path; no extra launches; adaLN terms stay unfused);
 * condition_scale != 1 enables the c_factor attention bias (generate.py:86-90). */
int rf_dit_prepare(rf_dit* h, int batch, int n_txt, int n_img, int n_cond, const void* txt_ids,
                   const void* img_ids, const void* cond_ids, int flags, float condition_scale,
                   void* stream);

/* One DiT forward == tranformer_forward(...)[0] / pipe.transformer(..., return_dict=False)[0].
 *   latents [B,n_img,64]; txt [B,n_txt,4096] (T5 states); pooled [B,768];
 *   timestep [B] bf16 (sigma, i.e. already / 1000 as generate.py:240 passes it);
 *   guidance [B] fp32 (nullable when guidance_embeds == 0); cond_latents [B,n_cond,64] nullable;
 *   out [B,n_img,64] bf16 noise prediction. */
int rf_dit_forward(rf_dit* h, const void* latents, const void* txt, const void* pooled,
                   const void* timestep, const float* guidance, const void* cond_latents,
                   void* out, void* stream);

/* The whole denoise loop of generate() / FluxPipeline.__call__ (generate.py:217-276):
 * n_steps x (forward + Euler step), latents updated in place.  timesteps: HOST bf16 [n_steps]
 * (the bf16(t)/1000 values the reference feeds), sigmas: HOST fp32 [n_steps+1].  The step body is
 * captured once into a CUDA graph and replayed. */
int rf_dit_denoise(rf_dit* h, void* latents_inout, const void* txt, const void* pooled,
                   const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps,
                   float guidance_scale, const void* cond_latents, void* stream);

/* ------------------------------------------------------------------------------------------
 * FLUX VAE decoder (next-tier row: `vae.decode` + `image_processor.postprocess`,
 * train_flux/flux/generate.py:302-307).
 * ---------------------------------------------------------------------------------------- */
typedef struct rf_vae rf_vae;
int rf_vae_create(rf_vae** out);
void rf_vae_destroy(rf_vae* h);
/* diffusers AutoencoderKL state-dict keys ("decoder.conv_in.weight", "encoder.down_blocks.0...",
 * torch conv layout [Cout, Cin, kh, kw]); src = device bf16.  decode needs the decoder.* keys,
 * encode the encoder.* keys. */
int rf_vae_load_weight(rf_vae* h, const char* key, const void* src, int64_t numel);
int rf_vae_missing_weights(rf_vae* h);
/* packed latents [(H/16)(W/16), 64] bf16 (one image) -> image.  Applies
 * `latents / scaling_factor + shift_factor` (bf16 ops), the decoder, and
 * VaeImageProcessor.postprocess: out_u8_hwc [H, W, 3] uint8 and/or out_bf16_chw [3, H, W] bf16
 * (either may be NULL).  height, width: multiples of 16 in [16, 16384]; the workspace (grown on demand, the
 * mid-block's (H/8 * W/8)^2 bf16 scores dominate it) must fit on the device. */
int rf_vae_decode(rf_vae* h, const void* packed_latents, int height, int width, float scaling_factor,
                  float shift_factor, uint8_t* out_u8_hwc, void* out_bf16_chw, void* stream);
/* encode_images() of train_flux/flux/pipeline_tools.py:7-30 (Condition.encode, condition.py:96-132):
 * image [H, W, 3] uint8 (or bf16 [3, H, W] already in [-1, 1]; exactly one non-NULL) ->
 * VaeImageProcessor.preprocess -> encoder -> posterior sample mean + std * eps with CALLER-PROVIDED
 * eps (bf16 [16, H/8, W/8]; NULL = posterior mode; the reference draws eps from the global RNG)
 * -> (z - shift) * scaling -> packed tokens [(H/16)(W/16), 64] bf16.  Sizes as for rf_vae_decode. */
int rf_vae_encode(rf_vae* h, const uint8_t* image_u8_hwc, const void* image_bf16_chw, int height,
                  int width, const void* eps_bf16_chw, float scaling_factor, float shift_factor,
                  void* packed_out, void* stream);

/* Per-kernel timing of everything launched between start and stop (CUDA events on the launching
 * stream around each launch; graph-captured launches are skipped).  rf_profile_stop synchronises
 * the device and writes a JSON object {kernel: {launches, ms, flops, bytes}} (algorithmic FLOPs /
 * HBM bytes as documented in DESIGN.md) into json_out. */
int rf_profile_start(void);
int rf_profile_stop(char* json_out, int capacity);

/* number of kernels this library launched since process start (for bench.py's gpu_launches) */
int64_t rf_launch_count(void);

/* ---- text encoders (T5 encoder + CLIP text model) --------------------------------------------
 * Replaces `pipe.text_encoder_2(ids)[0]` and `pipe.text_encoder(ids).pooler_output` inside diffusers
 * FluxPipeline.encode_prompt, called once per candidate prompt from train_flux/flux/generate.py:148-161
 * (via pipeline_tools.py:33-52); every reflection candidate carries its own refined prompt
 * (tts/tts_reflectionflow.py:286-294).  Token ids in (tokenisation stays on the host), embeddings out.
 * Rounding points follow the transformers "eager" attention path (T5Attention / CLIPAttention). */
typedef struct rf_text rf_text;
typedef struct rf_text_config {
  int t5_layers, t5_d_model, t5_d_ff, t5_heads, t5_vocab; /* T5-v1.1-XXL: 24, 4096, 10240, 64, 32128; d_kv = 64 */
  float t5_eps;                                           /* 1e-6 */
  int clip_layers, clip_d_model, clip_heads, clip_vocab, clip_max_pos; /* CLIP-L: 12, 768, 12, 49408, 77 */
} rf_text_config;

int rf_text_create(const rf_text_config* cfg, rf_text** out);
void rf_text_destroy(rf_text* h);
/* key = "t5." + T5EncoderModel state-dict key, or "clip." + CLIPTextModel state-dict key; src = device bf16 */
int rf_text_load_weight(rf_text* h, const char* key, const void* src, int64_t numel);
/* number of keys under `prefix` ("t5." / "clip.") not loaded yet (names in rf_last_error) */
int rf_text_missing_weights(rf_text* h, const char* prefix);
/* ids: device int32 [batch, seq]; position_bias: device bf16 [heads, seq, seq] (layer-0 relative
 * attention bias, shared by all layers; bucketed on the host); out: device bf16 [batch, seq, d_model] */
int rf_t5_encode(rf_text* h, const int* ids, int batch, int seq, const void* position_bias, void* out,
                 void* stream);
/* ids: device int32 [batch, seq <= 77]; eos_pos: device int32 [batch] (pooling position, = ids.argmax(-1)
 * for the stock CLIP-L config); pooled_out bf16 [batch, d_model]; hidden_out (nullable) bf16 [batch, seq, d_model] */
int rf_clip_encode(rf_text* h, const int* ids, const int* eos_pos, int batch, int seq, void* pooled_out,
                   void* hidden_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RF_B200_H_ */
