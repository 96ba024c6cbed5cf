// dit.cu — host orchestration of the FLUX.1-dev DiT forward and denoise loop (C ABI:
// rf_dit_* in include/rf_b200.h) over the sm_90a kernels of this directory.
//
// Mirrors, launch by launch, what the reference executes per step:
//   train_flux/flux/transformer.py:47-252 (tranformer_forward; with n_cond == 0 the stock
//   diffusers FluxTransformer2DModel.forward), train_flux/flux/block.py:173-333 (block_forward,
//   single_block_forward, attn_forward), train_flux/flux/generate.py:217-276 (denoise loop),
//   train_flux/flux/lora_controller.py:5-42 (LoRA on condition tokens only; with latent_lora on every token
//   that passes a target Linear).
//
// HBM layout (token-major, one joint buffer per quantity; rows = [txt | img | cond]):
//   X   [N, D]      hidden state (residual stream), updated in place by the GEMM epilogues
//   XN  [N, D]      LayerNorm+modulate output = A operand of the projections
//   QKV [N, 3D]     q | k | v after bias, RMSNorm, RoPE (written by the QKV GEMM epilogue)
//   ACT [N, 5D]     double blocks: O (cols 0..D) and MLP hidden (cols D..5D);
//                   single blocks: cat(attn, gelu(mlp)) = A operand of proj_out (K = 5D)
//   MOD [n_mod]     all adaLN modulation vectors of the step (one GEMV), MODC same for cond_temb
// torch.cat / split / transpose of the reference never materialise: streams are row ranges.
#include <algorithm>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/rf_b200.h"
#include "rf_internal.h"

namespace rf {
int add2_launch(const bf16* a, const bf16* b, bf16* out, int n, cudaStream_t stream);
int select_row_launch(const bf16* table, int64_t row_elems, const int* row, bf16* out,
                      cudaStream_t stream);
int f32_to_bf16_launch(const float* src, bf16* dst, int n, cudaStream_t stream);
int gemm_init();
int attention_init();
int gemv_init();
}

using rf::bf16;

namespace {

struct Lin {  // a Linear's weights, or views into a packed one
  bf16* w = nullptr;
  bf16* b = nullptr;
};

struct LoraPack;
struct LoraT {  // one target Linear of an adapter
  int in = 0, out = 0;
  bool set = false;
  double scale = 1.0;  // lora_alpha / r
  LoraPack* pack = nullptr;
  int slot = 0;  // its factors are slot `slot` of the pack's stacked A / B
};

// The adapter of one packed weight: 1 target, or the 3 stacked q|k|v ones, with factors zero-padded to the handle's
// lora_pad.  The Linears of train_flux/config.yaml:53 are gated by enable_lora / latent_lora; the others (text
// stream, embedders, final layer, ff.net.0.proj) are "always" packs: no enable_lora block names them, so they apply
// to every row that reads their weight.  Factors of the gated packs are allocated at create, those of the always
// packs on their first rf_dit_set_lora (lora_storage), so a handle that never sees such an adapter keeps its footprint.
struct LoraPack {
  LoraT t[3];
  int n = 0;
  bool always = false;
  bf16* A = nullptr;        // [n lora_pad, in]
  bf16* B = nullptr;        // [n out, lora_pad] (rows of the packed projection)
  const bf16* W = nullptr;  // base weight [n out, in] of a projection (nullptr: a GEMV target, never merged)
  bf16* Wm = nullptr;       // merged W + s B A (fuse_lora mode), allocated on the first merge with a target set
};
bf16* lora_A(const LoraT& t, int pad) { return t.pack->A + static_cast<int64_t>(t.slot) * pad * t.in; }
bf16* lora_B(const LoraT& t, int pad) { return t.pack->B + static_cast<int64_t>(t.slot) * t.out * pad; }

struct DoubleBlk {
  Lin qkv, add_qkv, to_out, to_add_out, ff1, ff2, ffc1, ffc2;
  bf16 *norm_q, *norm_k, *norm_added_q, *norm_added_k;
  LoraPack l_norm1, l_qkv, l_out, l_ff2;
  // always: text stream (norm1_context, add_q|k|v, to_add_out, ff_context) and ff.net.0.proj
  LoraPack l_norm1c, l_add_qkv, l_add_out, l_ff1, l_ffc1, l_ffc2;
};
struct SingleBlk {
  Lin qkv, mlp, out;
  bf16 *norm_q, *norm_k;
  LoraPack l_norm, l_qkv, l_mlp, l_out;
};

}  // namespace

// one denoise step captured into a CUDA graph
struct StepGraph {
  cudaGraphExec_t exec = nullptr;
  int64_t kernels = 0;      // kernel launches inside the step
  double call_scale = 1.0;  // call_scale the step was built with (kernel parameters, launch list)
};

struct rf_dit {
  rf_dit_config cfg;
  int D = 0;
  int device = 0;
  // ---- weights
  rf::DeviceAllocs mem;      // weights, LoRA factors, merged copies: live until destroy
  rf::DeviceAllocs geo_mem;  // workspace of the current geometry: freed on re-prepare
  rf::WeightTable weights;
  std::unordered_map<std::string, LoraT*> lora_slots;
  Lin x_emb, ctx_emb, t1, t2, g1, g2, p1, p2, proj_out;
  LoraPack l_x_emb;
  // always packs at the top level: context_embedder, the time / guidance / text embedders, norm_out, proj_out
  LoraPack l_ctx, l_t1, l_t2, l_g1, l_g2, l_p1, l_p2, l_norm_out, l_proj_out;
  std::vector<LoraPack*> proj_packs;  // the packs of every projection (merge_all)
  bf16* modW = nullptr;
  bf16* modB = nullptr;
  int64_t n_mod = 0;
  std::vector<DoubleBlk> dbl;
  std::vector<SingleBlk> sgl;
  bool any_lora = false;
  bool any_always = false;  // some always target is set: its rows carry a LoRA whatever the flags
  // LoRA rank padding: 64 for lora_rank <= 64, else 128 (one or two 64-deep low-rank k-blocks per fused tile)
  int lora_pad = 64;
  // rf_dit_set_lora_scale: peft's call-level multiplier (joint_attention_kwargs["scale"]); a target's effective
  // scaling is float(scale * call_scale), formed in double like peft's `scaling *= scale`
  double call_scale = 1.0;
  bool lora_merged = false;   // merged copies are current for merged_call_scale
  double merged_call_scale = 1.0;
  bool use_merged = false;    // rf_dit_prepare flag bit 3
  // ---- geometry
  bool prepared = false;
  int batch = 0, n_txt = 0, n_img = 0, n_cond = 0, N = 0, n_main = 0;
  int flags = 0;
  int attn_cond_mode = 0;
  float attn_cond_bias = 0.f;
  float *rope_cos = nullptr, *rope_sin = nullptr, *crope_cos = nullptr, *crope_sin = nullptr;
  // ---- workspace
  bf16 *X = nullptr, *XN = nullptr, *QKV = nullptr, *ACT = nullptr, *MOD = nullptr, *MODC = nullptr;
  bf16 *LT = nullptr, *LL = nullptr;  // LoRA temporaries: T [lora_rows, 4 lora_pad], L [lora_rows, 4D]
  int lora_rows = 0;
  bf16* emb_ws = nullptr;             // temb_mod workspace of one vector (eager step, cond_temb)
  // ---- the denoise loop (rf_dit_denoise, rf_dit_denoise_image_guidance, rf_dit_denoise_begin / _step)
  // Staging of the captured step, one sample: before each replay the loop copies a sample's inputs here, and the
  // step's sigma index into s_step and its table row into s_row.
  bf16 *s_lat = nullptr, *s_txt = nullptr, *s_cond = nullptr, *s_v = nullptr;
  bf16 *s_tsteps = nullptr, *s_guid = nullptr, *s_zero_one = nullptr;
  float* s_sigmas = nullptr;
  int *s_step = nullptr, *s_row = nullptr;
  // image guidance: the uncond branch's condition input U_i and noise prediction, and the scale s (device fp32)
  bf16 *s_ucond = nullptr, *s_vu = nullptr;
  float* s_igs = nullptr;
  // The tables of the open loop, built when it opens (all timesteps are known up front): every sample's adaLN
  // modulation vectors of every step, tab [B n_steps, n_mod] (row b n_steps + i), with image guidance also the
  // uncond branch's tab_u at guidance bf16(1); every sample's cond_temb vectors tab_c [B, n_mod] and condition
  // latents loop_cond [B, n_cond, C]; idx = 0, 1, ..., B tab_steps - 1, the source of s_step and s_row.
  // s_tsteps, s_sigmas, tab, tab_u, temb_ws and idx hold tab_steps steps and grow with n_steps.
  bf16 *tab = nullptr, *tab_u = nullptr, *tab_c = nullptr, *loop_cond = nullptr, *temb_ws = nullptr;
  int* idx = nullptr;
  int tab_steps = 0;
  StepGraph graph, graph_ig;  // the captured step of the plain / of the image-guided loop
  rf::SideStream side;        // the denoise loop's stream
  // The open loop's step count and kind.  sess: rf_dit_denoise_begin opened it; everything that drops the captured
  // step or changes what the tables were built from closes it.
  bool sess = false, sess_guided = false;
  int sess_steps = 0;
};

namespace {

// the fp32 scaling peft multiplies the bf16 low-rank term of target t by
float lora_eff(const rf_dit* h, const LoraT& t) { return static_cast<float>(t.scale * h->call_scale); }
// a target whose effective scaling is 0 adds exactly nothing: it runs no launch at all
bool lora_on(const rf_dit* h, const LoraT& t) { return t.set && lora_eff(h, t) != 0.f; }

// Linear whose weight/bias may be a row range of a packed matrix
void reg_lin(rf_dit* h, const std::string& mod, bf16* w, bf16* b, int out, int in) {
  h->weights.add(mod + ".weight", w, static_cast<int64_t>(out) * in);
  h->weights.add(mod + ".bias", b, out);
}

// a Linear's own storage, registered under `mod` (empty: a packed one whose row ranges the caller registers)
int new_lin(rf_dit* h, Lin& l, const std::string& mod, int out, int in) {
  RF_TRY(h->mem.alloc(&l.w, static_cast<size_t>(out) * in));
  RF_TRY(h->mem.alloc(&l.b, out));
  if (!mod.empty()) reg_lin(h, mod, l.w, l.b, out, in);
  return 0;
}

// a weight vector's own storage, registered under `key`
int new_vec(rf_dit* h, bf16** v, const std::string& key, int n) {
  RF_TRY(h->mem.alloc(v, n));
  h->weights.add(key, *v, n);
  return 0;
}

// Zeroed factor storage of pack p, live until destroy: unset members must add exactly nothing (a q-only adapter
// still runs the stacked q|k|v path).  A preset A is a view into a larger stack and is only zeroed.
int lora_storage(rf_dit* h, LoraPack& p) {
  if (p.B != nullptr) return 0;
  const size_t a = static_cast<size_t>(p.n) * h->lora_pad * p.t[0].in;
  const size_t b = static_cast<size_t>(p.n) * p.t[0].out * h->lora_pad;
  if (p.A == nullptr) RF_TRY(h->mem.alloc(&p.A, a));
  RF_TRY(h->mem.alloc(&p.B, b));
  RF_CHECK_CUDA(cudaMemset(p.A, 0, a * 2));
  RF_CHECK_CUDA(cudaMemset(p.B, 0, b * 2));
  return 0;
}

// the pack of the targets `mods`, each out x in and stacked in that order; W: the packed projection weight
int new_pack(rf_dit* h, LoraPack& p, std::initializer_list<std::string> mods, int out, int in, const bf16* W,
             bool always) {
  if (h->cfg.lora_rank <= 0) return 0;
  for (const std::string& m : mods) {
    p.t[p.n] = LoraT{in, out, false, 1.0, &p, p.n};
    h->lora_slots[m] = &p.t[p.n++];
  }
  p.always = always;
  p.W = W;
  if (W) h->proj_packs.push_back(&p);
  return always ? 0 : lora_storage(h, p);
}

int build_storage(rf_dit* h) {
  const rf_dit_config& c = h->cfg;
  const int D = h->D, lpad = h->lora_pad;
  RF_TRY(new_lin(h, h->x_emb, "x_embedder", D, c.in_channels));
  RF_TRY(new_pack(h, h->l_x_emb, {"x_embedder"}, D, c.in_channels, h->x_emb.w, false));
  RF_TRY(new_lin(h, h->ctx_emb, "context_embedder", D, c.joint_attention_dim));
  RF_TRY(new_pack(h, h->l_ctx, {"context_embedder"}, D, c.joint_attention_dim, h->ctx_emb.w, true));
  const std::string tte = "time_text_embed.";
  RF_TRY(new_lin(h, h->t1, tte + "timestep_embedder.linear_1", D, 256));
  RF_TRY(new_lin(h, h->t2, tte + "timestep_embedder.linear_2", D, D));
  RF_TRY(new_pack(h, h->l_t1, {tte + "timestep_embedder.linear_1"}, D, 256, nullptr, true));
  RF_TRY(new_pack(h, h->l_t2, {tte + "timestep_embedder.linear_2"}, D, D, nullptr, true));
  if (c.guidance_embeds) {
    RF_TRY(new_lin(h, h->g1, tte + "guidance_embedder.linear_1", D, 256));
    RF_TRY(new_lin(h, h->g2, tte + "guidance_embedder.linear_2", D, D));
    RF_TRY(new_pack(h, h->l_g1, {tte + "guidance_embedder.linear_1"}, D, 256, nullptr, true));
    RF_TRY(new_pack(h, h->l_g2, {tte + "guidance_embedder.linear_2"}, D, D, nullptr, true));
  }
  RF_TRY(new_lin(h, h->p1, tte + "text_embedder.linear_1", D, c.pooled_projection_dim));
  RF_TRY(new_lin(h, h->p2, tte + "text_embedder.linear_2", D, D));
  RF_TRY(new_pack(h, h->l_p1, {tte + "text_embedder.linear_1"}, D, c.pooled_projection_dim, nullptr, true));
  RF_TRY(new_pack(h, h->l_p2, {tte + "text_embedder.linear_2"}, D, D, nullptr, true));
  RF_TRY(new_lin(h, h->proj_out, "proj_out", c.in_channels, D));
  RF_TRY(new_pack(h, h->l_proj_out, {"proj_out"}, c.in_channels, D, h->proj_out.w, true));

  h->n_mod = static_cast<int64_t>(c.num_layers) * 12 * D +
             static_cast<int64_t>(c.num_single_layers) * 3 * D + 2 * D;
  RF_TRY(h->mem.alloc(&h->modW, static_cast<size_t>(h->n_mod) * D));
  RF_TRY(h->mem.alloc(&h->modB, h->n_mod));

  h->dbl.resize(c.num_layers);
  for (int i = 0; i < c.num_layers; ++i) {
    DoubleBlk& b = h->dbl[i];
    const std::string p = "transformer_blocks." + std::to_string(i) + ".";
    const int64_t mo = static_cast<int64_t>(i) * 12 * D;
    reg_lin(h, p + "norm1.linear", h->modW + mo * D, h->modB + mo, 6 * D, D);
    reg_lin(h, p + "norm1_context.linear", h->modW + (mo + 6 * D) * D, h->modB + mo + 6 * D, 6 * D, D);
    RF_TRY(new_pack(h, b.l_norm1, {p + "norm1.linear"}, 6 * D, D, nullptr, false));
    RF_TRY(new_pack(h, b.l_norm1c, {p + "norm1_context.linear"}, 6 * D, D, nullptr, true));
    RF_TRY(new_lin(h, b.qkv, "", 3 * D, D));
    RF_TRY(new_lin(h, b.add_qkv, "", 3 * D, D));
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    const char* an[3] = {"add_q_proj", "add_k_proj", "add_v_proj"};
    for (int j = 0; j < 3; ++j) {
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
      reg_lin(h, p + "attn." + an[j], b.add_qkv.w + static_cast<int64_t>(j) * D * D,
              b.add_qkv.b + j * D, D, D);
    }
    RF_TRY(new_pack(h, b.l_qkv, {p + "attn.to_q", p + "attn.to_k", p + "attn.to_v"}, D, D, b.qkv.w, false));
    RF_TRY(new_pack(h, b.l_add_qkv, {p + "attn.add_q_proj", p + "attn.add_k_proj", p + "attn.add_v_proj"}, D, D,
                    b.add_qkv.w, true));
    RF_TRY(new_vec(h, &b.norm_q, p + "attn.norm_q.weight", 128));
    RF_TRY(new_vec(h, &b.norm_k, p + "attn.norm_k.weight", 128));
    RF_TRY(new_vec(h, &b.norm_added_q, p + "attn.norm_added_q.weight", 128));
    RF_TRY(new_vec(h, &b.norm_added_k, p + "attn.norm_added_k.weight", 128));
    RF_TRY(new_lin(h, b.to_out, p + "attn.to_out.0", D, D));
    RF_TRY(new_pack(h, b.l_out, {p + "attn.to_out.0"}, D, D, b.to_out.w, false));
    RF_TRY(new_lin(h, b.to_add_out, p + "attn.to_add_out", D, D));
    RF_TRY(new_pack(h, b.l_add_out, {p + "attn.to_add_out"}, D, D, b.to_add_out.w, true));
    RF_TRY(new_lin(h, b.ff1, p + "ff.net.0.proj", 4 * D, D));
    RF_TRY(new_pack(h, b.l_ff1, {p + "ff.net.0.proj"}, 4 * D, D, b.ff1.w, true));
    RF_TRY(new_lin(h, b.ff2, p + "ff.net.2", D, 4 * D));
    RF_TRY(new_pack(h, b.l_ff2, {p + "ff.net.2"}, D, 4 * D, b.ff2.w, false));
    RF_TRY(new_lin(h, b.ffc1, p + "ff_context.net.0.proj", 4 * D, D));
    RF_TRY(new_lin(h, b.ffc2, p + "ff_context.net.2", D, 4 * D));
    RF_TRY(new_pack(h, b.l_ffc1, {p + "ff_context.net.0.proj"}, 4 * D, D, b.ffc1.w, true));
    RF_TRY(new_pack(h, b.l_ffc2, {p + "ff_context.net.2"}, D, 4 * D, b.ffc2.w, true));
  }
  h->sgl.resize(c.num_single_layers);
  const int64_t so = static_cast<int64_t>(c.num_layers) * 12 * D;
  for (int i = 0; i < c.num_single_layers; ++i) {
    SingleBlk& b = h->sgl[i];
    const std::string p = "single_transformer_blocks." + std::to_string(i) + ".";
    const int64_t mo = so + static_cast<int64_t>(i) * 3 * D;
    reg_lin(h, p + "norm.linear", h->modW + mo * D, h->modB + mo, 3 * D, D);
    RF_TRY(new_pack(h, b.l_norm, {p + "norm.linear"}, 3 * D, D, nullptr, false));
    RF_TRY(new_lin(h, b.qkv, "", 3 * D, D));
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    for (int j = 0; j < 3; ++j)
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
    RF_TRY(new_lin(h, b.mlp, p + "proj_mlp", 4 * D, D));
    if (c.lora_rank > 0) {
      // A factors of to_q | to_k | to_v | proj_mlp stacked: all four read the same normalised tokens, so
      // ONE down-projection launch (NT = 4 lora_pad) serves the q|k|v and the MLP-in GEMMs of the block
      RF_TRY(h->mem.alloc(&b.l_qkv.A, static_cast<size_t>(4 * lpad) * D));
      b.l_mlp.A = b.l_qkv.A + static_cast<int64_t>(3 * lpad) * D;
    }
    RF_TRY(new_pack(h, b.l_qkv, {p + "attn.to_q", p + "attn.to_k", p + "attn.to_v"}, D, D, b.qkv.w, false));
    RF_TRY(new_pack(h, b.l_mlp, {p + "proj_mlp"}, 4 * D, D, b.mlp.w, false));
    RF_TRY(new_vec(h, &b.norm_q, p + "attn.norm_q.weight", 128));
    RF_TRY(new_vec(h, &b.norm_k, p + "attn.norm_k.weight", 128));
    RF_TRY(new_lin(h, b.out, p + "proj_out", D, 5 * D));
    RF_TRY(new_pack(h, b.l_out, {p + "proj_out"}, D, 5 * D, b.out.w, false));
  }
  const int64_t oo = so + static_cast<int64_t>(c.num_single_layers) * 3 * D;
  reg_lin(h, "norm_out.linear", h->modW + oo * D, h->modB + oo, 2 * D, D);
  return new_pack(h, h->l_norm_out, {"norm_out.linear"}, 2 * D, D, nullptr, true);
}

// modulation vector offsets inside MOD / MODC
inline int64_t mod_double(const rf_dit* h, int i, int stream_ctx, int which) {
  return static_cast<int64_t>(i) * 12 * h->D + (stream_ctx ? 6 * h->D : 0) +
         static_cast<int64_t>(which) * h->D;
}
inline int64_t mod_single(const rf_dit* h, int i, int which) {
  return static_cast<int64_t>(h->cfg.num_layers) * 12 * h->D + static_cast<int64_t>(i) * 3 * h->D +
         static_cast<int64_t>(which) * h->D;
}
inline int64_t mod_out(const rf_dit* h, int which) {
  return static_cast<int64_t>(h->cfg.num_layers) * 12 * h->D +
         static_cast<int64_t>(h->cfg.num_single_layers) * 3 * h->D + static_cast<int64_t>(which) * h->D;
}
enum { SHIFT_MSA = 0, SCALE_MSA = 1, GATE_MSA = 2, SHIFT_MLP = 3, SCALE_MLP = 4, GATE_MLP = 5 };

// The low-rank term of a Linear that runs as a GEMV (embedders, adaLN), for `batch` vectors:
// y[b] = bf16(y[b] + bf16(bf16(bf16(act(x_b) A^T) B^T) * scaling)) (peft), act = silu when act = 1, as in the GEMV of
// the Linear itself.  Two batched GEMVs and one strided add; tvec [batch, lora_pad], lvec [batch, t.out] scratch.
int add_vec_lora(rf_dit* h, const LoraT& t, const bf16* x, int ldx, int batch, int act, bf16* y, int64_t ldy,
                 bf16* tvec, bf16* lvec, cudaStream_t s) {
  if (!lora_on(h, t)) return 0;
  const int lpad = h->lora_pad;
  RF_TRY(rf::gemv_launch(x, ldx, batch, lora_A(t, lpad), nullptr, tvec, lpad, lpad, t.in, act, s));
  RF_TRY(rf::gemv_launch(tvec, lpad, batch, lora_B(t, lpad), nullptr, lvec, t.out, t.out, lpad, 0, s));
  return rf::add_rows_launch(y, ldy, lvec, t.out, batch, t.out, lora_eff(h, t), s);
}

// y = linear_2(silu(linear_1(x)))  (TimestepEmbedding / PixArtAlphaTextProjection) for `batch` vectors, each Linear
// with its LoRA term (always targets): linear_2's sees the same bf16(silu(.)) input as its GEMV.
// tvec [batch, lora_pad], lvec [batch, D] scratch.
int mlp2(rf_dit* h, const bf16* x, int in_dim, int batch, const Lin& l1, const LoraPack& lp1, const Lin& l2,
         const LoraPack& lp2, bf16* tmp, bf16* out, bf16* tvec, bf16* lvec, cudaStream_t s) {
  const int D = h->D;
  RF_TRY(rf::gemv_launch(x, in_dim, batch, l1.w, l1.b, tmp, D, D, in_dim, 0, s));
  RF_TRY(add_vec_lora(h, lp1.t[0], x, in_dim, batch, 0, tmp, D, tvec, lvec, s));
  RF_TRY(rf::gemv_launch(tmp, D, batch, l2.w, l2.b, out, D, D, D, 1, s));
  return add_vec_lora(h, lp2.t[0], tmp, D, batch, 1, out, D, tvec, lvec, s);
}

// L[rows, :] = bf16( bf16(x A^T) B^T ): the unfused peft low-rank term of `rows` tokens for pack p (n = 1 target, or
// the n = 3 stacked q|k|v targets: T = x A^T in one GEMM, L[:, jD:(j+1)D] = T_j B_j^T grouped).  T != nullptr:
// bf16(x A^T) of these rows was already computed (pitch ld_t); only the up-projection runs.  Otherwise T is computed
// here into LT.
int lora_term(rf_dit* h, const LoraPack& p, const bf16* x, int ldx, int rows, const bf16* T, int ld_t, bf16* L,
              int ldl, cudaStream_t s) {
  const int lpad = h->lora_pad;
  rf::GemmGroupArgs g[3];
  if (T == nullptr) {
    memset(g, 0, sizeof(g));
    g[0].A = x; g[0].lda = ldx; g[0].M = rows; g[0].W = p.A; g[0].out = h->LT; g[0].ldo = p.n * lpad;
    RF_TRY(rf::gemm_launch(rf::EPI_BIAS, p.n * lpad, p.t[0].in, 1, g, s));
    T = h->LT;
    ld_t = p.n * lpad;
  }
  memset(g, 0, sizeof(g));
  bool scaled = false;  // peft's bf16(bf16(T B^T) * scaling): the scale is the up-projection's output scale
  for (int j = 0; j < p.n; ++j) {
    const LoraT& t = p.t[j];
    g[j].A = T + j * lpad; g[j].lda = ld_t; g[j].M = rows;
    g[j].W = lora_B(t, lpad); g[j].out = L + static_cast<int64_t>(j) * t.out; g[j].ldo = ldl;
    g[j].lora_scale[0] = lora_eff(h, t);
    scaled |= g[j].lora_scale[0] != 1.f;
  }
  return rf::gemm_launch(scaled ? rf::EPI_SCALE : rf::EPI_BIAS, p.t[0].out, lpad, p.n, g, s);
}

// The low-rank term of the adaLN Linears added to their sections of `batch` modulation rows:
// mod[b * ld_mod + section] += bf16(bf16(bf16(silu(emb_b) A^T) B^T) * scaling) (peft: bf16(y + L)).  `gated`: the
// targets enable_lora names (norm1.linear of the double blocks, norm.linear of the single blocks); `always`: the
// text-stream norm1_context.linear and norm_out.linear, which no enable_lora names.
// M = batch is tiny: two batched GEMVs and one strided add per target.
// tvec: [batch, lora_pad], lvec: [batch, 6D] scratch.
int add_mod_lora(rf_dit* h, const bf16* emb, int batch, bool gated, bool always, bf16* mod, int64_t ld_mod,
                 bf16* tvec, bf16* lvec, cudaStream_t s) {
  const int D = h->D;
  auto one = [&](const LoraPack& p, int64_t off) {
    return add_vec_lora(h, p.t[0], emb, D, batch, 1, mod + off, ld_mod, tvec, lvec, s);
  };
  if (gated) {
    for (int i = 0; i < h->cfg.num_layers; ++i) RF_TRY(one(h->dbl[i].l_norm1, mod_double(h, i, 0, 0)));
    for (int i = 0; i < h->cfg.num_single_layers; ++i) RF_TRY(one(h->sgl[i].l_norm, mod_single(h, i, 0)));
  }
  if (always && h->any_always) {
    for (int i = 0; i < h->cfg.num_layers; ++i) RF_TRY(one(h->dbl[i].l_norm1c, mod_double(h, i, 1, 0)));
    RF_TRY(one(h->l_norm_out, mod_out(h, 0)));
  }
  return 0;
}

// elements of the temb_mod workspace for n vectors
int64_t temb_ws_elems(const rf_dit* h, int n) {
  return static_cast<int64_t>(n) * (256 + 9 * h->D + h->lora_pad) + 256 + 3 * h->D;
}

// temb_i = time(t_i) + guidance(g) + text(pooled) (CombinedTimestepGuidanceTextProjEmbeddings) for n timesteps, then
// every adaLN Linear of every block on silu(temb_i) into mod [n, n_mod], with the adaLN LoRA terms of add_mod_lora.
// The eager step and cond_temb take n = 1; the denoise loop takes every step at once, so the 6.5 GB modulation weight
// stack is streamed ceil(n/8) times per call instead of once per step.  Same kernels and per-vector arithmetic for
// any n (the GEMV's per-vector summation order does not depend on the batch width): bit-identical rows.
int temb_mod(rf_dit* h, int n, const bf16* t, const bf16* guid, const bf16* pooled, bool gated, bool always,
             bf16* mod, bf16* ws, cudaStream_t s) {
  const int D = h->D;
  // [n,256] | [n,D] tmp | [n,D] a | [n,D] temb | [256] gp | [D] tmp1 | [D] b | [D] c | [n,lora_pad] | [n,6D] (LoRA)
  bf16* tp = ws;
  bf16* tmp = tp + static_cast<int64_t>(n) * 256;
  bf16* a = tmp + static_cast<int64_t>(n) * D;
  bf16* temb = a + static_cast<int64_t>(n) * D;
  bf16* gp = temb + static_cast<int64_t>(n) * D;
  bf16 *tmp1 = gp + 256, *b = tmp1 + D, *c = b + D;
  bf16* tvec = c + D;                                         // [n, lora_pad]
  bf16* lvec = tvec + static_cast<int64_t>(n) * h->lora_pad;  // [n, 6D]
  RF_TRY(rf::timestep_embed_launch(t, nullptr, 1, 1000.0f, tp, n, s));
  RF_TRY(mlp2(h, tp, 256, n, h->t1, h->l_t1, h->t2, h->l_t2, tmp, a, tvec, lvec, s));
  RF_TRY(mlp2(h, pooled, h->cfg.pooled_projection_dim, 1, h->p1, h->l_p1, h->p2, h->l_p2, tmp1, c, tvec, lvec, s));
  if (h->cfg.guidance_embeds) {
    RF_TRY(rf::timestep_embed_launch(guid, nullptr, 1, 1000.0f, gp, 1, s));
    RF_TRY(mlp2(h, gp, 256, 1, h->g1, h->l_g1, h->g2, h->l_g2, tmp1, b, tvec, lvec, s));
  }
  for (int i = 0; i < n; ++i) {
    bf16* ai = a + static_cast<int64_t>(i) * D;
    bf16* ti = temb + static_cast<int64_t>(i) * D;
    if (h->cfg.guidance_embeds) RF_TRY(rf::add3_launch(ai, b, c, ti, D, s));
    else RF_TRY(rf::add2_launch(ai, c, ti, D, s));
  }
  RF_TRY(rf::gemv_launch(temb, D, n, h->modW, h->modB, mod, static_cast<int>(h->n_mod), static_cast<int>(h->n_mod),
                         D, 1, s));
  if (h->any_lora) RF_TRY(add_mod_lora(h, temb, n, gated, always, mod, h->n_mod, tvec, lvec, s));
  return 0;
}

// cond_temb and MODC: step-invariant (transformer.py:108-114 recomputes them every step).  t = c_t * 1000 = 0,
// guidance = 1000 (s_zero_one = {bf16 0, bf16 1}); the condition rows read no norm1_context / norm_out section of MODC.
int compute_cond_mod(rf_dit* h, const bf16* pooled, cudaStream_t s, bf16* out = nullptr) {
  return temb_mod(h, 1, h->s_zero_one, h->s_zero_one + 1, pooled, true, false, out ? out : h->MODC, h->emb_ws, s);
}

// some member of pack p adds a term (lora_on) / is set
bool pack_on(const rf_dit* h, const LoraPack& p) {
  for (int k = 0; k < p.n; ++k)
    if (lora_on(h, p.t[k])) return true;
  return false;
}
bool pack_set(const LoraPack& p) {
  for (int k = 0; k < p.n; ++k)
    if (p.t[k].set) return true;
  return false;
}

// fuse_lora mode: every projection pack with a target set gets its merged copy (the rows of its unset members are
// the base weight); the others have none and their groups read the base weight
int merge_all(rf_dit* h, cudaStream_t s) {
  const int lpad = h->lora_pad;
  for (LoraPack* p : h->proj_packs) {
    if (!pack_set(*p)) continue;
    const size_t elems = static_cast<size_t>(p->t[0].out) * p->t[0].in;
    if (p->Wm == nullptr) RF_TRY(h->mem.alloc(&p->Wm, p->n * elems));
    for (int k = 0; k < p->n; ++k) {
      const LoraT& t = p->t[k];
      const size_t off = k * elems;
      if (t.set)
        RF_TRY(rf::lora_merge_launch(p->W + off, lora_A(t, lpad), lora_B(t, lpad), p->Wm + off, t.out, t.in, lpad,
                                     lora_eff(h, t), s));
      else
        RF_CHECK_CUDA(cudaMemcpyAsync(p->Wm + off, p->W + off, elems * 2, cudaMemcpyDeviceToDevice, s));
    }
  }
  h->lora_merged = true;
  h->merged_call_scale = h->call_scale;
  return 0;
}

// rows [row0, row0 + rows) of the joint buffers; `cond`: the condition stream
struct StreamRows {
  int row0, rows;
  bool cond;
};

// One projection launch: a group per token stream, each with the adapter pack of the weight it reads
struct Proj {
  rf::GemmGroupArgs g[3];
  StreamRows sr[3];
  const LoraPack* pack[3];
  int n = 0;
  // rows r of out (pitch ldo) = rows r of A (pitch lda) times the Linear w
  rf::GemmGroupArgs& add(const StreamRows& r, const bf16* A, int lda, const Lin& w, const LoraPack& p, bf16* out,
                         int ldo) {
    rf::GemmGroupArgs& a = g[n];
    memset(&a, 0, sizeof(a));
    a.A = A + static_cast<int64_t>(r.row0) * lda; a.lda = lda; a.M = r.rows; a.W = w.w; a.bias = w.b;
    a.out = out + static_cast<int64_t>(r.row0) * ldo; a.ldo = ldo;
    sr[n] = r;
    pack[n] = &p;
    ++n;
    return a;
  }
};

// The rule for which rows carry an adapter: group j of pr carries its pack when the pack is always-on, or the group
// is the condition stream, or latent_lora is set (lora_controller.py:5-9) - and the pack is on (exact mode) / has a
// target set (merged mode).  Merged mode points those groups at the merged copy and returns 0.  Exact mode returns
// the carrying groups in lg, in joint-buffer row order (txt, img / main, cond), which is their order in LT / LL.
int lora_groups(const rf_dit* h, Proj& pr, int* lg) {
  int n = 0;
  for (int j = 0; j < pr.n; ++j) {
    const LoraPack& p = *pr.pack[j];
    if (!p.always && !pr.sr[j].cond && !(h->flags & 1)) continue;
    if (h->use_merged) {
      if (pack_set(p)) pr.g[j].W = p.Wm;
    } else if (pack_on(h, p)) {
      lg[n++] = j;
    }
  }
  std::sort(lg, lg + n, [&](int a, int b) { return pr.sr[a].row0 < pr.sr[b].row0; });
  return n;
}

// A projection launch with the LoRA of its carrying groups.  Fast path: T = bf16(x A^T) for all LoRA'd rows in one
// skinny grouped GEMM (one group per run of rows that are contiguous in the A operand and share their A factor), then
// ONE grouped launch of all streams in which the eligible groups' tiles carry the low-rank k-block
// (GemmGroupArgs::lora_T) - L = T B^T never reaches HBM.  Groups too small for it (gemm_lora_eligible) keep the
// unfused path: L materialised in their rows of LL and added in the epilogue (`addend`); they reuse T when it exists.
// (t_pre != nullptr: T was already produced by an earlier launch, [rows, ld_t] with this pack's columns at t_pre.)
int project(rf_dit* h, int epi, int N, int K, Proj& pr, cudaStream_t s, const bf16* t_pre = nullptr, int ld_t = 0) {
  int lg[3], row[3];
  const int nl = lora_groups(h, pr, lg);
  const int lpad = h->lora_pad;
  bool fused[3] = {false, false, false}, any_fused = false;
  for (int j = 0, r = 0; j < nl; r += pr.g[lg[j]].M, ++j) {
    row[j] = r;
    any_fused |= (fused[j] = rf::gemm_lora_eligible(epi, N, K, pr.g[lg[j]]));
  }
  if (any_fused && t_pre == nullptr) {
    ld_t = pr.pack[lg[0]]->n * lpad;
    rf::GemmGroupArgs dg[3];
    memset(dg, 0, sizeof(dg));
    int nd = 0;
    for (int j = 0; j < nl; ++j) {
      const rf::GemmGroupArgs& gc = pr.g[lg[j]];
      const bf16* A = pr.pack[lg[j]]->A;
      rf::GemmGroupArgs* last = nd ? &dg[nd - 1] : nullptr;
      if (last && last->W == A && last->lda == gc.lda && gc.A == last->A + static_cast<int64_t>(last->M) * last->lda) {
        last->M += gc.M;
        continue;
      }
      dg[nd].A = gc.A; dg[nd].lda = gc.lda; dg[nd].M = gc.M; dg[nd].W = A;
      dg[nd].out = h->LT + static_cast<int64_t>(row[j]) * ld_t; dg[nd].ldo = ld_t;
      ++nd;
    }
    RF_TRY(rf::lora_down_launch(K, ld_t, nd, dg, s));
    t_pre = h->LT;
  }
  for (int j = 0; j < nl; ++j) {
    const LoraPack& p = *pr.pack[lg[j]];
    rf::GemmGroupArgs& gc = pr.g[lg[j]];
    const bf16* t_rows = t_pre ? t_pre + static_cast<int64_t>(row[j]) * ld_t : nullptr;
    if (fused[j]) {
      gc.lora_T = t_rows; gc.ld_t = ld_t; gc.lora_B = p.B; gc.lora_sec_cols = p.n > 1 ? p.t[0].out : 0;
      gc.lora_pad = lpad;
      for (int k = 0; k < p.n; ++k) gc.lora_scale[k] = lora_eff(h, p.t[k]);
    } else {
      bf16* L = h->LL + static_cast<int64_t>(row[j]) * N;
      RF_TRY(lora_term(h, p, gc.A, gc.lda, gc.M, t_rows, ld_t, L, N, s));
      gc.addend = L; gc.ldadd = N;
    }
  }
  return rf::gemm_launch(epi, N, K, pr.n, pr.g, s);
}

// The body of one DiT forward for one sample.  All pointers are device pointers.  mod_all != nullptr: the step's
// modulation vectors are row *row of that table (pooled, tstep and guid are not read).
int enqueue_forward(rf_dit* h, const bf16* latents, const bf16* txt, const bf16* pooled,
                    const bf16* tstep, const int* row, const bf16* guid, const bf16* cond_lat,
                    bf16* out, cudaStream_t s, const bf16* mod_all = nullptr) {
  const int D = h->D, D3 = 3 * D, D4 = 4 * D, D5 = 5 * D, C = h->cfg.in_channels, lpad = h->lora_pad;
  const bool use_cond = h->n_cond > 0;
  const StreamRows S_txt{0, h->n_txt, false}, S_img{h->n_txt, h->n_img, false}, S_main{0, h->n_main, false},
      S_cond{h->n_main, h->n_cond, true};
  bf16 *X = h->X, *XN = h->XN, *QKV = h->QKV, *ACT = h->ACT;
  // the epilogue operands of a group: RMSNorm weights and RoPE rows (EPI_QKV), gate + residual in place (GATE_RES)
  auto qk = [&](rf::GemmGroupArgs& a, const StreamRows& r, const bf16* norm_q, const bf16* norm_k) {
    a.rope_cos = r.cond ? h->crope_cos : h->rope_cos + static_cast<int64_t>(r.row0) * 64;
    a.rope_sin = r.cond ? h->crope_sin : h->rope_sin + static_cast<int64_t>(r.row0) * 64;
    a.norm_q = norm_q; a.norm_k = norm_k;
  };
  auto gate = [](rf::GemmGroupArgs& a, const bf16* g) {
    a.res = a.out; a.ldr = a.ldo; a.gate = g;
  };

  // ---- embedders (transformer.py:91-93,115); x_embedder reads the latents / condition latents themselves
  Proj xe;
  xe.add(S_img, latents, C, h->x_emb, h->l_x_emb, X, D).A = latents;
  if (use_cond) xe.add(S_cond, cond_lat, C, h->x_emb, h->l_x_emb, X, D).A = cond_lat;
  RF_TRY(project(h, rf::EPI_BIAS, D, C, xe, s));
  Proj ce;
  ce.add(S_txt, txt, h->cfg.joint_attention_dim, h->ctx_emb, h->l_ctx, X, D);
  RF_TRY(project(h, rf::EPI_BIAS, D, h->cfg.joint_attention_dim, ce, s));

  // ---- temb and every modulation vector of the step (transformer.py:95-107 + all adaLN linears)
  if (mod_all != nullptr) {  // denoise loop: this step's row of the precomputed table
    RF_TRY(rf::select_row_launch(mod_all, h->n_mod, row, h->MOD, s));
  } else {
    RF_TRY(temb_mod(h, 1, tstep, guid, pooled, (h->flags & 1) != 0, true, h->MOD, h->emb_ws, s));
  }
  const bf16* MOD = h->MOD;
  const bf16* MODC = h->MODC;

  // all token streams of a norm in ONE launch: rows are [txt | img | cond] of the joint buffers
  auto ln3 = [&](const bf16* sc_txt, const bf16* sh_txt, const bf16* sc_img, const bf16* sh_img,
                 const bf16* sc_cond, const bf16* sh_cond) {
    const int ends[3] = {h->n_txt, h->n_main, h->N};
    const bf16* sc[3] = {sc_txt, sc_img, sc_cond};
    const bf16* sh[3] = {sh_txt, sh_img, sh_cond};
    return rf::ln_modulate_grouped_launch(X, D, XN, D, D, use_cond ? 3 : 2, ends, sc, sh, s);
  };
  rf::AttnArgs at;
  at.q = QKV; at.k = QKV + D; at.v = QKV + 2 * D; at.ld_qkv = D3;
  at.n_tok = h->N; at.heads = h->cfg.num_heads; at.batch = 1;
  at.n_main = h->n_main; at.cond_mode = use_cond ? h->attn_cond_mode : 0;
  at.cond_bias = h->attn_cond_bias;

  // ================= double-stream blocks (block.py:173-272) =================
  // groups: img, txt, cond (this order sets the tile schedule); the txt group reads the text stream's own Linears
  for (int i = 0; i < h->cfg.num_layers; ++i) {
    const DoubleBlk& b = h->dbl[i];
    const bf16* mi = MOD + mod_double(h, i, 0, 0);
    const bf16* mt = MOD + mod_double(h, i, 1, 0);
    const bf16* mc = MODC + mod_double(h, i, 0, 0);
    // norm1 / norm1_context
    RF_TRY(ln3(mt + SCALE_MSA * D, mt + SHIFT_MSA * D, mi + SCALE_MSA * D, mi + SHIFT_MSA * D,
               mc + SCALE_MSA * D, mc + SHIFT_MSA * D));
    // q|k|v projections + RMSNorm + RoPE, all streams in one grouped launch
    Proj q;
    qk(q.add(S_img, XN, D, b.qkv, b.l_qkv, QKV, D3), S_img, b.norm_q, b.norm_k);
    qk(q.add(S_txt, XN, D, b.add_qkv, b.l_add_qkv, QKV, D3), S_txt, b.norm_added_q, b.norm_added_k);
    if (use_cond) qk(q.add(S_cond, XN, D, b.qkv, b.l_qkv, QKV, D3), S_cond, b.norm_q, b.norm_k);
    RF_TRY(project(h, rf::EPI_QKV, D3, D, q, s));
    // joint attention -> ACT[:, 0:D]
    at.out = ACT; at.ldo = D5;
    RF_TRY(rf::attention_launch(at, s));
    // out projections + gate + residual (in place on X)
    Proj o;
    gate(o.add(S_img, ACT, D5, b.to_out, b.l_out, X, D), mi + GATE_MSA * D);
    gate(o.add(S_txt, ACT, D5, b.to_add_out, b.l_add_out, X, D), mt + GATE_MSA * D);
    if (use_cond) gate(o.add(S_cond, ACT, D5, b.to_out, b.l_out, X, D), mc + GATE_MSA * D);
    RF_TRY(project(h, rf::EPI_GATE_RES, D, D, o, s));
    // norm2 + modulate
    RF_TRY(ln3(mt + SCALE_MLP * D, mt + SHIFT_MLP * D, mi + SCALE_MLP * D, mi + SHIFT_MLP * D,
               mc + SCALE_MLP * D, mc + SHIFT_MLP * D));
    // MLP in (GELU-tanh) -> ACT[:, D:5D]; ff.net.0.proj is inside no enable_lora (block.py:250 names ff.net[2] only)
    Proj f1;
    f1.add(S_img, XN, D, b.ff1, b.l_ff1, ACT + D, D5);
    f1.add(S_txt, XN, D, b.ffc1, b.l_ffc1, ACT + D, D5);
    if (use_cond) f1.add(S_cond, XN, D, b.ff1, b.l_ff1, ACT + D, D5);
    RF_TRY(project(h, rf::EPI_GELU, D4, D, f1, s));
    // MLP out + gate + residual
    Proj f2;
    gate(f2.add(S_img, ACT + D, D5, b.ff2, b.l_ff2, X, D), mi + GATE_MLP * D);
    gate(f2.add(S_txt, ACT + D, D5, b.ffc2, b.l_ffc2, X, D), mt + GATE_MLP * D);
    if (use_cond) gate(f2.add(S_cond, ACT + D, D5, b.ff2, b.l_ff2, X, D), mc + GATE_MLP * D);
    RF_TRY(project(h, rf::EPI_GATE_RES, D, D4, f2, s));
  }

  // ================= single-stream blocks (block.py:275-333) =================
  for (int i = 0; i < h->cfg.num_single_layers; ++i) {
    const SingleBlk& b = h->sgl[i];
    const bf16* mm = MOD + mod_single(h, i, 0);
    const bf16* mc = MODC + mod_single(h, i, 0);
    // txt and img rows share the block's vectors; the cond rows use the cond_temb ones
    RF_TRY(ln3(mm + 1 * D, mm + 0 * D, mm + 1 * D, mm + 0 * D, mc + 1 * D, mc + 0 * D));
    // q|k|v
    Proj q;
    qk(q.add(S_main, XN, D, b.qkv, b.l_qkv, QKV, D3), S_main, b.norm_q, b.norm_k);
    if (use_cond) qk(q.add(S_cond, XN, D, b.qkv, b.l_qkv, QKV, D3), S_cond, b.norm_q, b.norm_k);
    // exact-mode fast path: T for to_q|to_k|to_v|proj_mlp of all LoRA'd rows in one launch (both GEMMs read the
    // same XN rows; the q|k|v and the MLP-in launches have the same LoRA groups)
    int lg[3], t_rows = 0;
    const int nl = lora_groups(h, q, lg);
    bool t4 = false;
    for (int j = 0; j < nl; ++j) {
      t4 |= rf::gemm_lora_eligible(rf::EPI_QKV, D3, D, q.g[lg[j]]);
      t_rows += q.g[lg[j]].M;
    }
    t4 = t4 && pack_on(h, b.l_mlp);
    if (t4) RF_TRY(rf::lora_down_launch(q.g[lg[0]].A, D, t_rows, D, b.l_qkv.A, 4 * lpad, h->LT, 4 * lpad, s));
    RF_TRY(project(h, rf::EPI_QKV, D3, D, q, s, t4 ? h->LT : nullptr, 4 * lpad));
    // proj_mlp + GELU -> ACT[:, D:5D]
    Proj m;
    m.add(S_main, XN, D, b.mlp, b.l_mlp, ACT + D, D5);
    if (use_cond) m.add(S_cond, XN, D, b.mlp, b.l_mlp, ACT + D, D5);
    RF_TRY(project(h, rf::EPI_GELU, D4, D, m, s, t4 ? h->LT + 3 * lpad : nullptr, 4 * lpad));
    // attention -> ACT[:, 0:D]
    at.out = ACT; at.ldo = D5;
    RF_TRY(rf::attention_launch(at, s));
    // proj_out over cat(attn, mlp) (K = 5D) + gate + residual
    Proj o;
    gate(o.add(S_main, ACT, D5, b.out, b.l_out, X, D), mm + 2 * D);
    if (use_cond) gate(o.add(S_cond, ACT, D5, b.out, b.l_out, X, D), mc + 2 * D);
    RF_TRY(project(h, rf::EPI_GATE_RES, D, D5, o, s));
  }

  // ================= norm_out + proj_out (transformer.py:241-244) =================
  const bf16* mo = MOD + mod_out(h, 0);  // [scale | shift]
  const int64_t img0 = static_cast<int64_t>(S_img.row0) * D;
  RF_TRY(rf::ln_modulate_launch(X + img0, D, XN + img0, D, S_img.rows, D, mo, mo + D, S_img.rows, 0, s));
  Proj po;
  po.add(S_img, XN, D, h->proj_out, h->l_proj_out, out, C).out = out;
  return project(h, rf::EPI_BIAS, C, D, po, s);
}

// fuse_lora mode applies when some group carries a LoRA: the condition stream, the image under latent_lora, or the
// rows of an always target
bool wants_merged(const rf_dit* h, int n_cond) {
  return (h->flags & 8) != 0 && h->any_lora && (n_cond > 0 || (h->flags & 1) != 0 || h->any_always);
}

// rows that can carry a LoRA term (LT / LL): the condition stream, plus txt + img under latent_lora (the single
// blocks LoRA every main row) or with an always target set (text stream, image rows of ff.net.0.proj / proj_out)
int lora_rows_needed(const rf_dit* h, int flags, int N, int n_cond) {
  return std::max(((flags & 1) || h->any_always) ? N : n_cond, 1);
}
// LT [rows, 4 lora_pad] and LL [rows, 4D]
int alloc_lora_ws(rf_dit* h, int rows) {
  const size_t r = static_cast<size_t>(rows);
  RF_TRY(h->geo_mem.alloc(&h->LT, r * 4 * h->lora_pad));
  RF_TRY(h->geo_mem.alloc(&h->LL, r * 4 * h->D));
  h->lora_rows = rows;
  return 0;
}
// the merged copies hold W + (B A) * scaling for the current weights, adapters and call scale
bool merged_current(const rf_dit* h) { return h->lora_merged && h->merged_call_scale == h->call_scale; }

void drop_graph(rf_dit* h) {
  h->sess = false;  // the session replays this graph
  for (StepGraph* g : {&h->graph, &h->graph_ig}) {
    if (g->exec) {
      cudaGraphExecDestroy(g->exec);
      g->exec = nullptr;
    }
  }
}
void free_geometry(rf_dit* h) {
  drop_graph(h);
  h->geo_mem.release_all();
  h->prepared = false;
  h->lora_rows = 0;
  h->tab_steps = 0;
  h->s_tsteps = h->tab = h->tab_u = h->temb_ws = nullptr;
  h->s_sigmas = nullptr;
  h->idx = nullptr;
}

}  // namespace

namespace rf {
__global__ void add2_kernel(const bf16* a, const bf16* b, bf16* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16_rn(__bfloat162float(a[i]) + __bfloat162float(b[i]));
}
int add2_launch(const bf16* a, const bf16* b, bf16* out, int n, cudaStream_t stream) {
  add2_kernel<<<(n + 255) / 256, 256, 0, stream>>>(a, b, out, n);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
__global__ void add_rows_kernel(bf16* dst, int64_t ldd, const bf16* src, int lds, int cols, float scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (c >= cols) return;
  bf16* d = dst + r * ldd + c;
  const float v = __bfloat162float(__float2bfloat16_rn(__bfloat162float(src[static_cast<int64_t>(r) * lds + c]) * scale));
  *d = __float2bfloat16_rn(__bfloat162float(*d) + v);
}
int add_rows_launch(bf16* dst, int64_t ldd, const bf16* src, int lds, int rows, int cols, float scale,
                    cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return 0;
  add_rows_kernel<<<dim3((cols + 255) / 256, rows), 256, 0, stream>>>(dst, ldd, src, lds, cols, scale);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
// out[0:row_elems] = table[*row]  (16-byte vectors; row_elems % 8 == 0)
__global__ void select_row_kernel(const uint4* __restrict__ table, int64_t row_vecs,
                                  const int* __restrict__ row, uint4* __restrict__ out) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // PDL: see rf_ptx.cuh
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < row_vecs) out[i] = table[static_cast<int64_t>(*row) * row_vecs + i];
}
int select_row_launch(const bf16* table, int64_t row_elems, const int* row, bf16* out,
                      cudaStream_t stream) {
  if (row_elems % 8 != 0) {
    set_error("select_row: row length must be a multiple of 8");
    return -1;
  }
  const int64_t vecs = row_elems / 8;
  RF_CHECK_CUDA(launch_pdl(select_row_kernel, dim3(static_cast<unsigned>((vecs + 255) / 256)), dim3(256), 0, stream,
                           reinterpret_cast<const uint4*>(table), vecs, row, reinterpret_cast<uint4*>(out)));
  count_launch();
  return 0;
}
__global__ void f32_to_bf16_kernel(const float* src, bf16* dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __float2bfloat16_rn(src[i]);
}
int f32_to_bf16_launch(const float* src, bf16* dst, int n, cudaStream_t stream) {
  f32_to_bf16_kernel<<<(n + 255) / 256, 256, 0, stream>>>(src, dst, n);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
// Wm[n, k] = bf16( W[n, k] + scale * sum_r B[n, r] * A[r, k] ): what peft's fuse_lora / merge() produces
// (delta = (B A) * scaling, get_delta_weight), with one rounding
__global__ void lora_merge_kernel(const bf16* __restrict__ W, const bf16* __restrict__ A,
                                  const bf16* __restrict__ B, bf16* __restrict__ Wm, int N, int K,
                                  int R, float scale) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  if (k >= K) return;
  float acc = 0.f;
  for (int r = 0; r < R; ++r)
    acc = fmaf(__bfloat162float(B[static_cast<size_t>(n) * R + r]),
               __bfloat162float(A[static_cast<size_t>(r) * K + k]), acc);
  const size_t i = static_cast<size_t>(n) * K + k;
  Wm[i] = __float2bfloat16_rn(__bfloat162float(W[i]) + __fmul_rn(scale, acc));
}
int lora_merge_launch(const bf16* W, const bf16* A, const bf16* B, bf16* Wm, int N, int K, int R, float scale,
                      cudaStream_t stream) {
  dim3 grid((K + 255) / 256, N);
  lora_merge_kernel<<<grid, 256, 0, stream>>>(W, A, B, Wm, N, K, R, scale);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
// bf16 ids [n,3] -> pair-compact fp32 cos/sin [n,64] (diffusers FluxPosEmbed, axes 16/56/56,
// theta 1e4, angles in float64 like the reference; transformer.py:130-134)
__global__ void rope_table_kernel(const bf16* ids, int n, float* cosv, float* sinv) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * 64) return;
  const int r = idx / 64, p = idx % 64;
  int axis, j, dim;
  if (p < 8) { axis = 0; j = p; dim = 16; }
  else if (p < 36) { axis = 1; j = p - 8; dim = 56; }
  else { axis = 2; j = p - 36; dim = 56; }
  const double pos = static_cast<double>(__bfloat162float(ids[r * 3 + axis]));
  const double freq = 1.0 / pow(10000.0, static_cast<double>(2 * j) / static_cast<double>(dim));
  const double ang = pos * freq;
  cosv[idx] = static_cast<float>(cos(ang));
  sinv[idx] = static_cast<float>(sin(ang));
}
}  // namespace rf

extern "C" {

int rf_dit_create(const rf_dit_config* cfg, rf_dit** out) {
  if (!cfg || !out) {
    rf::set_error("rf_dit_create: null argument");
    return -1;
  }
  if (cfg->lora_rank < 0 || cfg->lora_rank > 128) {
    rf::set_error("rf_dit_create: lora_rank must be 0..128, got " + std::to_string(cfg->lora_rank));
    return -1;
  }
  RF_TRY(rf::require_device("rf_dit_create"));
  if (cfg->num_heads <= 0 || cfg->in_channels % 64 != 0 || cfg->joint_attention_dim % 64 != 0 ||
      cfg->pooled_projection_dim % 8 != 0) {
    rf::set_error("rf_dit_create: unsupported config");
    return -1;
  }
  rf_dit* h = new rf_dit();
  h->cfg = *cfg;
  h->lora_pad = cfg->lora_rank <= 64 ? 64 : 128;
  h->D = cfg->num_heads * 128;
  if (h->D % 256 != 0 || h->D > 3072) {
    rf::set_error("rf_dit_create: inner dim must be a multiple of 256, <= 3072");
    delete h;
    return -1;
  }
  cudaGetDevice(&h->device);
  // opt in to the large dynamic shared-memory carve-outs up front (not inside a graph capture)
  if (rf::gemm_init() || rf::attention_init() || rf::gemv_init()) {
    delete h;
    return -2;
  }
  int rc = build_storage(h);
  if (rc) {
    rf_dit_destroy(h);
    return rc;
  }
  // zero LoRA storage (padding rows/cols must be zero) happens lazily in set_lora
  *out = h;
  return 0;
}

void rf_dit_destroy(rf_dit* h) {
  if (!h) return;
  free_geometry(h);
  h->side.destroy();
  h->mem.release_all();
  delete h;
}

int rf_dit_load_weight(rf_dit* h, const char* key, const void* src, int64_t numel) {
  if (!h || !key || !src) {
    rf::set_error("rf_dit_load_weight: null argument");
    return -1;
  }
  RF_TRY(h->weights.load("rf_dit_load_weight", key, src, numel));
  h->lora_merged = false;  // merged W + BA copies (fuse_lora mode) are stale now
  h->sess = false;         // and so are the session's modulation tables
  return 0;
}

int rf_dit_set_lora(rf_dit* h, const char* module, const void* A, const void* B, int r,
                    int in_features, int out_features, float scale) {
  if (!h || !module || !A || !B) {
    rf::set_error("rf_dit_set_lora: null argument");
    return -1;
  }
  auto it = h->lora_slots.find(module);
  if (it == h->lora_slots.end()) {
    rf::set_error(std::string("rf_dit_set_lora: not a Linear of FluxTransformer2DModel (or lora_rank == 0): ") +
                  module);
    return -4;
  }
  if (r <= 0 || r > h->cfg.lora_rank) {
    rf::set_error("rf_dit_set_lora: rank " + std::to_string(r) + " of " + module + " exceeds the handle's lora_rank " +
                  std::to_string(h->cfg.lora_rank));
    return -1;
  }
  if (!std::isfinite(scale)) {
    rf::set_error(std::string("rf_dit_set_lora: scale (lora_alpha / r) of ") + module + " must be finite");
    return -1;
  }
  const int lpad = h->lora_pad;
  LoraT& t = *it->second;
  if (in_features != t.in || out_features != t.out) {
    rf::set_error(std::string("rf_dit_set_lora: ") + module + " expects A [r, " + std::to_string(t.in) +
                  "], B [" + std::to_string(t.out) + ", r]; got in=" + std::to_string(in_features) +
                  " out=" + std::to_string(out_features));
    return -4;
  }
  RF_TRY(lora_storage(h, *t.pack));
  bf16 *tA = lora_A(t, lpad), *tB = lora_B(t, lpad);
  RF_CHECK_CUDA(cudaMemset(tA, 0, static_cast<size_t>(lpad) * t.in * 2));
  RF_CHECK_CUDA(cudaMemset(tB, 0, static_cast<size_t>(t.out) * lpad * 2));
  RF_CHECK_CUDA(cudaMemcpy(tA, A, static_cast<size_t>(r) * t.in * 2, cudaMemcpyDeviceToDevice));
  RF_CHECK_CUDA(cudaMemcpy2D(tB, lpad * 2, B, static_cast<size_t>(r) * 2,
                             static_cast<size_t>(r) * 2, t.out, cudaMemcpyDeviceToDevice));
  t.set = true;
  t.scale = scale;
  h->any_lora = true;
  h->any_always |= t.pack->always;
  h->lora_merged = false;
  drop_graph(h);  // the captured step may predate this adapter (different launch list)
  return 0;
}

int rf_dit_clear_lora(rf_dit* h) {
  if (!h) {
    rf::set_error("rf_dit_clear_lora: null handle");
    return -1;
  }
  const int lpad = h->lora_pad;
  for (auto& kv : h->lora_slots) {
    LoraT& t = *kv.second;
    // zeroed: an unset member of a stacked q|k|v pack still runs in its pack's GEMMs and must add exactly nothing
    if (t.set) {
      RF_CHECK_CUDA(cudaMemset(lora_A(t, lpad), 0, static_cast<size_t>(lpad) * t.in * 2));
      RF_CHECK_CUDA(cudaMemset(lora_B(t, lpad), 0, static_cast<size_t>(t.out) * lpad * 2));
    }
    t.set = false;
    t.scale = 1.0;
  }
  h->any_lora = false;
  h->any_always = false;
  h->lora_merged = false;
  drop_graph(h);
  return 0;
}

int rf_dit_set_lora_scale(rf_dit* h, double scale) {
  if (!h) {
    rf::set_error("rf_dit_set_lora_scale: null handle");
    return -1;
  }
  if (!std::isfinite(scale)) {
    rf::set_error("rf_dit_set_lora_scale: scale must be finite");
    return -1;
  }
  // takes effect at the next call: the merged copies are re-merged (check_ready) and the captured step is
  // re-captured (rf_dit_denoise) when they were built for another scale; the session's tables hold the old scale
  h->call_scale = scale;
  h->sess = false;
  return 0;
}

int rf_dit_missing_weights(rf_dit* h) { return h ? h->weights.missing("", "missing weights") : -1; }

int rf_dit_prepare(rf_dit* h, int batch, int n_txt, int n_img, int n_cond, const void* txt_ids,
                   const void* img_ids, const void* cond_ids, int flags, float condition_scale,
                   void* stream) {
  if (!h || !txt_ids || !img_ids || (n_cond > 0 && !cond_ids)) {
    rf::set_error("rf_dit_prepare: null argument");
    return -1;
  }
  if (batch <= 0 || n_txt <= 0 || n_img <= 0 || n_cond < 0) {
    rf::set_error("rf_dit_prepare: bad geometry");
    return -1;
  }
  if (flags & 2) {
    rf::set_error("rf_dit_prepare: add_cond_attn=true is not implemented");
    return -1;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int n_main = n_txt + n_img, N = n_main + n_cond, D = h->D;
  int mode = 0;
  float bias = 0.f;
  if (n_cond > 0) {
    if (condition_scale != 1.0f) {
      mode = 1;
      // the reference builds the mask in the query dtype: log(c) rounded to bf16
      bias = __bfloat162float(__float2bfloat16_rn(logf(condition_scale)));
    }
    if (flags & 4) mode = 2;  // union_cond_attn == False wins only if no c_factor...
    if ((flags & 4) && condition_scale != 1.0f) mode = 1;  // c_factor mask overrides (block.py:115)
  }
  const int lora_rows = lora_rows_needed(h, flags, N, n_cond);
  const bool same = h->prepared && h->batch == batch && h->n_txt == n_txt && h->n_img == n_img &&
                    h->n_cond == n_cond && h->lora_rows >= lora_rows;
  if (same) drop_graph(h); else free_geometry(h);
  h->flags = flags;
  h->use_merged = wants_merged(h, n_cond);
  if (h->use_merged && !merged_current(h)) {
    int mrc = merge_all(h, s);
    if (mrc) return mrc;
  }
  h->attn_cond_mode = mode;
  h->attn_cond_bias = bias;
  if (!same) {
    h->prepared = false;
    h->batch = batch; h->n_txt = n_txt; h->n_img = n_img; h->n_cond = n_cond;
    h->N = N; h->n_main = n_main;
    rf::DeviceAllocs& g = h->geo_mem;
    const size_t nc = std::max(n_cond, 1);
    RF_TRY(g.alloc(&h->rope_cos, static_cast<size_t>(n_main) * 64));
    RF_TRY(g.alloc(&h->rope_sin, static_cast<size_t>(n_main) * 64));
    RF_TRY(g.alloc(&h->crope_cos, nc * 64));
    RF_TRY(g.alloc(&h->crope_sin, nc * 64));
    RF_TRY(g.alloc(&h->X, static_cast<size_t>(N) * D));
    RF_TRY(g.alloc(&h->XN, static_cast<size_t>(N) * D));
    RF_TRY(g.alloc(&h->QKV, static_cast<size_t>(N) * 3 * D));
    RF_TRY(g.alloc(&h->ACT, static_cast<size_t>(N) * 5 * D));
    RF_TRY(g.alloc(&h->MOD, h->n_mod));
    RF_TRY(g.alloc(&h->MODC, h->n_mod));
    RF_TRY(alloc_lora_ws(h, lora_rows));
    RF_TRY(g.alloc(&h->emb_ws, temb_ws_elems(h, 1)));
    const int C = h->cfg.in_channels;
    RF_TRY(g.alloc(&h->s_lat, static_cast<size_t>(n_img) * C));
    RF_TRY(g.alloc(&h->s_v, static_cast<size_t>(n_img) * C));
    RF_TRY(g.alloc(&h->s_txt, static_cast<size_t>(n_txt) * h->cfg.joint_attention_dim));
    RF_TRY(g.alloc(&h->s_cond, nc * C));
    RF_TRY(g.alloc(&h->s_guid, static_cast<size_t>(batch) + 8));
    RF_TRY(g.alloc(&h->s_zero_one, 8));
    RF_TRY(g.alloc(&h->s_step, 4));
    RF_TRY(g.alloc(&h->s_row, 4));
    if (n_cond > 0) {
      RF_TRY(g.alloc(&h->tab_c, static_cast<size_t>(batch) * h->n_mod));
      RF_TRY(g.alloc(&h->loop_cond, static_cast<size_t>(batch) * n_cond * C));
      // image guidance needs a condition stream
      RF_TRY(g.alloc(&h->s_ucond, static_cast<size_t>(n_cond) * C));
      RF_TRY(g.alloc(&h->s_vu, static_cast<size_t>(n_img) * C));
      RF_TRY(g.alloc(&h->s_igs, 4));
    }
    const uint16_t zo[2] = {0x0000, 0x3F80};  // bf16 0.0, 1.0
    RF_CHECK_CUDA(cudaMemcpy(h->s_zero_one, zo, sizeof(zo), cudaMemcpyHostToDevice));
  }
  // RoPE tables: once per geometry instead of every step (SURVEY App. B.14)
  {
    // ids of the joint sequence = cat(txt_ids, img_ids); gather into X as scratch
    bf16* ids = h->XN;  // scratch
    RF_CHECK_CUDA(cudaMemcpyAsync(ids, txt_ids, static_cast<size_t>(n_txt) * 3 * 2,
                                  cudaMemcpyDeviceToDevice, s));
    RF_CHECK_CUDA(cudaMemcpyAsync(ids + static_cast<size_t>(n_txt) * 3, img_ids,
                                  static_cast<size_t>(n_img) * 3 * 2, cudaMemcpyDeviceToDevice, s));
    const int tot = n_main * 64;
    rf::rope_table_kernel<<<(tot + 255) / 256, 256, 0, s>>>(ids, n_main, h->rope_cos, h->rope_sin);
    RF_CHECK_CUDA(cudaGetLastError());
    rf::count_launch();
    if (n_cond > 0) {
      const int totc = n_cond * 64;
      rf::rope_table_kernel<<<(totc + 255) / 256, 256, 0, s>>>(
          static_cast<const bf16*>(cond_ids), n_cond, h->crope_cos, h->crope_sin);
      RF_CHECK_CUDA(cudaGetLastError());
      rf::count_launch();
    }
    RF_CHECK_CUDA(cudaStreamSynchronize(s));
  }
  h->prepared = true;
  return 0;
}

static int check_ready(rf_dit* h, const char* who, cudaStream_t s) {
  if (!h) {
    rf::set_error(std::string(who) + ": null handle");
    return -1;
  }
  if (!h->prepared) {
    rf::set_error(std::string(who) + ": call rf_dit_prepare first");
    return -1;
  }
  if (rf_dit_missing_weights(h) != 0) return -4;
  // an always target set after rf_dit_prepare puts a LoRA on rows the workspace may not cover yet
  const int rows = lora_rows_needed(h, h->flags, h->N, h->n_cond);
  if (rows > h->lora_rows) {
    drop_graph(h);
    h->geo_mem.release(h->LT);
    h->geo_mem.release(h->LL);
    RF_TRY(alloc_lora_ws(h, rows));
  }
  // fuse_lora mode: weights or adapters changed since the last merge -> re-merge before use
  h->use_merged = wants_merged(h, h->n_cond);
  if (h->use_merged && !merged_current(h)) {
    drop_graph(h);
    RF_TRY(merge_all(h, s));
  }
  return 0;
}

int rf_dit_forward(rf_dit* h, const void* latents, const void* txt, const void* pooled,
                   const void* timestep, const float* guidance, const void* cond_latents,
                   void* out, void* stream) {
  int rc = check_ready(h, "rf_dit_forward", static_cast<cudaStream_t>(stream));
  if (rc) return rc;
  if (!latents || !txt || !pooled || !timestep || !out || (h->n_cond > 0 && !cond_latents) ||
      (h->cfg.guidance_embeds && !guidance)) {
    rf::set_error("rf_dit_forward: null argument");
    return -1;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int C = h->cfg.in_channels;
  // guidance arrives as fp32 (generate.py:226) and is cast to bf16 by the model (transformer.py:98)
  if (h->cfg.guidance_embeds) RF_TRY(rf::f32_to_bf16_launch(guidance, h->s_guid, h->batch, s));
  for (int b = 0; b < h->batch; ++b) {
    const bf16* lat_b = static_cast<const bf16*>(latents) + static_cast<int64_t>(b) * h->n_img * C;
    const bf16* txt_b = static_cast<const bf16*>(txt) +
                        static_cast<int64_t>(b) * h->n_txt * h->cfg.joint_attention_dim;
    const bf16* pool_b = static_cast<const bf16*>(pooled) +
                         static_cast<int64_t>(b) * h->cfg.pooled_projection_dim;
    const bf16* t_b = static_cast<const bf16*>(timestep) + b;
    const bf16* cond_b = h->n_cond > 0 ? static_cast<const bf16*>(cond_latents) +
                                             static_cast<int64_t>(b) * h->n_cond * C
                                       : nullptr;
    bf16* out_b = static_cast<bf16*>(out) + static_cast<int64_t>(b) * h->n_img * C;
    if (h->n_cond > 0) RF_TRY(compute_cond_mod(h, pool_b, s));
    RF_TRY(enqueue_forward(h, lat_b, txt_b, pool_b, t_b, nullptr, h->s_guid + b, cond_b, out_b, s));
  }
  return 0;
}

// Capture one step of the denoise loop into g: forward -> Euler update, or with image guidance forward (cond) ->
// forward (uncond: its own modulation table, condition input U_i) -> guidance + Euler.  Both forwards read the table
// row at s_row, the update reads the sigmas at s_step.
static int capture_step(rf_dit* h, bool guided, StepGraph* g, cudaStream_t s) {
  const int C = h->cfg.in_channels;
  g->call_scale = h->call_scale;
  auto step = [&]() {
    RF_TRY(enqueue_forward(h, h->s_lat, h->s_txt, nullptr, nullptr, h->s_row, nullptr,
                           h->n_cond > 0 ? h->s_cond : nullptr, h->s_v, s, h->tab));
    if (!guided) return rf::euler_step_launch(h->s_lat, h->s_v, h->s_sigmas, h->s_step, h->n_img * C, s);
    RF_TRY(enqueue_forward(h, h->s_lat, h->s_txt, nullptr, nullptr, h->s_row, nullptr, h->s_ucond, h->s_vu, s,
                           h->tab_u));
    return rf::image_guidance_step_launch(h->s_lat, h->s_v, h->s_vu, h->s_igs, h->s_sigmas, h->s_step, h->n_img * C,
                                          s);
  };
  return rf::capture_graph(s, "rf_dit", step, &g->exec, &g->kernels);
}

// The checks of the three loop entry points; who names the entry point in the messages.  inputs_ok: the whole
// loop's own inputs are there (begin has none).  On a ready handle the call closes the step session first.
static int check_loop(rf_dit* h, const char* who, cudaStream_t s, bool inputs_ok, const void* pooled,
                      const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps,
                      const void* cond_latents, bool guided, float image_guidance_scale) {
  RF_TRY(check_ready(h, who, s));
  h->sess = false;
  if (!inputs_ok || !pooled || !timesteps_bf16_host || !sigmas_host || n_steps <= 0 ||
      (h->n_cond > 0 && !cond_latents)) {
    rf::set_error(std::string(who) + ": bad argument");
    return -1;
  }
  if (guided && (h->n_cond <= 0 || !h->cfg.guidance_embeds)) {
    rf::set_error(std::string(who) + ": image guidance needs a condition stream (n_cond > 0) and guidance_embeds");
    return -1;
  }
  if (!std::isfinite(image_guidance_scale)) {
    rf::set_error(std::string(who) + ": image_guidance_scale must be finite");
    return -1;
  }
  return 0;
}

// Open a loop of n_steps on stream s: upload the schedule, build every sample's tables (by the temb_mod calls of the
// eager forward: bit-identical rows), stage the condition latents, and capture the step unless the current one was
// built for this call scale.  Growing the tables drops the captured step, which reads them.
static int open_loop(rf_dit* h, const void* pooled, const uint16_t* timesteps_bf16_host, const float* sigmas_host,
                     int n_steps, float guidance_scale, const void* cond_latents, bool guided,
                     float image_guidance_scale, cudaStream_t s) {
  rf::DeviceAllocs& gm = h->geo_mem;
  const int B = h->batch;
  // growing keeps the old arrays until the geometry is freed: cudaFree would synchronise the device mid-call
  if (n_steps > h->tab_steps) {
    const size_t rows = static_cast<size_t>(B) * n_steps;
    RF_TRY(gm.alloc(&h->s_tsteps, n_steps));
    RF_TRY(gm.alloc(&h->s_sigmas, n_steps + 1));
    RF_TRY(gm.alloc(&h->tab, rows * h->n_mod));
    RF_TRY(gm.alloc(&h->temb_ws, temb_ws_elems(h, n_steps)));
    RF_TRY(gm.alloc(&h->idx, rows));
    h->tab_u = nullptr;
    std::vector<int> idx(rows);
    for (size_t r = 0; r < rows; ++r) idx[r] = static_cast<int>(r);
    RF_CHECK_CUDA(cudaMemcpyAsync(h->idx, idx.data(), rows * sizeof(int), cudaMemcpyHostToDevice, s));
    h->tab_steps = n_steps;
    drop_graph(h);
  }
  // no guided step exists without tab_u
  if (guided && !h->tab_u) RF_TRY(gm.alloc(&h->tab_u, static_cast<size_t>(B) * h->tab_steps * h->n_mod));
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_tsteps, timesteps_bf16_host, static_cast<size_t>(n_steps) * 2,
                                cudaMemcpyHostToDevice, s));
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_sigmas, sigmas_host, static_cast<size_t>(n_steps + 1) * 4,
                                cudaMemcpyHostToDevice, s));
  const bf16 gb = __float2bfloat16_rn(guidance_scale);
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_guid, &gb, 2, cudaMemcpyHostToDevice, s));
  if (guided)
    RF_CHECK_CUDA(cudaMemcpyAsync(h->s_igs, &image_guidance_scale, 4, cudaMemcpyHostToDevice, s));
  if (h->n_cond > 0)
    RF_CHECK_CUDA(cudaMemcpyAsync(h->loop_cond, cond_latents,
                                  static_cast<size_t>(B) * h->n_cond * h->cfg.in_channels * 2,
                                  cudaMemcpyDeviceToDevice, s));
  for (int b = 0; b < B; ++b) {
    const bf16* pool_b = static_cast<const bf16*>(pooled) + static_cast<int64_t>(b) * h->cfg.pooled_projection_dim;
    const int64_t row0 = static_cast<int64_t>(b) * n_steps * h->n_mod;
    if (h->n_cond > 0) RF_TRY(compute_cond_mod(h, pool_b, s, h->tab_c + static_cast<int64_t>(b) * h->n_mod));
    RF_TRY(temb_mod(h, n_steps, h->s_tsteps, h->s_guid, pool_b, (h->flags & 1) != 0, true, h->tab + row0,
                    h->temb_ws, s));
    // the uncond branch: guidance = torch.ones_like(guidance) -> bf16(1) * 1000 in the model (generate.py:262)
    if (guided)
      RF_TRY(temb_mod(h, n_steps, h->s_tsteps, h->s_zero_one + 1, pool_b, (h->flags & 1) != 0, true,
                      h->tab_u + row0, h->temb_ws, s));
  }
  h->sess_steps = n_steps;
  h->sess_guided = guided;
  // the captured step holds the LoRA scalings as kernel parameters (and skips the terms a zero scaling
  // removes): a changed call scale is re-captured
  StepGraph* g = guided ? &h->graph_ig : &h->graph;
  if (g->exec && g->call_scale != h->call_scale) drop_graph(h);
  if (!g->exec) RF_TRY(capture_step(h, guided, g, s));
  return 0;
}

// Step i of sample b of the open loop: stage sample b of latents [B, n_img, C] and txt [B, n_txt, 4096], its condition
// latents, cond_temb vectors and (image-guided loops) U_i `ucond`, set the sigma index and the table row, replay the
// captured step and copy the sample's latents back.  Device-to-device copies only.
static int loop_step(rf_dit* h, int b, int i, void* latents, const void* txt, const bf16* ucond, cudaStream_t s) {
  const size_t lat_bytes = static_cast<size_t>(h->n_img) * h->cfg.in_channels * 2;
  const size_t txt_bytes = static_cast<size_t>(h->n_txt) * h->cfg.joint_attention_dim * 2;
  char* lat = static_cast<char*>(latents) + b * lat_bytes;
  const size_t cond_elems = static_cast<size_t>(h->n_cond) * h->cfg.in_channels;
  const size_t mod_bytes = static_cast<size_t>(h->n_mod) * 2;
  auto d2d = [&](void* dst, const void* src, size_t bytes) {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s);
  };
  RF_CHECK_CUDA(d2d(h->s_lat, lat, lat_bytes));
  RF_CHECK_CUDA(d2d(h->s_txt, static_cast<const char*>(txt) + b * txt_bytes, txt_bytes));
  if (h->n_cond > 0) {
    RF_CHECK_CUDA(d2d(h->s_cond, h->loop_cond + b * cond_elems, cond_elems * 2));
    RF_CHECK_CUDA(d2d(h->MODC, h->tab_c + static_cast<int64_t>(b) * h->n_mod, mod_bytes));
  }
  if (h->sess_guided) RF_CHECK_CUDA(d2d(h->s_ucond, ucond, cond_elems * 2));
  RF_CHECK_CUDA(d2d(h->s_step, h->idx + i, sizeof(int)));
  RF_CHECK_CUDA(d2d(h->s_row, h->idx + b * h->sess_steps + i, sizeof(int)));
  const StepGraph& g = h->sess_guided ? h->graph_ig : h->graph;
  RF_CHECK_CUDA(cudaGraphLaunch(g.exec, s));
  rf::count_launch(static_cast<int>(g.kernels));
  RF_CHECK_CUDA(d2d(lat, h->s_lat, lat_bytes));
  return 0;
}

// rf_dit_denoise and rf_dit_denoise_image_guidance: open the loop, then step 0 .. n_steps-1 of every sample.
// uncond_latents: [B, n_steps, n_cond, C] (guided).
static int run_loop(rf_dit* h, const char* who, bool guided, void* latents_inout, const void* txt, const void* pooled,
                    const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps, float guidance_scale,
                    const void* cond_latents, const void* uncond_latents, float image_guidance_scale, void* stream) {
  // The loop runs on the handle's side stream, so the step can be captured whatever stream the caller passes
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  const bool inputs_ok = latents_inout && txt && (!guided || (cond_latents && uncond_latents));
  RF_TRY(check_loop(h, who, caller, inputs_ok, pooled, timesteps_bf16_host, sigmas_host, n_steps, cond_latents,
                    guided, image_guidance_scale));
  cudaStream_t s = nullptr;
  RF_TRY(h->side.enter(caller, &s));
  RF_TRY(open_loop(h, pooled, timesteps_bf16_host, sigmas_host, n_steps, guidance_scale, cond_latents, guided,
                   image_guidance_scale, s));
  const int64_t cond_elems = static_cast<int64_t>(h->n_cond) * h->cfg.in_channels;
  for (int i = 0; i < n_steps; ++i) {
    for (int b = 0; b < h->batch; ++b) {
      const int64_t u = (static_cast<int64_t>(b) * n_steps + i) * cond_elems;  // U_i of sample b
      const bf16* ucond = guided ? static_cast<const bf16*>(uncond_latents) + u : nullptr;
      RF_TRY(loop_step(h, b, i, latents_inout, txt, ucond, s));
    }
  }
  return h->side.leave(caller);
}

int rf_dit_denoise(rf_dit* h, void* latents_inout, const void* txt, const void* pooled,
                   const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps,
                   float guidance_scale, const void* cond_latents, void* stream) {
  return run_loop(h, "rf_dit_denoise", false, latents_inout, txt, pooled, timesteps_bf16_host, sigmas_host, n_steps,
                  guidance_scale, cond_latents, nullptr, 1.0f, stream);
}

int rf_dit_denoise_image_guidance(rf_dit* h, void* latents_inout, const void* txt, const void* pooled,
                                  const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps,
                                  float guidance_scale, const void* cond_latents, const void* uncond_latents,
                                  float image_guidance_scale, void* stream) {
  return run_loop(h, "rf_dit_denoise_image_guidance", true, latents_inout, txt, pooled, timesteps_bf16_host,
                  sigmas_host, n_steps, guidance_scale, cond_latents, uncond_latents, image_guidance_scale, stream);
}

int rf_dit_denoise_begin(rf_dit* h, const void* pooled, const uint16_t* timesteps_bf16_host, const float* sigmas_host,
                         int n_steps, float guidance_scale, const void* cond_latents, float image_guidance_scale,
                         void* stream) {
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  const bool guided = image_guidance_scale != 1.0f;
  RF_TRY(check_loop(h, "rf_dit_denoise_begin", caller, true, pooled, timesteps_bf16_host, sigmas_host, n_steps,
                    cond_latents, guided, image_guidance_scale));
  cudaStream_t s = nullptr;
  RF_TRY(h->side.enter(caller, &s));
  RF_TRY(open_loop(h, pooled, timesteps_bf16_host, sigmas_host, n_steps, guidance_scale, cond_latents, guided,
                   image_guidance_scale, s));
  h->sess = true;
  return h->side.leave(caller);
}

int rf_dit_denoise_step(rf_dit* h, int i, void* latents_inout, const void* txt, const void* uncond_latents_i,
                        void* stream) {
  if (!h) {
    rf::set_error("rf_dit_denoise_step: null handle");
    return -1;
  }
  if (!h->sess) {
    rf::set_error("rf_dit_denoise_step: no open session: call rf_dit_denoise_begin (rf_dit_prepare, LoRA and "
                  "weight changes, the LoRA call scale and a whole-loop denoise close it)");
    return -1;
  }
  if (i < 0 || i >= h->sess_steps) {
    rf::set_error("rf_dit_denoise_step: step " + std::to_string(i) + " outside [0, " +
                  std::to_string(h->sess_steps) + ")");
    return -1;
  }
  if (!latents_inout || !txt || (uncond_latents_i != nullptr) != h->sess_guided) {
    rf::set_error(h->sess_guided ? "rf_dit_denoise_step: bad argument (an image-guided session needs uncond_latents_i)"
                                 : "rf_dit_denoise_step: bad argument (uncond_latents_i is for image-guided sessions)");
    return -1;
  }
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  cudaStream_t s = nullptr;
  RF_TRY(h->side.enter(caller, &s));
  const int64_t cond_elems = static_cast<int64_t>(h->n_cond) * h->cfg.in_channels;
  for (int b = 0; b < h->batch; ++b) {
    const bf16* ucond = h->sess_guided ? static_cast<const bf16*>(uncond_latents_i) + b * cond_elems : nullptr;
    RF_TRY(loop_step(h, b, i, latents_inout, txt, ucond, s));
  }
  return h->side.leave(caller);
}

}  // extern "C"
