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

#define RF_TRY(expr)            \
  do {                          \
    int _rc = (expr);           \
    if (_rc != 0) return _rc;   \
  } while (0)

namespace {

struct Slot {
  bf16* dst;
  int64_t numel;
  bool loaded;
};

struct Lin {  // views into the weight arena
  bf16* w = nullptr;
  bf16* b = nullptr;
};

struct LoraT {  // factors of one target, rank zero-padded to the handle's lora_pad
  bf16* A = nullptr;  // [lora_pad, in]
  bf16* B = nullptr;  // [out, lora_pad]
  int in = 0, out = 0;
  bool set = false;
  double scale = 1.0;  // lora_alpha / r
  // The Linears outside train_flux/config.yaml:53 (text stream, embedders, final layer, ff.net.0.proj) are "always"
  // targets: no enable_lora block names them, so every call applies them, latent_lora or not.  Their factors are
  // allocated on the first rf_dit_set_lora, so a handle that never sees such an adapter keeps its footprint.  A
  // member of a stacked pack (add_q|k|v) allocates the whole pack, zeroed, and points its siblings into it.
  bool always = false;
  LoraT* pack[3] = {nullptr, nullptr, nullptr};
  int npack = 0;
  bf16** packA = nullptr;
  bf16** packB = nullptr;
};
// (merged weights W + B A of a whole packed projection live in the block structs: *_m)

struct DoubleBlk {
  Lin qkv, add_qkv, to_out, to_add_out, ff1, ff2, ffc1, ffc2;
  bf16 *norm_q, *norm_k, *norm_added_q, *norm_added_k;
  LoraT l_norm1, l_q, l_k, l_v, l_out, l_ff2;
  // always targets: text stream (norm1_context, add_q|k|v, to_add_out, ff_context) and ff.net.0.proj
  LoraT l_norm1c, l_aq, l_ak, l_av, l_add_out, l_ff1, l_ffc1, l_ffc2;
  bf16* qkvA = nullptr;  // [3 lora_pad, D] = stacked A of to_q/to_k/to_v
  bf16* qkvB = nullptr;  // [3D, lora_pad] = stacked B (rows of the packed q|k|v projection)
  bf16* add_qkvA = nullptr;  // the same for add_q_proj / add_k_proj / add_v_proj (allocated on first use)
  bf16* add_qkvB = nullptr;
  bf16 *qkv_m = nullptr, *to_out_m = nullptr, *ff2_m = nullptr;  // merged W + B A (fuse_lora mode)
  bf16 *add_qkv_m = nullptr, *to_add_out_m = nullptr, *ff1_m = nullptr, *ffc1_m = nullptr, *ffc2_m = nullptr;
};
struct SingleBlk {
  Lin qkv, mlp, out;
  bf16 *norm_q, *norm_k;
  LoraT l_norm, l_q, l_k, l_v, l_mlp, l_out;
  bf16* qkvA = nullptr;
  bf16* qkvB = nullptr;
  bf16 *qkv_m = nullptr, *mlp_m = nullptr, *out_m = nullptr;
};

}  // namespace

struct rf_dit {
  rf_dit_config cfg;
  int D = 0;
  int device = 0;
  // ---- weights
  std::vector<void*> allocs;      // weights: live until destroy
  std::vector<void*> geo_allocs;  // workspace of the current geometry: freed on re-prepare
  std::unordered_map<std::string, Slot> slots;
  std::unordered_map<std::string, LoraT*> lora_slots;
  Lin x_emb, ctx_emb, t1, t2, g1, g2, p1, p2, proj_out;
  LoraT l_x_emb;
  // always targets at the top level: context_embedder, the time / guidance / text embedders, norm_out, proj_out
  LoraT l_ctx, l_t1, l_t2, l_g1, l_g2, l_p1, l_p2, l_norm_out, l_proj_out;
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
  bf16* x_emb_m = nullptr;
  bf16 *ctx_emb_m = nullptr, *proj_out_m = nullptr;
  // ---- geometry
  bool prepared = false;
  int batch = 0, n_txt = 0, n_img = 0, n_cond = 0, N = 0, n_main = 0;
  int flags = 0;
  int attn_cond_mode = 0;
  float attn_cond_bias = 0.f;
  float *rope_cos = nullptr, *rope_sin = nullptr, *crope_cos = nullptr, *crope_sin = nullptr;
  // ---- workspace
  bf16 *X = nullptr, *XN = nullptr, *QKV = nullptr, *ACT = nullptr, *MOD = nullptr, *MODC = nullptr;
  bf16 *LT = nullptr, *LL = nullptr;  // LoRA temporaries: T [lora_rows, 256], L [lora_rows, 4D]
  int lora_rows = 0;
  bf16 *emb_tmp = nullptr;            // small vectors for the temb path
  bf16 *temb = nullptr, *ctemb = nullptr;
  // ---- staging for the graph-captured denoise loop
  bf16 *s_lat = nullptr, *s_txt = nullptr, *s_pooled = nullptr, *s_cond = nullptr, *s_v = nullptr;
  bf16 *s_tsteps = nullptr, *s_guid = nullptr, *s_zero_one = nullptr;
  float* s_sigmas = nullptr;
  int* s_step = nullptr;
  // every step's adaLN modulation vectors, computed BEFORE the loop (all timesteps are known up
  // front): MOD_ALL [n_steps, n_mod]; the captured step only selects its row
  bf16 *s_mod_all = nullptr, *s_temb_ws = nullptr;
  int s_cap_steps = 0;
  cudaGraphExec_t graph_exec = nullptr;
  cudaStream_t own_stream = nullptr;  // capture is illegal on the legacy default stream
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  int64_t graph_kernels = 0;  // kernel launches inside one captured step
  double graph_call_scale = 1.0;  // call_scale the captured step was built with (kernel parameters, launch list)
};

namespace {

// the fp32 scaling peft multiplies the bf16 low-rank term of target t by
float lora_eff(const rf_dit* h, const LoraT& t) { return static_cast<float>(t.scale * h->call_scale); }
// a target whose effective scaling is 0 adds exactly nothing: it runs no launch at all
bool lora_on(const rf_dit* h, const LoraT& t) { return t.set && lora_eff(h, t) != 0.f; }

int dev_alloc(rf_dit* h, void** p, size_t bytes, bool geometry = false) {
  RF_CHECK_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  (geometry ? h->geo_allocs : h->allocs).push_back(*p);
  return 0;
}

struct Arena {
  rf_dit* h;
  int fail = 0;
  bf16* take(int64_t numel) {
    void* p = nullptr;
    if (dev_alloc(h, &p, static_cast<size_t>(numel) * 2)) fail = -2;
    return static_cast<bf16*>(p);
  }
};

void reg(rf_dit* h, const std::string& key, bf16* dst, int64_t numel) {
  h->slots[key] = Slot{dst, numel, false};
}

// Linear whose weight/bias may be a row range of a packed matrix
void reg_lin(rf_dit* h, const std::string& mod, bf16* w, bf16* b, int out, int in) {
  reg(h, mod + ".weight", w, static_cast<int64_t>(out) * in);
  reg(h, mod + ".bias", b, out);
}

Lin new_lin(rf_dit* h, Arena& ar, const std::string& mod, int out, int in) {
  Lin l;
  l.w = ar.take(static_cast<int64_t>(out) * in);
  l.b = ar.take(out);
  if (!mod.empty()) reg_lin(h, mod, l.w, l.b, out, in);
  return l;
}

void new_lora(rf_dit* h, Arena& ar, const std::string& mod, LoraT& t, int out, int in,
              bf16* A_view = nullptr, bf16* B_view = nullptr) {
  if (h->cfg.lora_rank <= 0) return;
  t.in = in;
  t.out = out;
  const int pad = h->lora_pad;
  t.A = A_view ? A_view : ar.take(static_cast<int64_t>(pad) * in);
  t.B = B_view ? B_view : ar.take(static_cast<int64_t>(out) * pad);
  // unset targets must contribute exactly zero (a q-only adapter still runs the stacked q|k|v path)
  if (t.A) cudaMemset(t.A, 0, static_cast<size_t>(pad) * in * 2);
  if (t.B) cudaMemset(t.B, 0, static_cast<size_t>(out) * pad * 2);
  h->lora_slots[mod] = &t;
}

// an always target: shape checks now, factor storage on its first rf_dit_set_lora (lora_storage)
void new_always_lora(rf_dit* h, const std::string& mod, LoraT& t, int out, int in) {
  if (h->cfg.lora_rank <= 0) return;
  t.in = in;
  t.out = out;
  t.always = true;
  h->lora_slots[mod] = &t;
}

// zeroed factor storage of target t (of its whole pack), allocated on first use; live until destroy
int lora_storage(rf_dit* h, LoraT& t) {
  if (t.A != nullptr) return 0;
  const int64_t pad = h->lora_pad, n = t.npack ? t.npack : 1;
  const int64_t a_elems = pad * t.in, b_elems = static_cast<int64_t>(t.out) * pad;
  void *pa = nullptr, *pb = nullptr;
  RF_TRY(dev_alloc(h, &pa, static_cast<size_t>(n * a_elems) * 2));
  RF_TRY(dev_alloc(h, &pb, static_cast<size_t>(n * b_elems) * 2));
  RF_CHECK_CUDA(cudaMemset(pa, 0, static_cast<size_t>(n * a_elems) * 2));
  RF_CHECK_CUDA(cudaMemset(pb, 0, static_cast<size_t>(n * b_elems) * 2));
  bf16 *A = static_cast<bf16*>(pa), *B = static_cast<bf16*>(pb);
  if (t.npack == 0) {
    t.A = A;
    t.B = B;
    return 0;
  }
  *t.packA = A;
  *t.packB = B;
  for (int k = 0; k < t.npack; ++k) {
    t.pack[k]->A = A + k * a_elems;
    t.pack[k]->B = B + k * b_elems;
  }
  return 0;
}

int build_storage(rf_dit* h) {
  const rf_dit_config& c = h->cfg;
  const int D = h->D, lpad = h->lora_pad;
  Arena ar{h};
  h->x_emb = new_lin(h, ar, "x_embedder", D, c.in_channels);
  new_lora(h, ar, "x_embedder", h->l_x_emb, D, c.in_channels);
  h->ctx_emb = new_lin(h, ar, "context_embedder", D, c.joint_attention_dim);
  new_always_lora(h, "context_embedder", h->l_ctx, D, c.joint_attention_dim);
  const std::string tte = "time_text_embed.";
  h->t1 = new_lin(h, ar, tte + "timestep_embedder.linear_1", D, 256);
  h->t2 = new_lin(h, ar, tte + "timestep_embedder.linear_2", D, D);
  new_always_lora(h, tte + "timestep_embedder.linear_1", h->l_t1, D, 256);
  new_always_lora(h, tte + "timestep_embedder.linear_2", h->l_t2, D, D);
  if (c.guidance_embeds) {
    h->g1 = new_lin(h, ar, tte + "guidance_embedder.linear_1", D, 256);
    h->g2 = new_lin(h, ar, tte + "guidance_embedder.linear_2", D, D);
    new_always_lora(h, tte + "guidance_embedder.linear_1", h->l_g1, D, 256);
    new_always_lora(h, tte + "guidance_embedder.linear_2", h->l_g2, D, D);
  }
  h->p1 = new_lin(h, ar, tte + "text_embedder.linear_1", D, c.pooled_projection_dim);
  h->p2 = new_lin(h, ar, tte + "text_embedder.linear_2", D, D);
  new_always_lora(h, tte + "text_embedder.linear_1", h->l_p1, D, c.pooled_projection_dim);
  new_always_lora(h, tte + "text_embedder.linear_2", h->l_p2, D, D);
  h->proj_out = new_lin(h, ar, "proj_out", c.in_channels, D);
  new_always_lora(h, "proj_out", h->l_proj_out, c.in_channels, D);

  h->n_mod = static_cast<int64_t>(c.num_layers) * 12 * D +
             static_cast<int64_t>(c.num_single_layers) * 3 * D + 2 * D;
  h->modW = ar.take(h->n_mod * D);
  h->modB = ar.take(h->n_mod);

  h->dbl.resize(c.num_layers);
  for (int i = 0; i < c.num_layers; ++i) {
    DoubleBlk& b = h->dbl[i];
    const std::string p = "transformer_blocks." + std::to_string(i) + ".";
    const int64_t mo = static_cast<int64_t>(i) * 12 * D;
    reg_lin(h, p + "norm1.linear", h->modW + mo * D, h->modB + mo, 6 * D, D);
    reg_lin(h, p + "norm1_context.linear", h->modW + (mo + 6 * D) * D, h->modB + mo + 6 * D, 6 * D, D);
    new_lora(h, ar, p + "norm1.linear", b.l_norm1, 6 * D, D);
    new_always_lora(h, p + "norm1_context.linear", b.l_norm1c, 6 * D, D);
    b.qkv = new_lin(h, ar, "", 3 * D, D);
    b.add_qkv = new_lin(h, ar, "", 3 * D, D);
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    const char* an[3] = {"add_q_proj", "add_k_proj", "add_v_proj"};
    if (c.lora_rank > 0) {
      b.qkvA = ar.take(static_cast<int64_t>(3 * lpad) * D);
      b.qkvB = ar.take(static_cast<int64_t>(3 * D) * lpad);
    }
    LoraT* lq[3] = {&b.l_q, &b.l_k, &b.l_v};
    LoraT* la[3] = {&b.l_aq, &b.l_ak, &b.l_av};
    for (int j = 0; j < 3; ++j) {
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
      reg_lin(h, p + "attn." + an[j], b.add_qkv.w + static_cast<int64_t>(j) * D * D,
              b.add_qkv.b + j * D, D, D);
      new_lora(h, ar, p + "attn." + nm[j], *lq[j], D, D,
               b.qkvA ? b.qkvA + static_cast<int64_t>(j) * lpad * D : nullptr,
               b.qkvB ? b.qkvB + static_cast<int64_t>(j) * D * lpad : nullptr);
      new_always_lora(h, p + "attn." + an[j], *la[j], D, D);
      la[j]->npack = 3;
      la[j]->packA = &b.add_qkvA;
      la[j]->packB = &b.add_qkvB;
      for (int k = 0; k < 3; ++k) la[j]->pack[k] = la[k];
    }
    b.norm_q = ar.take(128); reg(h, p + "attn.norm_q.weight", b.norm_q, 128);
    b.norm_k = ar.take(128); reg(h, p + "attn.norm_k.weight", b.norm_k, 128);
    b.norm_added_q = ar.take(128); reg(h, p + "attn.norm_added_q.weight", b.norm_added_q, 128);
    b.norm_added_k = ar.take(128); reg(h, p + "attn.norm_added_k.weight", b.norm_added_k, 128);
    b.to_out = new_lin(h, ar, p + "attn.to_out.0", D, D);
    new_lora(h, ar, p + "attn.to_out.0", b.l_out, D, D);
    b.to_add_out = new_lin(h, ar, p + "attn.to_add_out", D, D);
    new_always_lora(h, p + "attn.to_add_out", b.l_add_out, D, D);
    b.ff1 = new_lin(h, ar, p + "ff.net.0.proj", 4 * D, D);
    new_always_lora(h, p + "ff.net.0.proj", b.l_ff1, 4 * D, D);
    b.ff2 = new_lin(h, ar, p + "ff.net.2", D, 4 * D);
    new_lora(h, ar, p + "ff.net.2", b.l_ff2, D, 4 * D);
    b.ffc1 = new_lin(h, ar, p + "ff_context.net.0.proj", 4 * D, D);
    b.ffc2 = new_lin(h, ar, p + "ff_context.net.2", D, 4 * D);
    new_always_lora(h, p + "ff_context.net.0.proj", b.l_ffc1, 4 * D, D);
    new_always_lora(h, p + "ff_context.net.2", b.l_ffc2, D, 4 * D);
  }
  h->sgl.resize(c.num_single_layers);
  const int64_t so = static_cast<int64_t>(c.num_layers) * 12 * D;
  for (int i = 0; i < c.num_single_layers; ++i) {
    SingleBlk& b = h->sgl[i];
    const std::string p = "single_transformer_blocks." + std::to_string(i) + ".";
    const int64_t mo = so + static_cast<int64_t>(i) * 3 * D;
    reg_lin(h, p + "norm.linear", h->modW + mo * D, h->modB + mo, 3 * D, D);
    new_lora(h, ar, p + "norm.linear", b.l_norm, 3 * D, D);
    b.qkv = new_lin(h, ar, "", 3 * D, D);
    if (c.lora_rank > 0) {
      // A factors of to_q | to_k | to_v | proj_mlp stacked: all four read the same normalised tokens, so
      // ONE down-projection launch (NT = 256) serves the q|k|v and the MLP-in GEMMs of the block
      b.qkvA = ar.take(static_cast<int64_t>(4 * lpad) * D);
      b.qkvB = ar.take(static_cast<int64_t>(3 * D) * lpad);
    }
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    LoraT* lq[3] = {&b.l_q, &b.l_k, &b.l_v};
    for (int j = 0; j < 3; ++j) {
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
      new_lora(h, ar, p + "attn." + nm[j], *lq[j], D, D,
               b.qkvA ? b.qkvA + static_cast<int64_t>(j) * lpad * D : nullptr,
               b.qkvB ? b.qkvB + static_cast<int64_t>(j) * D * lpad : nullptr);
    }
    b.norm_q = ar.take(128); reg(h, p + "attn.norm_q.weight", b.norm_q, 128);
    b.norm_k = ar.take(128); reg(h, p + "attn.norm_k.weight", b.norm_k, 128);
    b.mlp = new_lin(h, ar, p + "proj_mlp", 4 * D, D);
    new_lora(h, ar, p + "proj_mlp", b.l_mlp, 4 * D, D,
             b.qkvA ? b.qkvA + static_cast<int64_t>(3 * lpad) * D : nullptr);
    b.out = new_lin(h, ar, p + "proj_out", D, 5 * D);
    new_lora(h, ar, p + "proj_out", b.l_out, D, 5 * D);
  }
  const int64_t oo = so + static_cast<int64_t>(c.num_single_layers) * 3 * D;
  reg_lin(h, "norm_out.linear", h->modW + oo * D, h->modB + oo, 2 * D, D);
  new_always_lora(h, "norm_out.linear", h->l_norm_out, 2 * D, D);
  return ar.fail;
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
  RF_TRY(rf::gemv_launch(x, ldx, batch, t.A, nullptr, tvec, lpad, lpad, t.in, act, s));
  RF_TRY(rf::gemv_launch(tvec, lpad, batch, t.B, nullptr, lvec, t.out, t.out, lpad, 0, s));
  return rf::add_rows_launch(y, ldy, lvec, t.out, batch, t.out, lora_eff(h, t), s);
}

// y = linear_2(silu(linear_1(x)))  (TimestepEmbedding / PixArtAlphaTextProjection) for `batch` vectors, each Linear
// with its LoRA term (always targets): linear_2's sees the same bf16(silu(.)) input as its GEMV.
// tvec [batch, lora_pad], lvec [batch, D] scratch.
int mlp2(rf_dit* h, const bf16* x, int in_dim, int batch, const Lin& l1, const LoraT& lt1, const Lin& l2,
         const LoraT& lt2, bf16* tmp, bf16* out, bf16* tvec, bf16* lvec, cudaStream_t s) {
  const int D = h->D;
  RF_TRY(rf::gemv_launch(x, in_dim, batch, l1.w, l1.b, tmp, D, D, in_dim, 0, s));
  RF_TRY(add_vec_lora(h, lt1, x, in_dim, batch, 0, tmp, D, tvec, lvec, s));
  RF_TRY(rf::gemv_launch(tmp, D, batch, l2.w, l2.b, out, D, D, D, 1, s));
  return add_vec_lora(h, lt2, tmp, D, batch, 1, out, D, tvec, lvec, s);
}

// temb = time(t) + guidance(g) + text(pooled)   (CombinedTimestepGuidanceTextProjEmbeddings)
int compute_temb(rf_dit* h, const bf16* t, const int* step, const bf16* guid, const bf16* pooled,
                 bf16* out, cudaStream_t s) {
  const int D = h->D;
  bf16* e = h->emb_tmp;  // [256 | 256 | D tmp | D a | D b | D c]
  bf16 *tp = e, *gp = e + 256, *tmp = e + 512, *a = tmp + D, *b = a + D, *c = b + D;
  bf16 *tvec = h->LT, *lvec = h->LT + 256;  // embedder LoRA scratch: [lora_pad] | [D] (LT holds >= 8D)
  RF_TRY(rf::timestep_embed_launch(t, step, 1, 1000.0f, tp, 1, s));
  RF_TRY(mlp2(h, tp, 256, 1, h->t1, h->l_t1, h->t2, h->l_t2, tmp, a, tvec, lvec, s));
  RF_TRY(mlp2(h, pooled, h->cfg.pooled_projection_dim, 1, h->p1, h->l_p1, h->p2, h->l_p2, tmp, c, tvec, lvec, s));
  if (h->cfg.guidance_embeds) {
    RF_TRY(rf::timestep_embed_launch(guid, nullptr, 1, 1000.0f, gp, 1, s));
    RF_TRY(mlp2(h, gp, 256, 1, h->g1, h->l_g1, h->g2, h->l_g2, tmp, b, tvec, lvec, s));
    RF_TRY(rf::add3_launch(a, b, c, out, D, s));
  } else {
    RF_TRY(rf::add2_launch(a, c, out, D, s));
  }
  return 0;
}

// L[rows, :] = bf16( bf16(x A^T) B^T ): the unfused peft low-rank term of `rows` tokens for n = 1 target, or for
// the n = 3 stacked q|k|v targets (A_all = [Aq;Ak;Av]: T = x A_all^T in one GEMM, L[:, jD:(j+1)D] = T_j B_j^T
// grouped).  T != nullptr: bf16(x A_all^T) of these rows was already computed (pitch ld_t); only the up-projection
// runs.  Otherwise T is computed here into LT.
int lora_term(rf_dit* h, const LoraT* const* ls, int n, const bf16* A_all, const bf16* x, int ldx, int rows,
              const bf16* T, int ld_t, bf16* L, int ldl, cudaStream_t s) {
  const int lpad = h->lora_pad;
  rf::GemmGroupArgs g[3];
  if (T == nullptr) {
    memset(g, 0, sizeof(g));
    g[0].A = x; g[0].lda = ldx; g[0].M = rows; g[0].W = A_all; g[0].out = h->LT; g[0].ldo = n * lpad;
    RF_TRY(rf::gemm_launch(rf::EPI_BIAS, n * lpad, ls[0]->in, 1, g, s));
    T = h->LT;
    ld_t = n * lpad;
  }
  memset(g, 0, sizeof(g));
  bool scaled = false;  // peft's bf16(bf16(T B^T) * scaling): the scale is the up-projection's output scale
  for (int j = 0; j < n; ++j) {
    g[j].A = T + j * lpad; g[j].lda = ld_t; g[j].M = rows;
    g[j].W = ls[j]->B; g[j].out = L + static_cast<int64_t>(j) * ls[j]->out; g[j].ldo = ldl;
    g[j].lora_scale[0] = lora_eff(h, *ls[j]);
    scaled |= g[j].lora_scale[0] != 1.f;
  }
  return rf::gemm_launch(scaled ? rf::EPI_SCALE : rf::EPI_BIAS, ls[0]->out, lpad, n, g, s);
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
  auto one = [&](const LoraT& t, int64_t off) {
    return add_vec_lora(h, t, emb, D, batch, 1, mod + off, ld_mod, tvec, lvec, s);
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

// cond_temb and MODC: step-invariant (transformer.py:108-114 recomputes them every step)
int compute_cond_mod(rf_dit* h, const bf16* pooled, cudaStream_t s) {
  const int D = h->D;
  // t = c_t * 1000 = 0, guidance = 1000 (s_zero_one = {bf16 0, bf16 1})
  RF_TRY(compute_temb(h, h->s_zero_one, nullptr, h->s_zero_one + 1, pooled, h->ctemb, s));
  RF_TRY(rf::gemv_launch(h->ctemb, D, 1, h->modW, h->modB, h->MODC, static_cast<int>(h->n_mod),
                         static_cast<int>(h->n_mod), D, 1, s));
  if (!h->any_lora) return 0;
  // LoRA of norm1.linear / norm.linear acts on silu(cond_temb); tvec [1, lora_pad <= 256] at the front of LT.  (The
  // condition rows read no norm1_context / norm_out section of MODC.)
  return add_mod_lora(h, h->ctemb, 1, true, false, h->MODC, h->n_mod, h->LT, h->LT + 256, s);
}

// fuse_lora mode: merged weights for the condition-token groups (allocated on first use)
int merge_one(rf_dit* h, const LoraT& t, const bf16* W, bf16** Wm, int rows_off, int out_total,
              cudaStream_t s) {
  // target occupies rows [rows_off, rows_off + t.out) of a packed [out_total, t.in] matrix
  if (*Wm == nullptr) {
    void* p = nullptr;
    if (dev_alloc(h, &p, static_cast<size_t>(out_total) * t.in * 2)) return -2;
    *Wm = static_cast<bf16*>(p);
  }
  const size_t off = static_cast<size_t>(rows_off) * t.in;
  if (!t.set) {  // no adapter on this target: the merged copy is the (possibly reloaded) base weight
    RF_CHECK_CUDA(cudaMemcpyAsync(*Wm + off, W + off, static_cast<size_t>(t.out) * t.in * 2,
                                  cudaMemcpyDeviceToDevice, s));
    return 0;
  }
  return rf::lora_merge_launch(W + off, t.A, t.B, *Wm + off, t.out, t.in, h->lora_pad, lora_eff(h, t), s);
}
// an always target (or pack) has a merged copy only once one of its targets is set; until then its groups read the
// base weight (any_set), so a handle without such adapters allocates nothing here
bool any_set(const LoraT* const* ls, int n) {
  for (int k = 0; k < n; ++k)
    if (ls[k]->set) return true;
  return false;
}
int merge_always(rf_dit* h, const LoraT* const* ls, int n, const bf16* W, bf16** Wm, cudaStream_t s) {
  if (!any_set(ls, n)) return 0;
  for (int k = 0; k < n; ++k) RF_TRY(merge_one(h, *ls[k], W, Wm, k * ls[k]->out, n * ls[k]->out, s));
  return 0;
}
int merge_all(rf_dit* h, cudaStream_t s) {
  const int D = h->D;
  RF_TRY(merge_one(h, h->l_x_emb, h->x_emb.w, &h->x_emb_m, 0, D, s));
  const LoraT* lctx = &h->l_ctx;
  const LoraT* lpo = &h->l_proj_out;
  RF_TRY(merge_always(h, &lctx, 1, h->ctx_emb.w, &h->ctx_emb_m, s));
  RF_TRY(merge_always(h, &lpo, 1, h->proj_out.w, &h->proj_out_m, s));
  for (auto& b : h->dbl) {
    RF_TRY(merge_one(h, b.l_q, b.qkv.w, &b.qkv_m, 0, 3 * D, s));
    RF_TRY(merge_one(h, b.l_k, b.qkv.w, &b.qkv_m, D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_v, b.qkv.w, &b.qkv_m, 2 * D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_out, b.to_out.w, &b.to_out_m, 0, D, s));
    RF_TRY(merge_one(h, b.l_ff2, b.ff2.w, &b.ff2_m, 0, D, s));
    const LoraT* la[3] = {&b.l_aq, &b.l_ak, &b.l_av};
    const LoraT *lao = &b.l_add_out, *lf1 = &b.l_ff1, *lc1 = &b.l_ffc1, *lc2 = &b.l_ffc2;
    RF_TRY(merge_always(h, la, 3, b.add_qkv.w, &b.add_qkv_m, s));
    RF_TRY(merge_always(h, &lao, 1, b.to_add_out.w, &b.to_add_out_m, s));
    RF_TRY(merge_always(h, &lf1, 1, b.ff1.w, &b.ff1_m, s));
    RF_TRY(merge_always(h, &lc1, 1, b.ffc1.w, &b.ffc1_m, s));
    RF_TRY(merge_always(h, &lc2, 1, b.ffc2.w, &b.ffc2_m, s));
  }
  for (auto& b : h->sgl) {
    RF_TRY(merge_one(h, b.l_q, b.qkv.w, &b.qkv_m, 0, 3 * D, s));
    RF_TRY(merge_one(h, b.l_k, b.qkv.w, &b.qkv_m, D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_v, b.qkv.w, &b.qkv_m, 2 * D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_mlp, b.mlp.w, &b.mlp_m, 0, 4 * D, s));
    RF_TRY(merge_one(h, b.l_out, b.out.w, &b.out_m, 0, D, s));
  }
  h->lora_merged = true;
  h->merged_call_scale = h->call_scale;
  return 0;
}

// temb_i = time(t_i) + guidance(g) + text(pooled) for ALL steps, then every adaLN Linear of every
// block for all steps: the 6.5 GB modulation weight stack is streamed ceil(n/8) times per denoise
// call instead of once per step.  Same kernels, same per-vector arithmetic as compute_temb + gemv
// (the GEMV's per-vector summation order does not depend on the batch width): bit-identical.
int precompute_step_mods(rf_dit* h, int n_steps, const bf16* tsteps, const bf16* guid,
                         const bf16* pooled, cudaStream_t s) {
  const int D = h->D;
  // [n,256] | [n,D] tmp | [n,D] a | [n,D] temb | [256] gp | [D] tmp1 | [D] b | [D] c | [n,lora_pad] | [n,6D] (LoRA)
  bf16* ws = h->s_temb_ws;
  bf16* tp = ws;
  bf16* tmp = tp + static_cast<int64_t>(n_steps) * 256;
  bf16* a = tmp + static_cast<int64_t>(n_steps) * D;
  bf16* temb = a + static_cast<int64_t>(n_steps) * D;
  bf16* gp = temb + static_cast<int64_t>(n_steps) * D;
  bf16 *tmp1 = gp + 256, *b = tmp1 + D, *c = b + D;
  bf16* tvec = c + D;                                               // [n, lora_pad]
  bf16* lvec = tvec + static_cast<int64_t>(n_steps) * h->lora_pad;  // [n, 6D]
  RF_TRY(rf::timestep_embed_launch(tsteps, nullptr, 1, 1000.0f, tp, n_steps, s));
  // the timestep embedder and its LoRA terms batched over every step, like compute_temb per vector
  RF_TRY(mlp2(h, tp, 256, n_steps, h->t1, h->l_t1, h->t2, h->l_t2, tmp, a, tvec, lvec, s));
  RF_TRY(mlp2(h, pooled, h->cfg.pooled_projection_dim, 1, h->p1, h->l_p1, h->p2, h->l_p2, tmp1, c, tvec, lvec, s));
  if (h->cfg.guidance_embeds) {
    RF_TRY(rf::timestep_embed_launch(guid, nullptr, 1, 1000.0f, gp, 1, s));
    RF_TRY(mlp2(h, gp, 256, 1, h->g1, h->l_g1, h->g2, h->l_g2, tmp1, b, tvec, lvec, s));
  }
  for (int i = 0; i < n_steps; ++i) {
    bf16* ai = a + static_cast<int64_t>(i) * D;
    bf16* ti = temb + static_cast<int64_t>(i) * D;
    if (h->cfg.guidance_embeds) RF_TRY(rf::add3_launch(ai, b, c, ti, D, s));
    else RF_TRY(rf::add2_launch(ai, c, ti, D, s));
  }
  RF_TRY(rf::gemv_launch(temb, D, n_steps, h->modW, h->modB, h->s_mod_all, static_cast<int>(h->n_mod),
                         static_cast<int>(h->n_mod), D, 1, s));
  // the adaLN LoRA terms act on silu(temb_i), which every step knows before the loop: they join the table here too
  // (latent_lora: the image stream of the double blocks / the txt+img rows of the single blocks; always:
  // norm1_context and norm_out)
  if (h->any_lora) RF_TRY(add_mod_lora(h, temb, n_steps, (h->flags & 1) != 0, true, h->s_mod_all, h->n_mod, tvec,
                                       lvec, s));
  return 0;
}

struct StreamRows {
  int row0, rows;
};

// The body of one DiT forward for one sample.  All pointers are device pointers.
int enqueue_forward(rf_dit* h, const bf16* latents, const bf16* txt, const bf16* pooled,
                    const bf16* tstep, const int* step_idx, const bf16* guid, const bf16* cond_lat,
                    bf16* out, cudaStream_t s, const bf16* mod_all = nullptr) {
  const int D = h->D, D3 = 3 * D, D4 = 4 * D, D5 = 5 * D, lpad = h->lora_pad;
  const bool use_cond = h->n_cond > 0;
  // latent_lora (lora_controller.py:5-9): the LoRA also acts on the image stream of the double blocks and on the
  // txt + img rows of the single blocks (the text stream of the double blocks has no LoRA target)
  const bool ll = (h->flags & 1) != 0;
  const StreamRows S_txt{0, h->n_txt}, S_img{h->n_txt, h->n_img}, S_cond{h->n_main, h->n_cond};
  bf16 *X = h->X, *XN = h->XN, *QKV = h->QKV, *ACT = h->ACT;
  auto rowp = [&](bf16* base, int ld, int row) { return base + static_cast<int64_t>(row) * ld; };
  rf::GemmGroupArgs g[3];

  // ---- embedders (transformer.py:91-93,115)
  memset(g, 0, sizeof(g));
  g[0].A = latents; g[0].lda = h->cfg.in_channels; g[0].M = h->n_img; g[0].W = h->x_emb.w;
  g[0].bias = h->x_emb.b; g[0].out = rowp(X, D, S_img.row0); g[0].ldo = D;
  int ng = 1;
  if (use_cond) {
    g[1] = g[0];
    g[1].A = cond_lat; g[1].M = h->n_cond; g[1].out = rowp(X, D, S_cond.row0);
    ng = 2;
  }
  if (h->use_merged) {
    if (ll) g[0].W = h->x_emb_m;
    if (use_cond) g[1].W = h->x_emb_m;
  } else if (lora_on(h, h->l_x_emb)) {
    // K = 64, EPI_BIAS: the unfused low-rank term, each LoRA'd group's L in its own rows of LL
    const LoraT* xl = &h->l_x_emb;
    int row = 0;
    for (int j = ll ? 0 : 1; j < ng; ++j) {
      bf16* L = rowp(h->LL, D, row);
      RF_TRY(lora_term(h, &xl, 1, xl->A, g[j].A, g[j].lda, g[j].M, nullptr, 0, L, D, s));
      g[j].addend = L; g[j].ldadd = D;
      row += g[j].M;
    }
  }
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, D, h->cfg.in_channels, ng, g, s));
  memset(g, 0, sizeof(g));
  g[0].A = txt; g[0].lda = h->cfg.joint_attention_dim; g[0].M = h->n_txt; g[0].W = h->ctx_emb.w;
  g[0].bias = h->ctx_emb.b; g[0].out = rowp(X, D, 0); g[0].ldo = D;
  // context_embedder (always target; EPI_BIAS, K = 4096): the unfused term, like x_embedder's
  const LoraT* lctx = &h->l_ctx;
  if (h->use_merged) {
    if (lctx->set) g[0].W = h->ctx_emb_m;
  } else if (lora_on(h, *lctx)) {
    RF_TRY(lora_term(h, &lctx, 1, lctx->A, txt, g[0].lda, g[0].M, nullptr, 0, h->LL, D, s));
    g[0].addend = h->LL; g[0].ldadd = D;
  }
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, D, h->cfg.joint_attention_dim, 1, g, s));

  // ---- temb and every modulation vector of the step (transformer.py:95-107 + all adaLN linears)
  if (mod_all != nullptr) {  // denoise loop: this step's row of the precomputed table
    RF_TRY(rf::select_row_launch(mod_all, h->n_mod, step_idx, h->MOD, s));
  } else {
    RF_TRY(compute_temb(h, tstep, step_idx, guid, pooled, h->temb, s));
    RF_TRY(rf::gemv_launch(h->temb, D, 1, h->modW, h->modB, h->MOD, static_cast<int>(h->n_mod),
                           static_cast<int>(h->n_mod), D, 1, s));
    if (h->any_lora) RF_TRY(add_mod_lora(h, h->temb, 1, ll, true, h->MOD, h->n_mod, h->LT, h->LT + 256, s));
  }
  const bf16* MOD = h->MOD;
  const bf16* MODC = h->MODC;

  auto ln = [&](const StreamRows& sr, const bf16* scale, const bf16* shift) {
    return rf::ln_modulate_launch(rowp(X, D, sr.row0), D, rowp(XN, D, sr.row0), D, sr.rows, D, scale,
                                  shift, sr.rows, 0, s);
  };
  // The groups of a projection launch that carry the LoRA in exact mode, in row order, each with its target(s) `ls`
  // and stacked factors A_all / B_all: in the double blocks the text group (its own add_* / to_add_out / ff_context
  // targets, always on), the image group (under latent_lora; always for ff.net.0.proj), the condition group; in the
  // single blocks the txt + img group under latent_lora, then the condition group.  `row` is each group's row in
  // LT / LL: groups are stacked there in this order.
  struct LoraGrp {
    int idx, row;
    const LoraT* const* ls;
    const bf16 *A_all, *B_all;
  };
  struct LoraGroups {
    int n = 0, rows = 0;
    LoraGrp e[3];
    void add(int i, int m, const LoraT* const* ls, const bf16* A_all, const bf16* B_all) {
      e[n] = LoraGrp{i, rows, ls, A_all, B_all};
      rows += m;
      ++n;
    }
  };
  // on: the target(s) of the image (double) / main (single) and condition groups add a term; main_always: the image
  // group carries it whatever latent_lora says (ff.net.0.proj)
  auto lora_groups = [&](bool on, int main_idx, int main_rows, int cond_idx, const LoraT* const* ls,
                         const bf16* A_all, const bf16* B_all, bool main_always = false) {
    LoraGroups lg;
    if (!on || h->use_merged) return lg;
    if (ll || main_always) lg.add(main_idx, main_rows, ls, A_all, B_all);
    if (use_cond) lg.add(cond_idx, h->n_cond, ls, A_all, B_all);
    return lg;
  };
  // the double blocks: the text group (always targets) first, then the image / condition groups
  auto lora_groups_dbl = [&](bool txt_on, const LoraT* const* txt_ls, const bf16* txt_A, const bf16* txt_B,
                             bool on, const LoraT* const* ls, const bf16* A_all, const bf16* B_all,
                             bool main_always = false) {
    LoraGroups lg;
    if (h->use_merged) return lg;
    if (txt_on) lg.add(1, h->n_txt, txt_ls, txt_A, txt_B);
    if (on && (ll || main_always)) lg.add(0, h->n_img, ls, A_all, B_all);
    if (on && use_cond) lg.add(2, h->n_cond, ls, A_all, B_all);
    return lg;
  };
  // merged mode (fuse_lora): the same groups read the merged weights W + B A instead
  auto merged_w = [&](rf::GemmGroupArgs* gr, int main_idx, int cond_idx, const bf16* Wm, bool main_always = false) {
    if (!h->use_merged) return;
    if (ll || main_always) gr[main_idx].W = Wm;
    if (use_cond) gr[cond_idx].W = Wm;
  };
  // A grouped GEMM in which the groups `lg` carry their LoRA (nls = 1 target each, or 3 stacked q|k|v targets).
  // Fast path: T = bf16(x A^T) for all LoRA'd rows in one skinny grouped GEMM (one group per run of rows that are
  // contiguous in the A operand and share their A factors), then ONE grouped launch of all streams in which the
  // eligible groups' tiles carry the low-rank k-block (GemmGroupArgs::lora_T) — L = T B^T never reaches HBM.  Groups
  // too small for it (gemm_lora_eligible) keep the unfused path: L materialised in their rows of LL and added in the
  // epilogue (`addend`); they reuse T when it exists.  (t_pre != nullptr: T was already produced by an earlier
  // launch, [rows, ld_t] with this target's columns at t_pre.)
  auto gemm_lora = [&](int epi, int N, int K, int ngr, rf::GemmGroupArgs* gr, const LoraGroups& lg, int nls,
                       int ldl, const bf16* t_pre = nullptr, int ld_t = 0) -> int {
    bool fused[3] = {false, false, false}, any_fused = false;
    for (int j = 0; j < lg.n; ++j) any_fused |= (fused[j] = rf::gemm_lora_eligible(epi, N, K, gr[lg.e[j].idx]));
    if (any_fused && t_pre == nullptr) {
      ld_t = nls * lpad;
      rf::GemmGroupArgs dg[3];
      memset(dg, 0, sizeof(dg));
      int nd = 0;
      for (int j = 0; j < lg.n; ++j) {
        const rf::GemmGroupArgs& gc = gr[lg.e[j].idx];
        rf::GemmGroupArgs* last = nd ? &dg[nd - 1] : nullptr;
        if (last && last->W == lg.e[j].A_all && last->lda == gc.lda &&
            gc.A == last->A + static_cast<int64_t>(last->M) * last->lda) {
          last->M += gc.M;
          continue;
        }
        dg[nd].A = gc.A; dg[nd].lda = gc.lda; dg[nd].M = gc.M; dg[nd].W = lg.e[j].A_all;
        dg[nd].out = h->LT + static_cast<int64_t>(lg.e[j].row) * ld_t; dg[nd].ldo = ld_t;
        ++nd;
      }
      RF_TRY(rf::lora_down_launch(K, ld_t, nd, dg, s));
      t_pre = h->LT;
    }
    for (int j = 0; j < lg.n; ++j) {
      const LoraGrp& e = lg.e[j];
      rf::GemmGroupArgs& gc = gr[e.idx];
      const bf16* t_rows = t_pre ? t_pre + static_cast<int64_t>(e.row) * ld_t : nullptr;
      if (fused[j]) {
        gc.lora_T = t_rows; gc.ld_t = ld_t; gc.lora_B = e.B_all; gc.lora_sec_cols = nls > 1 ? e.ls[0]->out : 0;
        gc.lora_pad = lpad;
        for (int k = 0; k < nls; ++k) gc.lora_scale[k] = lora_eff(h, *e.ls[k]);
      } else {
        bf16* L = rowp(h->LL, ldl, e.row);
        RF_TRY(lora_term(h, e.ls, nls, e.A_all, gc.A, gc.lda, gc.M, t_rows, ld_t, L, ldl, s));
        gc.addend = L; gc.ldadd = ldl;
      }
    }
    return rf::gemm_launch(epi, N, K, ngr, gr, s);
  };
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
  for (int i = 0; i < h->cfg.num_layers; ++i) {
    const DoubleBlk& b = h->dbl[i];
    const bf16* mi = MOD + mod_double(h, i, 0, 0);
    const bf16* mt = MOD + mod_double(h, i, 1, 0);
    const bf16* mc = MODC + mod_double(h, i, 0, 0);
    // norm1 / norm1_context
    RF_TRY(ln3(mt + SCALE_MSA * D, mt + SHIFT_MSA * D, mi + SCALE_MSA * D, mi + SHIFT_MSA * D,
               mc + SCALE_MSA * D, mc + SHIFT_MSA * D));
    // q|k|v projections + RMSNorm + RoPE, all streams in one grouped launch
    memset(g, 0, sizeof(g));
    g[0].A = rowp(XN, D, S_img.row0); g[0].lda = D; g[0].M = S_img.rows; g[0].W = b.qkv.w;
    g[0].bias = b.qkv.b; g[0].out = rowp(QKV, D3, S_img.row0); g[0].ldo = D3;
    g[0].rope_cos = h->rope_cos + static_cast<int64_t>(S_img.row0) * 64;
    g[0].rope_sin = h->rope_sin + static_cast<int64_t>(S_img.row0) * 64;
    g[0].norm_q = b.norm_q; g[0].norm_k = b.norm_k;
    g[1].A = rowp(XN, D, 0); g[1].lda = D; g[1].M = S_txt.rows; g[1].W = b.add_qkv.w;
    g[1].bias = b.add_qkv.b; g[1].out = rowp(QKV, D3, 0); g[1].ldo = D3;
    g[1].rope_cos = h->rope_cos; g[1].rope_sin = h->rope_sin;
    g[1].norm_q = b.norm_added_q; g[1].norm_k = b.norm_added_k;
    ng = 2;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(XN, D, S_cond.row0); g[2].M = S_cond.rows;
      g[2].out = rowp(QKV, D3, S_cond.row0);
      g[2].rope_cos = h->crope_cos; g[2].rope_sin = h->crope_sin;
      ng = 3;
    }
    merged_w(g, 0, 2, b.qkv_m);
    const LoraT* dqkv[3] = {&b.l_q, &b.l_k, &b.l_v};
    const LoraT* dadd[3] = {&b.l_aq, &b.l_ak, &b.l_av};
    if (h->use_merged && any_set(dadd, 3)) g[1].W = b.add_qkv_m;
    LoraGroups lg = lora_groups_dbl(lora_on(h, b.l_aq) || lora_on(h, b.l_ak) || lora_on(h, b.l_av), dadd,
                                    b.add_qkvA, b.add_qkvB,
                                    lora_on(h, b.l_q) || lora_on(h, b.l_k) || lora_on(h, b.l_v), dqkv, b.qkvA,
                                    b.qkvB);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_QKV, D3, D, ng, g, lg, 3, D3));
    else RF_TRY(rf::gemm_launch(rf::EPI_QKV, D3, D, ng, g, s));
    // joint attention -> ACT[:, 0:D]
    at.out = ACT; at.ldo = D5;
    RF_TRY(rf::attention_launch(at, s));
    // out projections + gate + residual (in place on X)
    memset(g, 0, sizeof(g));
    g[0].A = rowp(ACT, D5, S_img.row0); g[0].lda = D5; g[0].M = S_img.rows; g[0].W = b.to_out.w;
    g[0].bias = b.to_out.b; g[0].out = rowp(X, D, S_img.row0); g[0].ldo = D;
    g[0].res = g[0].out; g[0].ldr = D; g[0].gate = mi + GATE_MSA * D;
    g[1].A = rowp(ACT, D5, 0); g[1].lda = D5; g[1].M = S_txt.rows; g[1].W = b.to_add_out.w;
    g[1].bias = b.to_add_out.b; g[1].out = rowp(X, D, 0); g[1].ldo = D;
    g[1].res = g[1].out; g[1].ldr = D; g[1].gate = mt + GATE_MSA * D;
    ng = 2;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(ACT, D5, S_cond.row0); g[2].M = S_cond.rows;
      g[2].out = rowp(X, D, S_cond.row0); g[2].res = g[2].out; g[2].gate = mc + GATE_MSA * D;
      ng = 3;
    }
    merged_w(g, 0, 2, b.to_out_m);
    const LoraT* dout = &b.l_out;
    const LoraT* dadd_out = &b.l_add_out;
    if (h->use_merged && b.l_add_out.set) g[1].W = b.to_add_out_m;
    lg = lora_groups_dbl(lora_on(h, b.l_add_out), &dadd_out, b.l_add_out.A, b.l_add_out.B, lora_on(h, b.l_out),
                         &dout, b.l_out.A, b.l_out.B);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_GATE_RES, D, D, ng, g, lg, 1, D));
    else RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D, ng, g, s));
    // norm2 + modulate
    RF_TRY(ln3(mt + SCALE_MLP * D, mt + SHIFT_MLP * D, mi + SCALE_MLP * D, mi + SHIFT_MLP * D,
               mc + SCALE_MLP * D, mc + SHIFT_MLP * D));
    // MLP in (GELU-tanh) -> ACT[:, D:5D]
    memset(g, 0, sizeof(g));
    g[0].A = rowp(XN, D, S_img.row0); g[0].lda = D; g[0].M = S_img.rows; g[0].W = b.ff1.w;
    g[0].bias = b.ff1.b; g[0].out = rowp(ACT, D5, S_img.row0) + D; g[0].ldo = D5;
    g[1] = g[0];
    g[1].A = rowp(XN, D, 0); g[1].M = S_txt.rows; g[1].W = b.ffc1.w; g[1].bias = b.ffc1.b;
    g[1].out = rowp(ACT, D5, 0) + D;
    ng = 2;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(XN, D, S_cond.row0); g[2].M = S_cond.rows;
      g[2].out = rowp(ACT, D5, S_cond.row0) + D;
      ng = 3;
    }
    // ff.net.0.proj is inside no enable_lora (block.py:250 names ff.net[2] only): its image rows always carry it
    if (b.l_ff1.set) merged_w(g, 0, 2, b.ff1_m, true);
    if (h->use_merged && b.l_ffc1.set) g[1].W = b.ffc1_m;
    const LoraT* dff1 = &b.l_ff1;
    const LoraT* dffc1 = &b.l_ffc1;
    lg = lora_groups_dbl(lora_on(h, b.l_ffc1), &dffc1, b.l_ffc1.A, b.l_ffc1.B, lora_on(h, b.l_ff1), &dff1,
                         b.l_ff1.A, b.l_ff1.B, true);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_GELU, D4, D, ng, g, lg, 1, D4));
    else RF_TRY(rf::gemm_launch(rf::EPI_GELU, D4, D, ng, g, s));
    // MLP out + gate + residual
    memset(g, 0, sizeof(g));
    g[0].A = rowp(ACT, D5, S_img.row0) + D; g[0].lda = D5; g[0].M = S_img.rows; g[0].W = b.ff2.w;
    g[0].bias = b.ff2.b; g[0].out = rowp(X, D, S_img.row0); g[0].ldo = D;
    g[0].res = g[0].out; g[0].ldr = D; g[0].gate = mi + GATE_MLP * D;
    g[1] = g[0];
    g[1].A = rowp(ACT, D5, 0) + D; g[1].M = S_txt.rows; g[1].W = b.ffc2.w; g[1].bias = b.ffc2.b;
    g[1].out = rowp(X, D, 0); g[1].res = g[1].out; g[1].gate = mt + GATE_MLP * D;
    ng = 2;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(ACT, D5, S_cond.row0) + D; g[2].M = S_cond.rows;
      g[2].out = rowp(X, D, S_cond.row0); g[2].res = g[2].out; g[2].gate = mc + GATE_MLP * D;
      ng = 3;
    }
    merged_w(g, 0, 2, b.ff2_m);
    if (h->use_merged && b.l_ffc2.set) g[1].W = b.ffc2_m;
    const LoraT* dff2 = &b.l_ff2;
    const LoraT* dffc2 = &b.l_ffc2;
    lg = lora_groups_dbl(lora_on(h, b.l_ffc2), &dffc2, b.l_ffc2.A, b.l_ffc2.B, lora_on(h, b.l_ff2), &dff2,
                         b.l_ff2.A, b.l_ff2.B);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_GATE_RES, D, D4, ng, g, lg, 1, D));
    else RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D4, ng, g, s));
  }

  // ================= single-stream blocks (block.py:275-333) =================
  const StreamRows S_main{0, h->n_main};
  for (int i = 0; i < h->cfg.num_single_layers; ++i) {
    const SingleBlk& b = h->sgl[i];
    const bf16* mm = MOD + mod_single(h, i, 0);
    const bf16* mc = MODC + mod_single(h, i, 0);
    // txt and img rows share the block's vectors; the cond rows use the cond_temb ones
    RF_TRY(ln3(mm + 1 * D, mm + 0 * D, mm + 1 * D, mm + 0 * D, mc + 1 * D, mc + 0 * D));
    // q|k|v
    memset(g, 0, sizeof(g));
    g[0].A = XN; g[0].lda = D; g[0].M = S_main.rows; g[0].W = b.qkv.w; g[0].bias = b.qkv.b;
    g[0].out = QKV; g[0].ldo = D3; g[0].rope_cos = h->rope_cos; g[0].rope_sin = h->rope_sin;
    g[0].norm_q = b.norm_q; g[0].norm_k = b.norm_k;
    ng = 1;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(XN, D, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(QKV, D3, S_cond.row0);
      g[1].rope_cos = h->crope_cos; g[1].rope_sin = h->crope_sin;
      ng = 2;
    }
    merged_w(g, 0, 1, b.qkv_m);
    const LoraT* sqkv[3] = {&b.l_q, &b.l_k, &b.l_v};
    LoraGroups lg = lora_groups(lora_on(h, b.l_q) || lora_on(h, b.l_k) || lora_on(h, b.l_v), 0, S_main.rows, 1,
                                sqkv, b.qkvA, b.qkvB);
    // exact-mode fast path: T for to_q|to_k|to_v|proj_mlp of all LoRA'd rows in one launch (both GEMMs read the
    // same XN rows; the q|k|v and the MLP-in launches have the same groups)
    bool t4 = lg.n > 0 && lora_on(h, b.l_mlp);
    if (t4) {
      bool any_fused = false;
      for (int j = 0; j < lg.n; ++j) any_fused |= rf::gemm_lora_eligible(rf::EPI_QKV, D3, D, g[lg.e[j].idx]);
      t4 = any_fused;
    }
    if (t4)
      RF_TRY(rf::lora_down_launch(g[lg.e[0].idx].A, D, lg.rows, D, b.qkvA, 4 * lpad, h->LT, 4 * lpad, s));
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_QKV, D3, D, ng, g, lg, 3, D3, t4 ? h->LT : nullptr, 4 * lpad));
    else RF_TRY(rf::gemm_launch(rf::EPI_QKV, D3, D, ng, g, s));
    // proj_mlp + GELU -> ACT[:, D:5D]
    memset(g, 0, sizeof(g));
    g[0].A = XN; g[0].lda = D; g[0].M = S_main.rows; g[0].W = b.mlp.w; g[0].bias = b.mlp.b;
    g[0].out = ACT + D; g[0].ldo = D5;
    ng = 1;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(XN, D, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(ACT, D5, S_cond.row0) + D;
      ng = 2;
    }
    merged_w(g, 0, 1, b.mlp_m);
    const LoraT* smlp = &b.l_mlp;
    lg = lora_groups(lora_on(h, b.l_mlp), 0, S_main.rows, 1, &smlp, b.l_mlp.A, b.l_mlp.B);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_GELU, D4, D, ng, g, lg, 1, D4, t4 ? h->LT + 3 * lpad : nullptr, 4 * lpad));
    else RF_TRY(rf::gemm_launch(rf::EPI_GELU, D4, D, ng, g, s));
    // attention -> ACT[:, 0:D]
    at.out = ACT; at.ldo = D5;
    RF_TRY(rf::attention_launch(at, s));
    // proj_out over cat(attn, mlp) (K = 5D) + gate + residual
    memset(g, 0, sizeof(g));
    g[0].A = ACT; g[0].lda = D5; g[0].M = S_main.rows; g[0].W = b.out.w; g[0].bias = b.out.b;
    g[0].out = X; g[0].ldo = D; g[0].res = X; g[0].ldr = D; g[0].gate = mm + 2 * D;
    ng = 1;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(ACT, D5, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(X, D, S_cond.row0); g[1].res = g[1].out; g[1].gate = mc + 2 * D;
      ng = 2;
    }
    merged_w(g, 0, 1, b.out_m);
    const LoraT* sout = &b.l_out;
    lg = lora_groups(lora_on(h, b.l_out), 0, S_main.rows, 1, &sout, b.l_out.A, b.l_out.B);
    if (lg.n) RF_TRY(gemm_lora(rf::EPI_GATE_RES, D, D5, ng, g, lg, 1, D));
    else RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D5, ng, g, s));
  }

  // ================= norm_out + proj_out (transformer.py:241-244) =================
  const bf16* mo = MOD + mod_out(h, 0);  // [scale | shift]
  RF_TRY(ln(S_img, mo, mo + D));
  memset(g, 0, sizeof(g));
  g[0].A = rowp(XN, D, S_img.row0); g[0].lda = D; g[0].M = S_img.rows; g[0].W = h->proj_out.w;
  g[0].bias = h->proj_out.b; g[0].out = out; g[0].ldo = h->cfg.in_channels;
  // proj_out (always target; N = 64): the unfused term
  const LoraT* lpo = &h->l_proj_out;
  if (h->use_merged) {
    if (lpo->set) g[0].W = h->proj_out_m;
  } else if (lora_on(h, *lpo)) {
    RF_TRY(lora_term(h, &lpo, 1, lpo->A, g[0].A, g[0].lda, g[0].M, nullptr, 0, h->LL, h->cfg.in_channels, s));
    g[0].addend = h->LL; g[0].ldadd = h->cfg.in_channels;
  }
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, h->cfg.in_channels, D, 1, g, s));
  return 0;
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
// LT [rows, 4 lora_pad] and LL [rows, 4D], each at least 8D (the adaLN / embedder LoRA scratch)
int alloc_lora_ws(rf_dit* h, int rows) {
  const size_t r = static_cast<size_t>(rows), least = static_cast<size_t>(8 * h->D) * 2;
  void* p = nullptr;
  RF_TRY(dev_alloc(h, &p, std::max(r * 4 * h->lora_pad * 2, least), true));
  h->LT = static_cast<bf16*>(p);
  RF_TRY(dev_alloc(h, &p, std::max(r * 4 * h->D * 2, least), true));
  h->LL = static_cast<bf16*>(p);
  h->lora_rows = rows;
  return 0;
}
// the merged copies hold W + (B A) * scaling for the current weights, adapters and call scale
bool merged_current(const rf_dit* h) { return h->lora_merged && h->merged_call_scale == h->call_scale; }

void drop_graph(rf_dit* h) {
  if (h->graph_exec) {
    cudaGraphExecDestroy(h->graph_exec);
    h->graph_exec = nullptr;
  }
}
void free_geometry(rf_dit* h) {
  drop_graph(h);
  for (void* p : h->geo_allocs) cudaFree(p);
  h->geo_allocs.clear();
  h->prepared = false;
  h->lora_rows = 0;
  h->s_cap_steps = 0;
  h->s_tsteps = nullptr;
  h->s_sigmas = nullptr;
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
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    rf::set_error("rf_dit_create: no CUDA device (this library has no CPU fallback)");
    return -3;
  }
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
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  if (h->ev_in) cudaEventDestroy(h->ev_in);
  if (h->ev_out) cudaEventDestroy(h->ev_out);
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

int rf_dit_load_weight(rf_dit* h, const char* key, const void* src, int64_t numel) {
  if (!h || !key || !src) {
    rf::set_error("rf_dit_load_weight: null argument");
    return -1;
  }
  auto it = h->slots.find(key);
  if (it == h->slots.end()) {
    rf::set_error(std::string("rf_dit_load_weight: unknown key ") + key);
    return -4;
  }
  if (it->second.numel != numel) {
    rf::set_error(std::string("rf_dit_load_weight: size mismatch for ") + key + ": got " +
                  std::to_string(numel) + ", want " + std::to_string(it->second.numel));
    return -4;
  }
  RF_CHECK_CUDA(cudaMemcpy(it->second.dst, src, static_cast<size_t>(numel) * 2,
                           cudaMemcpyDeviceToDevice));
  it->second.loaded = true;
  h->lora_merged = false;  // merged W + BA copies (fuse_lora mode) are stale now
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
  RF_TRY(lora_storage(h, t));
  RF_CHECK_CUDA(cudaMemset(t.A, 0, static_cast<size_t>(lpad) * t.in * 2));
  RF_CHECK_CUDA(cudaMemset(t.B, 0, static_cast<size_t>(t.out) * lpad * 2));
  RF_CHECK_CUDA(cudaMemcpy(t.A, A, static_cast<size_t>(r) * t.in * 2, cudaMemcpyDeviceToDevice));
  RF_CHECK_CUDA(cudaMemcpy2D(t.B, lpad * 2, B, static_cast<size_t>(r) * 2,
                             static_cast<size_t>(r) * 2, t.out, cudaMemcpyDeviceToDevice));
  t.set = true;
  t.scale = scale;
  h->any_lora = true;
  h->any_always |= t.always;
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
      RF_CHECK_CUDA(cudaMemset(t.A, 0, static_cast<size_t>(lpad) * t.in * 2));
      RF_CHECK_CUDA(cudaMemset(t.B, 0, static_cast<size_t>(t.out) * lpad * 2));
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
  // re-captured (rf_dit_denoise) when they were built for another scale
  h->call_scale = scale;
  return 0;
}

int rf_dit_missing_weights(rf_dit* h) {
  if (!h) return -1;
  int missing = 0;
  std::string names;
  for (auto& kv : h->slots) {
    if (!kv.second.loaded) {
      if (missing < 8) names += kv.first + " ";
      ++missing;
    }
  }
  if (missing) rf::set_error("missing weights: " + names + (missing > 8 ? "..." : ""));
  return missing;
}

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
    void* p;
    auto A = [&](size_t bytes) -> void* {
      void* q = nullptr;
      if (dev_alloc(h, &q, bytes, true)) return nullptr;
      return q;
    };
    if (!(p = A(static_cast<size_t>(n_main) * 64 * 4))) return -2; h->rope_cos = static_cast<float*>(p);
    if (!(p = A(static_cast<size_t>(n_main) * 64 * 4))) return -2; h->rope_sin = static_cast<float*>(p);
    if (!(p = A(static_cast<size_t>(std::max(n_cond, 1)) * 64 * 4))) return -2; h->crope_cos = static_cast<float*>(p);
    if (!(p = A(static_cast<size_t>(std::max(n_cond, 1)) * 64 * 4))) return -2; h->crope_sin = static_cast<float*>(p);
    if (!(p = A(static_cast<size_t>(N) * D * 2))) return -2; h->X = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(N) * D * 2))) return -2; h->XN = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(N) * 3 * D * 2))) return -2; h->QKV = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(N) * 5 * D * 2))) return -2; h->ACT = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(h->n_mod) * 2))) return -2; h->MOD = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(h->n_mod) * 2))) return -2; h->MODC = static_cast<bf16*>(p);
    RF_TRY(alloc_lora_ws(h, lora_rows));
    if (!(p = A(static_cast<size_t>(512 + 4 * D) * 2))) return -2; h->emb_tmp = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(D) * 2))) return -2; h->temb = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(D) * 2))) return -2; h->ctemb = static_cast<bf16*>(p);
    const int C = h->cfg.in_channels;
    if (!(p = A(static_cast<size_t>(batch) * n_img * C * 2))) return -2; h->s_lat = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(batch) * n_img * C * 2))) return -2; h->s_v = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(batch) * n_txt * h->cfg.joint_attention_dim * 2))) return -2; h->s_txt = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(batch) * h->cfg.pooled_projection_dim * 2))) return -2; h->s_pooled = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(batch) * std::max(n_cond, 1) * C * 2))) return -2; h->s_cond = static_cast<bf16*>(p);
    if (!(p = A(static_cast<size_t>(batch) * 2 + 16))) return -2; h->s_guid = static_cast<bf16*>(p);
    if (!(p = A(16))) return -2; h->s_zero_one = static_cast<bf16*>(p);
    if (!(p = A(16))) return -2; h->s_step = static_cast<int*>(p);
    h->s_cap_steps = 0;
    h->s_tsteps = nullptr;
    h->s_sigmas = nullptr;
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
    for (bf16* old : {h->LT, h->LL}) {
      auto it = std::find(h->geo_allocs.begin(), h->geo_allocs.end(), static_cast<void*>(old));
      if (it != h->geo_allocs.end()) h->geo_allocs.erase(it);
      cudaFree(old);
    }
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

int rf_dit_denoise(rf_dit* h, void* latents_inout, const void* txt, const void* pooled,
                   const uint16_t* timesteps_bf16_host, const float* sigmas_host, int n_steps,
                   float guidance_scale, const void* cond_latents, void* stream) {
  int rc = check_ready(h, "rf_dit_denoise", static_cast<cudaStream_t>(stream));
  if (rc) return rc;
  if (!latents_inout || !txt || !pooled || !timesteps_bf16_host || !sigmas_host || n_steps <= 0 ||
      (h->n_cond > 0 && !cond_latents)) {
    rf::set_error("rf_dit_denoise: bad argument");
    return -1;
  }
  // The loop runs on a handle-owned stream (graph capture is not permitted on the legacy default
  // stream callers often pass); it is ordered after / before the caller's stream with events, so
  // the call still only enqueues work.
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  if (!h->own_stream) {
    RF_CHECK_CUDA(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
  }
  cudaStream_t s = h->own_stream;
  RF_CHECK_CUDA(cudaEventRecord(h->ev_in, caller));
  RF_CHECK_CUDA(cudaStreamWaitEvent(s, h->ev_in, 0));
  const int C = h->cfg.in_channels;
  if (n_steps > h->s_cap_steps) {
    void* p = nullptr;
    if (dev_alloc(h, &p, static_cast<size_t>(n_steps) * 2, true)) return -2;
    h->s_tsteps = static_cast<bf16*>(p);
    if (dev_alloc(h, &p, static_cast<size_t>(n_steps + 1) * 4, true)) return -2;
    h->s_sigmas = static_cast<float*>(p);
    if (dev_alloc(h, &p, static_cast<size_t>(n_steps) * h->n_mod * 2, true)) return -2;
    h->s_mod_all = static_cast<bf16*>(p);
    if (dev_alloc(h, &p, (static_cast<size_t>(n_steps) * (256 + 3 * h->D + h->lora_pad + 6 * h->D) + 256 + 3 * h->D) * 2,
                  true))
      return -2;
    h->s_temb_ws = static_cast<bf16*>(p);
    h->s_cap_steps = n_steps;
    drop_graph(h);  // graph referenced the old arrays
  }
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_tsteps, timesteps_bf16_host, static_cast<size_t>(n_steps) * 2,
                                cudaMemcpyHostToDevice, s));
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_sigmas, sigmas_host, static_cast<size_t>(n_steps + 1) * 4,
                                cudaMemcpyHostToDevice, s));
  const bf16 gb = __float2bfloat16_rn(guidance_scale);
  RF_CHECK_CUDA(cudaMemcpyAsync(h->s_guid, &gb, 2, cudaMemcpyHostToDevice, s));

  for (int b = 0; b < h->batch; ++b) {
    bf16* lat_b = static_cast<bf16*>(latents_inout) + static_cast<int64_t>(b) * h->n_img * C;
    // stage this sample's inputs so the captured graph always sees the same addresses
    RF_CHECK_CUDA(cudaMemcpyAsync(h->s_lat, lat_b, static_cast<size_t>(h->n_img) * C * 2,
                                  cudaMemcpyDeviceToDevice, s));
    RF_CHECK_CUDA(cudaMemcpyAsync(
        h->s_txt,
        static_cast<const bf16*>(txt) + static_cast<int64_t>(b) * h->n_txt * h->cfg.joint_attention_dim,
        static_cast<size_t>(h->n_txt) * h->cfg.joint_attention_dim * 2, cudaMemcpyDeviceToDevice, s));
    RF_CHECK_CUDA(cudaMemcpyAsync(
        h->s_pooled,
        static_cast<const bf16*>(pooled) + static_cast<int64_t>(b) * h->cfg.pooled_projection_dim,
        static_cast<size_t>(h->cfg.pooled_projection_dim) * 2, cudaMemcpyDeviceToDevice, s));
    if (h->n_cond > 0) {
      RF_CHECK_CUDA(cudaMemcpyAsync(
          h->s_cond, static_cast<const bf16*>(cond_latents) + static_cast<int64_t>(b) * h->n_cond * C,
          static_cast<size_t>(h->n_cond) * C * 2, cudaMemcpyDeviceToDevice, s));
      RF_TRY(compute_cond_mod(h, h->s_pooled, s));  // hoisted out of the step loop
    }
    RF_TRY(precompute_step_mods(h, n_steps, h->s_tsteps, h->s_guid, h->s_pooled, s));
    RF_CHECK_CUDA(cudaMemsetAsync(h->s_step, 0, sizeof(int), s));
    // the captured step holds the LoRA scalings as kernel parameters (and skips the terms a zero scaling
    // removes): a changed call scale is re-captured
    if (h->graph_exec && h->graph_call_scale != h->call_scale) drop_graph(h);
    if (!h->graph_exec) {
      h->graph_call_scale = h->call_scale;
      // capture one step: forward -> Euler update -> step counter
      cudaGraph_t graph = nullptr;
      const int64_t launches_before = rf::launch_count();
      RF_CHECK_CUDA(cudaStreamSynchronize(s));
      RF_CHECK_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      int erc = enqueue_forward(h, h->s_lat, h->s_txt, h->s_pooled, h->s_tsteps, h->s_step,
                                h->s_guid, h->n_cond > 0 ? h->s_cond : nullptr, h->s_v, s,
                                h->s_mod_all);
      if (!erc) erc = rf::euler_step_launch(h->s_lat, h->s_v, h->s_sigmas, h->s_step, h->n_img * C, s);
      if (!erc) erc = rf::advance_step_launch(h->s_step, s);
      cudaError_t ce = cudaStreamEndCapture(s, &graph);
      if (erc || ce != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        if (!erc) {
          rf::set_error(std::string("graph capture failed: ") + cudaGetErrorString(ce));
          erc = -2;
        }
        return erc;
      }
      h->graph_kernels = rf::launch_count() - launches_before;
      rf::count_launch(static_cast<int>(-h->graph_kernels));  // captured, not executed
      ce = cudaGraphInstantiate(&h->graph_exec, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) {
        h->graph_exec = nullptr;
        rf::set_error(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce));
        return -2;
      }
    }
    for (int i = 0; i < n_steps; ++i) {
      RF_CHECK_CUDA(cudaGraphLaunch(h->graph_exec, s));
      rf::count_launch(static_cast<int>(h->graph_kernels));
    }
    RF_CHECK_CUDA(cudaMemcpyAsync(lat_b, h->s_lat, static_cast<size_t>(h->n_img) * C * 2,
                                  cudaMemcpyDeviceToDevice, s));
  }
  RF_CHECK_CUDA(cudaEventRecord(h->ev_out, s));
  RF_CHECK_CUDA(cudaStreamWaitEvent(caller, h->ev_out, 0));
  return 0;
}

}  // extern "C"
