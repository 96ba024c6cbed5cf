// dit.cu — host orchestration of the FLUX.1-dev DiT forward and denoise loop (C ABI:
// rf_dit_* in include/rf_b200.h) over the sm_90a kernels of this directory.
//
// Mirrors, launch by launch, what the reference executes per step:
//   train_flux/flux/transformer.py:47-252 (tranformer_forward; with n_cond == 0 the stock
//   diffusers FluxTransformer2DModel.forward), train_flux/flux/block.py:173-333 (block_forward,
//   single_block_forward, attn_forward), train_flux/flux/generate.py:217-276 (denoise loop),
//   train_flux/flux/lora_controller.py:5-42 (LoRA on condition tokens only).
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
int lora_merge_launch(const bf16* W, const bf16* A, const bf16* B, bf16* Wm, int N, int K, int R,
                      cudaStream_t stream);
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

struct Slot {
  bf16* dst;
  int64_t numel;
  bool loaded;
};

struct Lin {  // views into the weight arena
  bf16* w = nullptr;
  bf16* b = nullptr;
};

struct LoraT {  // zero-padded rank-64 factors of one target
  bf16* A = nullptr;  // [64, in]
  bf16* B = nullptr;  // [out, 64]
  int in = 0, out = 0;
  bool set = false;
};
// (merged weights W + B A of a whole packed projection live in the block structs: *_m)

struct DoubleBlk {
  Lin qkv, add_qkv, to_out, to_add_out, ff1, ff2, ffc1, ffc2;
  bf16 *norm_q, *norm_k, *norm_added_q, *norm_added_k;
  LoraT l_norm1, l_q, l_k, l_v, l_out, l_ff2;
  bf16* qkvA = nullptr;  // [192, D] = stacked A of to_q/to_k/to_v
  bf16* qkvB = nullptr;  // [3D, 64] = stacked B (rows of the packed q|k|v projection)
  bf16 *qkv_m = nullptr, *to_out_m = nullptr, *ff2_m = nullptr;  // merged W + B A (fuse_lora mode)
};
struct SingleBlk {
  Lin qkv, mlp, out;
  bf16 *norm_q, *norm_k;
  LoraT l_norm, l_q, l_k, l_v, l_mlp, l_out;
  bf16* qkvA = nullptr;
  bf16* qkvB = nullptr;
  bf16 *qkv_m = nullptr, *mlp_m = nullptr, *out_m = nullptr;
};

constexpr int kLoraPad = 64;

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
  bf16* modW = nullptr;
  bf16* modB = nullptr;
  int64_t n_mod = 0;
  std::vector<DoubleBlk> dbl;
  std::vector<SingleBlk> sgl;
  bool any_lora = false;
  bool lora_merged = false;   // merged copies are current
  bool use_merged = false;    // rf_dit_prepare flag bit 3
  bf16* x_emb_m = nullptr;
  // ---- geometry
  bool prepared = false;
  int batch = 0, n_txt = 0, n_img = 0, n_cond = 0, N = 0, n_main = 0;
  int flags = 0;
  int attn_cond_mode = 0;
  float attn_cond_bias = 0.f;
  float *rope_cos = nullptr, *rope_sin = nullptr, *crope_cos = nullptr, *crope_sin = nullptr;
  // ---- workspace
  bf16 *X = nullptr, *XN = nullptr, *QKV = nullptr, *ACT = nullptr, *MOD = nullptr, *MODC = nullptr;
  bf16 *LT = nullptr, *LL = nullptr;  // LoRA temporaries: T [rows, 192], L [rows, 4D]
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
  // forked stream of the LoRA down-projections: they run on a few reserved SMs beside the other token streams'
  // GEMM of the same layer (lora_down_side_launch) and join before the condition stream's launch
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
};

namespace {

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
  t.A = A_view ? A_view : ar.take(static_cast<int64_t>(kLoraPad) * in);
  t.B = B_view ? B_view : ar.take(static_cast<int64_t>(out) * kLoraPad);
  // unset targets must contribute exactly zero (a q-only adapter still runs the stacked q|k|v path)
  if (t.A) cudaMemset(t.A, 0, static_cast<size_t>(kLoraPad) * in * 2);
  if (t.B) cudaMemset(t.B, 0, static_cast<size_t>(out) * kLoraPad * 2);
  h->lora_slots[mod] = &t;
}

int build_storage(rf_dit* h) {
  const rf_dit_config& c = h->cfg;
  const int D = h->D;
  Arena ar{h};
  h->x_emb = new_lin(h, ar, "x_embedder", D, c.in_channels);
  new_lora(h, ar, "x_embedder", h->l_x_emb, D, c.in_channels);
  h->ctx_emb = new_lin(h, ar, "context_embedder", D, c.joint_attention_dim);
  h->t1 = new_lin(h, ar, "time_text_embed.timestep_embedder.linear_1", D, 256);
  h->t2 = new_lin(h, ar, "time_text_embed.timestep_embedder.linear_2", D, D);
  if (c.guidance_embeds) {
    h->g1 = new_lin(h, ar, "time_text_embed.guidance_embedder.linear_1", D, 256);
    h->g2 = new_lin(h, ar, "time_text_embed.guidance_embedder.linear_2", D, D);
  }
  h->p1 = new_lin(h, ar, "time_text_embed.text_embedder.linear_1", D, c.pooled_projection_dim);
  h->p2 = new_lin(h, ar, "time_text_embed.text_embedder.linear_2", D, D);
  h->proj_out = new_lin(h, ar, "proj_out", c.in_channels, D);

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
    b.qkv = new_lin(h, ar, "", 3 * D, D);
    b.add_qkv = new_lin(h, ar, "", 3 * D, D);
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    const char* an[3] = {"add_q_proj", "add_k_proj", "add_v_proj"};
    if (c.lora_rank > 0) {
      b.qkvA = ar.take(static_cast<int64_t>(3 * kLoraPad) * D);
      b.qkvB = ar.take(static_cast<int64_t>(3 * D) * kLoraPad);
    }
    LoraT* lq[3] = {&b.l_q, &b.l_k, &b.l_v};
    for (int j = 0; j < 3; ++j) {
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
      reg_lin(h, p + "attn." + an[j], b.add_qkv.w + static_cast<int64_t>(j) * D * D,
              b.add_qkv.b + j * D, D, D);
      new_lora(h, ar, p + "attn." + nm[j], *lq[j], D, D,
               b.qkvA ? b.qkvA + static_cast<int64_t>(j) * kLoraPad * D : nullptr,
               b.qkvB ? b.qkvB + static_cast<int64_t>(j) * D * kLoraPad : nullptr);
    }
    b.norm_q = ar.take(128); reg(h, p + "attn.norm_q.weight", b.norm_q, 128);
    b.norm_k = ar.take(128); reg(h, p + "attn.norm_k.weight", b.norm_k, 128);
    b.norm_added_q = ar.take(128); reg(h, p + "attn.norm_added_q.weight", b.norm_added_q, 128);
    b.norm_added_k = ar.take(128); reg(h, p + "attn.norm_added_k.weight", b.norm_added_k, 128);
    b.to_out = new_lin(h, ar, p + "attn.to_out.0", D, D);
    new_lora(h, ar, p + "attn.to_out.0", b.l_out, D, D);
    b.to_add_out = new_lin(h, ar, p + "attn.to_add_out", D, D);
    b.ff1 = new_lin(h, ar, p + "ff.net.0.proj", 4 * D, D);
    b.ff2 = new_lin(h, ar, p + "ff.net.2", D, 4 * D);
    new_lora(h, ar, p + "ff.net.2", b.l_ff2, D, 4 * D);
    b.ffc1 = new_lin(h, ar, p + "ff_context.net.0.proj", 4 * D, D);
    b.ffc2 = new_lin(h, ar, p + "ff_context.net.2", D, 4 * D);
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
      b.qkvA = ar.take(static_cast<int64_t>(4 * kLoraPad) * D);
      b.qkvB = ar.take(static_cast<int64_t>(3 * D) * kLoraPad);
    }
    const char* nm[3] = {"to_q", "to_k", "to_v"};
    LoraT* lq[3] = {&b.l_q, &b.l_k, &b.l_v};
    for (int j = 0; j < 3; ++j) {
      reg_lin(h, p + "attn." + nm[j], b.qkv.w + static_cast<int64_t>(j) * D * D, b.qkv.b + j * D, D, D);
      new_lora(h, ar, p + "attn." + nm[j], *lq[j], D, D,
               b.qkvA ? b.qkvA + static_cast<int64_t>(j) * kLoraPad * D : nullptr,
               b.qkvB ? b.qkvB + static_cast<int64_t>(j) * D * kLoraPad : nullptr);
    }
    b.norm_q = ar.take(128); reg(h, p + "attn.norm_q.weight", b.norm_q, 128);
    b.norm_k = ar.take(128); reg(h, p + "attn.norm_k.weight", b.norm_k, 128);
    b.mlp = new_lin(h, ar, p + "proj_mlp", 4 * D, D);
    new_lora(h, ar, p + "proj_mlp", b.l_mlp, 4 * D, D,
             b.qkvA ? b.qkvA + static_cast<int64_t>(3 * kLoraPad) * D : nullptr);
    b.out = new_lin(h, ar, p + "proj_out", D, 5 * D);
    new_lora(h, ar, p + "proj_out", b.l_out, D, 5 * D);
  }
  const int64_t oo = so + static_cast<int64_t>(c.num_single_layers) * 3 * D;
  reg_lin(h, "norm_out.linear", h->modW + oo * D, h->modB + oo, 2 * D, D);
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

#define RF_TRY(expr)            \
  do {                          \
    int _rc = (expr);           \
    if (_rc != 0) return _rc;   \
  } while (0)

// y = linear_2(silu(linear_1(x)))  (TimestepEmbedding / PixArtAlphaTextProjection)
int mlp2(rf_dit* h, const bf16* x, int in_dim, const Lin& l1, const Lin& l2, bf16* tmp, bf16* out,
         cudaStream_t s) {
  RF_TRY(rf::gemv_launch(x, in_dim, 1, l1.w, l1.b, tmp, h->D, h->D, in_dim, 0, s));
  RF_TRY(rf::gemv_launch(tmp, h->D, 1, l2.w, l2.b, out, h->D, h->D, h->D, 1, s));
  return 0;
}

// temb = time(t) + guidance(g) + text(pooled)   (CombinedTimestepGuidanceTextProjEmbeddings)
int compute_temb(rf_dit* h, const bf16* t, const int* step, const bf16* guid, const bf16* pooled,
                 bf16* out, cudaStream_t s) {
  const int D = h->D;
  bf16* e = h->emb_tmp;  // [256 | 256 | D tmp | D a | D b | D c]
  bf16 *tp = e, *gp = e + 256, *tmp = e + 512, *a = tmp + D, *b = a + D, *c = b + D;
  RF_TRY(rf::timestep_embed_launch(t, step, 1, 1000.0f, tp, 1, s));
  RF_TRY(mlp2(h, tp, 256, h->t1, h->t2, tmp, a, s));
  RF_TRY(mlp2(h, pooled, h->cfg.pooled_projection_dim, h->p1, h->p2, tmp, c, s));
  if (h->cfg.guidance_embeds) {
    RF_TRY(rf::timestep_embed_launch(guid, nullptr, 1, 1000.0f, gp, 1, s));
    RF_TRY(mlp2(h, gp, 256, h->g1, h->g2, tmp, b, s));
    RF_TRY(rf::add3_launch(a, b, c, out, D, s));
  } else {
    RF_TRY(rf::add2_launch(a, c, out, D, s));
  }
  return 0;
}

// L[rows, out] = bf16( bf16(x A^T) B^T ): the peft low-rank term for `rows` condition tokens
int lora_term(rf_dit* h, const LoraT& t, const bf16* x, int ldx, int rows, bf16* L, int ldl,
              cudaStream_t s) {
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = x; g.lda = ldx; g.M = rows; g.W = t.A; g.out = h->LT; g.ldo = kLoraPad;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, kLoraPad, t.in, 1, &g, s));
  memset(&g, 0, sizeof(g));
  g.A = h->LT; g.lda = kLoraPad; g.M = rows; g.W = t.B; g.out = L; g.ldo = ldl;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, t.out, kLoraPad, 1, &g, s));
  return 0;
}

// fused q|k|v low-rank term: T = x [Aq;Ak;Av]^T (one GEMM), L[:, jD:(j+1)D] = T_j B_j^T (grouped)
int lora_term_qkv(rf_dit* h, const bf16* qkvA, const LoraT& lq, const LoraT& lk, const LoraT& lv,
                  const bf16* x, int ldx, int rows, bf16* L, int ldl, cudaStream_t s) {
  const int D = h->D;
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = x; g.lda = ldx; g.M = rows; g.W = qkvA; g.out = h->LT; g.ldo = 3 * kLoraPad;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, 3 * kLoraPad, D, 1, &g, s));
  rf::GemmGroupArgs gg[3];
  memset(gg, 0, sizeof(gg));
  const LoraT* ls[3] = {&lq, &lk, &lv};
  for (int j = 0; j < 3; ++j) {
    gg[j].A = h->LT + j * kLoraPad; gg[j].lda = 3 * kLoraPad; gg[j].M = rows;
    gg[j].W = ls[j]->B; gg[j].out = L + static_cast<int64_t>(j) * D; gg[j].ldo = ldl;
  }
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, D, kLoraPad, 3, gg, s));
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
  // LoRA of norm1.linear / norm.linear acts on silu(cond_temb): M = 1 -> two GEMVs + add
  bf16* tvec = h->LT;          // [64]
  bf16* lvec = h->LT + 256;    // [6D]
  for (int i = 0; i < h->cfg.num_layers; ++i) {
    const LoraT& t = h->dbl[i].l_norm1;
    if (!t.set) continue;
    bf16* dst = h->MODC + mod_double(h, i, 0, 0);
    RF_TRY(rf::gemv_launch(h->ctemb, D, 1, t.A, nullptr, tvec, kLoraPad, kLoraPad, D, 1, s));
    RF_TRY(rf::gemv_launch(tvec, kLoraPad, 1, t.B, nullptr, lvec, 6 * D, 6 * D, kLoraPad, 0, s));
    RF_TRY(rf::add2_launch(dst, lvec, dst, 6 * D, s));
  }
  for (int i = 0; i < h->cfg.num_single_layers; ++i) {
    const LoraT& t = h->sgl[i].l_norm;
    if (!t.set) continue;
    bf16* dst = h->MODC + mod_single(h, i, 0);
    RF_TRY(rf::gemv_launch(h->ctemb, D, 1, t.A, nullptr, tvec, kLoraPad, kLoraPad, D, 1, s));
    RF_TRY(rf::gemv_launch(tvec, kLoraPad, 1, t.B, nullptr, lvec, 3 * D, 3 * D, kLoraPad, 0, s));
    RF_TRY(rf::add2_launch(dst, lvec, dst, 3 * D, s));
  }
  return 0;
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
  return rf::lora_merge_launch(W + off, t.A, t.B, *Wm + off, t.out, t.in, kLoraPad, s);
}
int merge_all(rf_dit* h, cudaStream_t s) {
  const int D = h->D;
  RF_TRY(merge_one(h, h->l_x_emb, h->x_emb.w, &h->x_emb_m, 0, D, s));
  for (auto& b : h->dbl) {
    RF_TRY(merge_one(h, b.l_q, b.qkv.w, &b.qkv_m, 0, 3 * D, s));
    RF_TRY(merge_one(h, b.l_k, b.qkv.w, &b.qkv_m, D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_v, b.qkv.w, &b.qkv_m, 2 * D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_out, b.to_out.w, &b.to_out_m, 0, D, s));
    RF_TRY(merge_one(h, b.l_ff2, b.ff2.w, &b.ff2_m, 0, D, s));
  }
  for (auto& b : h->sgl) {
    RF_TRY(merge_one(h, b.l_q, b.qkv.w, &b.qkv_m, 0, 3 * D, s));
    RF_TRY(merge_one(h, b.l_k, b.qkv.w, &b.qkv_m, D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_v, b.qkv.w, &b.qkv_m, 2 * D, 3 * D, s));
    RF_TRY(merge_one(h, b.l_mlp, b.mlp.w, &b.mlp_m, 0, 4 * D, s));
    RF_TRY(merge_one(h, b.l_out, b.out.w, &b.out_m, 0, D, s));
  }
  h->lora_merged = true;
  return 0;
}

// temb_i = time(t_i) + guidance(g) + text(pooled) for ALL steps, then every adaLN Linear of every
// block for all steps: the 6.5 GB modulation weight stack is streamed ceil(n/8) times per denoise
// call instead of once per step.  Same kernels, same per-vector arithmetic as compute_temb + gemv
// (the GEMV's per-vector summation order does not depend on the batch width): bit-identical.
int precompute_step_mods(rf_dit* h, int n_steps, const bf16* tsteps, const bf16* guid,
                         const bf16* pooled, cudaStream_t s) {
  const int D = h->D;
  bf16* ws = h->s_temb_ws;  // [n,256] | [n,D] tmp | [n,D] a | [n,D] temb | [256] gp | [D] tmp1 | [D] b | [D] c
  bf16* tp = ws;
  bf16* tmp = tp + static_cast<int64_t>(n_steps) * 256;
  bf16* a = tmp + static_cast<int64_t>(n_steps) * D;
  bf16* temb = a + static_cast<int64_t>(n_steps) * D;
  bf16* gp = temb + static_cast<int64_t>(n_steps) * D;
  bf16 *tmp1 = gp + 256, *b = tmp1 + D, *c = b + D;
  RF_TRY(rf::timestep_embed_launch(tsteps, nullptr, 1, 1000.0f, tp, n_steps, s));
  RF_TRY(rf::gemv_launch(tp, 256, n_steps, h->t1.w, h->t1.b, tmp, D, D, 256, 0, s));
  RF_TRY(rf::gemv_launch(tmp, D, n_steps, h->t2.w, h->t2.b, a, D, D, D, 1, s));
  RF_TRY(mlp2(h, pooled, h->cfg.pooled_projection_dim, h->p1, h->p2, tmp1, c, s));
  if (h->cfg.guidance_embeds) {
    RF_TRY(rf::timestep_embed_launch(guid, nullptr, 1, 1000.0f, gp, 1, s));
    RF_TRY(mlp2(h, gp, 256, h->g1, h->g2, tmp1, b, s));
  }
  for (int i = 0; i < n_steps; ++i) {
    bf16* ai = a + static_cast<int64_t>(i) * D;
    bf16* ti = temb + static_cast<int64_t>(i) * D;
    if (h->cfg.guidance_embeds) RF_TRY(rf::add3_launch(ai, b, c, ti, D, s));
    else RF_TRY(rf::add2_launch(ai, c, ti, D, s));
  }
  RF_TRY(rf::gemv_launch(temb, D, n_steps, h->modW, h->modB, h->s_mod_all, static_cast<int>(h->n_mod),
                         static_cast<int>(h->n_mod), D, 1, s));
  return 0;
}

struct StreamRows {
  int row0, rows;
};

// The body of one DiT forward for one sample.  All pointers are device pointers.
int enqueue_forward(rf_dit* h, const bf16* latents, const bf16* txt, const bf16* pooled,
                    const bf16* tstep, const int* step_idx, const bf16* guid, const bf16* cond_lat,
                    bf16* out, cudaStream_t s, const bf16* mod_all = nullptr) {
  const int D = h->D, D3 = 3 * D, D4 = 4 * D, D5 = 5 * D;
  const bool use_cond = h->n_cond > 0;
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
    if (h->use_merged) {
      g[1].W = h->x_emb_m;
    } else if (h->l_x_emb.set) {
      RF_TRY(lora_term(h, h->l_x_emb, cond_lat, h->cfg.in_channels, h->n_cond, h->LL, D, s));
      g[1].addend = h->LL; g[1].ldadd = D;
    }
    ng = 2;
  }
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, D, h->cfg.in_channels, ng, g, s));
  memset(g, 0, sizeof(g));
  g[0].A = txt; g[0].lda = h->cfg.joint_attention_dim; g[0].M = h->n_txt; g[0].W = h->ctx_emb.w;
  g[0].bias = h->ctx_emb.b; g[0].out = rowp(X, D, 0); g[0].ldo = D;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, D, h->cfg.joint_attention_dim, 1, g, s));

  // ---- temb and every modulation vector of the step (transformer.py:95-107 + all adaLN linears)
  if (mod_all != nullptr) {  // denoise loop: this step's row of the precomputed table
    RF_TRY(rf::select_row_launch(mod_all, h->n_mod, step_idx, h->MOD, s));
  } else {
    RF_TRY(compute_temb(h, tstep, step_idx, guid, pooled, h->temb, s));
    RF_TRY(rf::gemv_launch(h->temb, D, 1, h->modW, h->modB, h->MOD, static_cast<int>(h->n_mod),
                           static_cast<int>(h->n_mod), D, 1, s));
  }
  const bf16* MOD = h->MOD;
  const bf16* MODC = h->MODC;

  auto ln = [&](const StreamRows& sr, const bf16* scale, const bf16* shift) {
    return rf::ln_modulate_launch(rowp(X, D, sr.row0), D, rowp(XN, D, sr.row0), D, sr.rows, D, scale,
                                  shift, sr.rows, 0, s);
  };
  // RF_SIDE_STREAM=0 keeps the down-projections on the main stream (single-stream schedule; A/B of the fork)
  const char* side_s = getenv("RF_SIDE_STREAM");  // read per enqueue (= per graph capture)
  const bool side_env = !(side_s && atoi(side_s) == 0);
  if (side_env && use_cond && !h->use_merged && h->any_lora && h->side_stream == nullptr) {
    RF_CHECK_CUDA(cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
  }
  const bool side_lora = side_env && h->side_stream != nullptr;
  // A grouped GEMM whose LAST group is the condition stream carrying a LoRA (exact mode).  Fast path:
  // T = bf16(x A^T) (one skinny GEMM), the other streams as one grouped launch, then the condition
  // stream with the low-rank k-block fused (gemm2_lora_launch) — L = T B^T never reaches HBM.  Small /
  // odd shapes keep the unfused path: L materialised by two GEMMs and added in the epilogue (`addend`).
  // (t_pre != nullptr: T was already produced by an earlier launch, [M, ld_t] with this target's columns at t_pre)
  auto gemm_cond_lora = [&](int epi, int N, int K, int ngr, rf::GemmGroupArgs* gr, const bf16* loraA,
                            int t_cols, const bf16* loraB, int sec_cols, auto&& unfused_term,
                            const bf16* t_pre = nullptr, int ld_t = 0) -> int {
    rf::GemmGroupArgs& gc = gr[ngr - 1];
    if (rf::gemm2_lora_eligible(epi, N, K, gc)) {
      const bf16* T = t_pre;
      if (T == nullptr && ngr > 1 && side_lora) {
        // fork: the down-projection runs on kLoraSideCtas reserved SMs while the other streams' GEMM has the rest
        RF_CHECK_CUDA(cudaEventRecord(h->ev_fork, s));
        const int prev = rf::gemm_reserve_sms(rf::kLoraSideCtas);
        const int mrc = rf::gemm_launch(epi, N, K, ngr - 1, gr, s);
        rf::gemm_reserve_sms(prev);
        if (mrc) return mrc;
        RF_CHECK_CUDA(cudaStreamWaitEvent(h->side_stream, h->ev_fork, 0));
        RF_TRY(rf::lora_down_side_launch(gc.A, gc.lda, gc.M, K, loraA, t_cols, h->LT, t_cols, h->side_stream));
        RF_CHECK_CUDA(cudaEventRecord(h->ev_join, h->side_stream));
        RF_CHECK_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
        return rf::gemm2_lora_launch(epi, N, K, gc, h->LT, t_cols, loraB, sec_cols, s);
      }
      if (T == nullptr) {
        RF_TRY(rf::lora_down_launch(gc.A, gc.lda, gc.M, K, loraA, t_cols, h->LT, t_cols, s));
        T = h->LT;
        ld_t = t_cols;
      }
      if (ngr > 1) RF_TRY(rf::gemm_launch(epi, N, K, ngr - 1, gr, s));
      return rf::gemm2_lora_launch(epi, N, K, gc, T, ld_t, loraB, sec_cols, s);
    }
    RF_TRY(unfused_term(gc));
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
    bool cond_lora = false;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(XN, D, S_cond.row0); g[2].M = S_cond.rows;
      g[2].out = rowp(QKV, D3, S_cond.row0);
      g[2].rope_cos = h->crope_cos; g[2].rope_sin = h->crope_sin;
      if (h->use_merged) {
        g[2].W = b.qkv_m;
      } else if (b.l_q.set || b.l_k.set || b.l_v.set) {
        cond_lora = true;
      }
      ng = 3;
    }
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_QKV, D3, D, ng, g, b.qkvA, 3 * kLoraPad, b.qkvB, D, [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term_qkv(h, b.qkvA, b.l_q, b.l_k, b.l_v, gc.A, D, S_cond.rows, h->LL, D3, s));
        gc.addend = h->LL; gc.ldadd = D3;
        return 0;
      }));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_QKV, D3, D, ng, g, s));
    }
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
    cond_lora = false;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(ACT, D5, S_cond.row0); g[2].M = S_cond.rows;
      g[2].out = rowp(X, D, S_cond.row0); g[2].res = g[2].out; g[2].gate = mc + GATE_MSA * D;
      if (h->use_merged) {
        g[2].W = b.to_out_m;
      } else if (b.l_out.set) {
        cond_lora = true;
      }
      ng = 3;
    }
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_GATE_RES, D, D, ng, g, b.l_out.A, kLoraPad, b.l_out.B, 0, [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term(h, b.l_out, gc.A, D5, S_cond.rows, h->LL, D, s));
        gc.addend = h->LL; gc.ldadd = D;
        return 0;
      }));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D, ng, g, s));
    }
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
    RF_TRY(rf::gemm_launch(rf::EPI_GELU, D4, D, ng, g, s));
    // MLP out + gate + residual
    memset(g, 0, sizeof(g));
    g[0].A = rowp(ACT, D5, S_img.row0) + D; g[0].lda = D5; g[0].M = S_img.rows; g[0].W = b.ff2.w;
    g[0].bias = b.ff2.b; g[0].out = rowp(X, D, S_img.row0); g[0].ldo = D;
    g[0].res = g[0].out; g[0].ldr = D; g[0].gate = mi + GATE_MLP * D;
    g[1] = g[0];
    g[1].A = rowp(ACT, D5, 0) + D; g[1].M = S_txt.rows; g[1].W = b.ffc2.w; g[1].bias = b.ffc2.b;
    g[1].out = rowp(X, D, 0); g[1].res = g[1].out; g[1].gate = mt + GATE_MLP * D;
    ng = 2;
    cond_lora = false;
    if (use_cond) {
      g[2] = g[0];
      g[2].A = rowp(ACT, D5, S_cond.row0) + D; g[2].M = S_cond.rows;
      g[2].out = rowp(X, D, S_cond.row0); g[2].res = g[2].out; g[2].gate = mc + GATE_MLP * D;
      if (h->use_merged) {
        g[2].W = b.ff2_m;
      } else if (b.l_ff2.set) {
        cond_lora = true;
      }
      ng = 3;
    }
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_GATE_RES, D, D4, ng, g, b.l_ff2.A, kLoraPad, b.l_ff2.B, 0, [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term(h, b.l_ff2, gc.A, D5, S_cond.rows, h->LL, D, s));
        gc.addend = h->LL; gc.ldadd = D;
        return 0;
      }));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D4, ng, g, s));
    }
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
    bool cond_lora = false;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(XN, D, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(QKV, D3, S_cond.row0);
      g[1].rope_cos = h->crope_cos; g[1].rope_sin = h->crope_sin;
      if (h->use_merged) {
        g[1].W = b.qkv_m;
      } else if (b.l_q.set || b.l_k.set || b.l_v.set) {
        cond_lora = true;
      }
      ng = 2;
    }
    // exact-mode fast path: T for to_q|to_k|to_v|proj_mlp in one launch (both GEMMs read the same XN rows)
    const bool t4 = use_cond && !h->use_merged && (b.l_q.set || b.l_k.set || b.l_v.set) && b.l_mlp.set &&
                    rf::gemm2_lora_eligible(rf::EPI_QKV, D3, D, g[ng - 1]);
    // (forked form: the launch of T happens inside gemm_cond_lora, with all 4 x 64 columns)
    const bool t4_side = t4 && side_lora && ng > 1;
    if (t4 && !t4_side)
      RF_TRY(rf::lora_down_launch(g[ng - 1].A, D, S_cond.rows, D, b.qkvA, 4 * kLoraPad, h->LT, 4 * kLoraPad, s));
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_QKV, D3, D, ng, g, b.qkvA, t4_side ? 4 * kLoraPad : 3 * kLoraPad, b.qkvB, D,
                            [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term_qkv(h, b.qkvA, b.l_q, b.l_k, b.l_v, gc.A, D, S_cond.rows, h->LL, D3, s));
        gc.addend = h->LL; gc.ldadd = D3;
        return 0;
      }, (t4 && !t4_side) ? h->LT : nullptr, 4 * kLoraPad));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_QKV, D3, D, ng, g, s));
    }
    // proj_mlp + GELU -> ACT[:, D:5D]
    memset(g, 0, sizeof(g));
    g[0].A = XN; g[0].lda = D; g[0].M = S_main.rows; g[0].W = b.mlp.w; g[0].bias = b.mlp.b;
    g[0].out = ACT + D; g[0].ldo = D5;
    ng = 1;
    cond_lora = false;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(XN, D, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(ACT, D5, S_cond.row0) + D;
      if (h->use_merged) {
        g[1].W = b.mlp_m;
      } else if (b.l_mlp.set) {
        cond_lora = true;
      }
      ng = 2;
    }
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_GELU, D4, D, ng, g, b.l_mlp.A, kLoraPad, b.l_mlp.B, 0, [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term(h, b.l_mlp, gc.A, D, S_cond.rows, h->LL, D4, s));
        gc.addend = h->LL; gc.ldadd = D4;
        return 0;
      }, t4 ? h->LT + 3 * kLoraPad : nullptr, 4 * kLoraPad));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_GELU, D4, D, ng, g, s));
    }
    // attention -> ACT[:, 0:D]
    at.out = ACT; at.ldo = D5;
    RF_TRY(rf::attention_launch(at, s));
    // proj_out over cat(attn, mlp) (K = 5D) + gate + residual
    memset(g, 0, sizeof(g));
    g[0].A = ACT; g[0].lda = D5; g[0].M = S_main.rows; g[0].W = b.out.w; g[0].bias = b.out.b;
    g[0].out = X; g[0].ldo = D; g[0].res = X; g[0].ldr = D; g[0].gate = mm + 2 * D;
    ng = 1;
    cond_lora = false;
    if (use_cond) {
      g[1] = g[0];
      g[1].A = rowp(ACT, D5, S_cond.row0); g[1].M = S_cond.rows;
      g[1].out = rowp(X, D, S_cond.row0); g[1].res = g[1].out; g[1].gate = mc + 2 * D;
      if (h->use_merged) {
        g[1].W = b.out_m;
      } else if (b.l_out.set) {
        cond_lora = true;
      }
      ng = 2;
    }
    if (cond_lora) {
      RF_TRY(gemm_cond_lora(rf::EPI_GATE_RES, D, D5, ng, g, b.l_out.A, kLoraPad, b.l_out.B, 0, [&](rf::GemmGroupArgs& gc) {
        RF_TRY(lora_term(h, b.l_out, gc.A, D5, S_cond.rows, h->LL, D, s));
        gc.addend = h->LL; gc.ldadd = D;
        return 0;
      }));
    } else {
      RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, D, D5, ng, g, s));
    }
  }

  // ================= norm_out + proj_out (transformer.py:241-244) =================
  const bf16* mo = MOD + mod_out(h, 0);  // [scale | shift]
  RF_TRY(ln(S_img, mo, mo + D));
  memset(g, 0, sizeof(g));
  g[0].A = rowp(XN, D, S_img.row0); g[0].lda = D; g[0].M = S_img.rows; g[0].W = h->proj_out.w;
  g[0].bias = h->proj_out.b; g[0].out = out; g[0].ldo = h->cfg.in_channels;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, h->cfg.in_channels, D, 1, g, s));
  return 0;
}

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
// Wm[n, k] = bf16( W[n, k] + sum_r B[n, r] * A[r, k] ): what peft's fuse_lora / merge() produces
__global__ void lora_merge_kernel(const bf16* __restrict__ W, const bf16* __restrict__ A,
                                  const bf16* __restrict__ B, bf16* __restrict__ Wm, int N, int K,
                                  int R) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  if (k >= K) return;
  float acc = 0.f;
  for (int r = 0; r < R; ++r)
    acc = fmaf(__bfloat162float(B[static_cast<size_t>(n) * R + r]),
               __bfloat162float(A[static_cast<size_t>(r) * K + k]), acc);
  const size_t i = static_cast<size_t>(n) * K + k;
  Wm[i] = __float2bfloat16_rn(__bfloat162float(W[i]) + acc);
}
int lora_merge_launch(const bf16* W, const bf16* A, const bf16* B, bf16* Wm, int N, int K, int R,
                      cudaStream_t stream) {
  dim3 grid((K + 255) / 256, N);
  lora_merge_kernel<<<grid, 256, 0, stream>>>(W, A, B, Wm, N, K, R);
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
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    rf::set_error("rf_dit_create: no CUDA device (this library has no CPU fallback)");
    return -3;
  }
  if (cfg->num_heads <= 0 || cfg->in_channels % 64 != 0 || cfg->joint_attention_dim % 64 != 0 ||
      cfg->pooled_projection_dim % 8 != 0 || cfg->lora_rank < 0 || cfg->lora_rank > kLoraPad) {
    rf::set_error("rf_dit_create: unsupported config");
    return -1;
  }
  rf_dit* h = new rf_dit();
  h->cfg = *cfg;
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
  if (h->side_stream) cudaStreamDestroy(h->side_stream);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
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
    rf::set_error(std::string("rf_dit_set_lora: not a LoRA target (or lora_rank == 0): ") + module);
    return -4;
  }
  if (r <= 0 || r > kLoraPad) {
    rf::set_error("rf_dit_set_lora: rank must be 1..64");
    return -1;
  }
  if (scale != 1.0f) {
    rf::set_error("rf_dit_set_lora: only scaling == 1 (lora_alpha == r, train_flux/config.yaml:50-51) is bit-faithful; other scalings unsupported");
    return -1;
  }
  LoraT& t = *it->second;
  if (in_features != t.in || out_features != t.out) {
    rf::set_error(std::string("rf_dit_set_lora: ") + module + " expects A [r, " + std::to_string(t.in) +
                  "], B [" + std::to_string(t.out) + ", r]; got in=" + std::to_string(in_features) +
                  " out=" + std::to_string(out_features));
    return -4;
  }
  RF_CHECK_CUDA(cudaMemset(t.A, 0, static_cast<size_t>(kLoraPad) * t.in * 2));
  RF_CHECK_CUDA(cudaMemset(t.B, 0, static_cast<size_t>(t.out) * kLoraPad * 2));
  RF_CHECK_CUDA(cudaMemcpy(t.A, A, static_cast<size_t>(r) * t.in * 2, cudaMemcpyDeviceToDevice));
  RF_CHECK_CUDA(cudaMemcpy2D(t.B, kLoraPad * 2, B, static_cast<size_t>(r) * 2,
                             static_cast<size_t>(r) * 2, t.out, cudaMemcpyDeviceToDevice));
  t.set = true;
  h->any_lora = true;
  h->lora_merged = false;
  drop_graph(h);  // the captured step may predate this adapter (different launch list)
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
  if (flags & 1) {
    rf::set_error("rf_dit_prepare: latent_lora=true (LoRA on image tokens) is not implemented");
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
    if (mode != 0 && n_main % 128 != 0) {
      rf::set_error("rf_dit_prepare: cond attention modes need (n_txt + n_img) % 128 == 0");
      return -1;
    }
  }
  const bool same = h->prepared && h->batch == batch && h->n_txt == n_txt && h->n_img == n_img &&
                    h->n_cond == n_cond;
  if (same) drop_graph(h); else free_geometry(h);
  h->flags = flags;
  h->use_merged = (flags & 8) != 0 && h->any_lora && n_cond > 0;
  if (h->use_merged && !h->lora_merged) {
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
    const size_t lrows = static_cast<size_t>(std::max(n_cond, 1));
    if (!(p = A(std::max(lrows * 4 * kLoraPad * 2, static_cast<size_t>(8 * D) * 2)))) return -2; h->LT = static_cast<bf16*>(p);
    if (!(p = A(std::max(lrows * 4 * D * 2, static_cast<size_t>(8 * D) * 2)))) return -2; h->LL = static_cast<bf16*>(p);
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
  // fuse_lora mode: weights or adapters changed since the last merge -> re-merge before use
  h->use_merged = (h->flags & 8) != 0 && h->any_lora && h->n_cond > 0;
  if (h->use_merged && !h->lora_merged) {
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
    if (dev_alloc(h, &p, (static_cast<size_t>(n_steps) * (256 + 3 * h->D) + 256 + 3 * h->D) * 2, true)) return -2;
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
    if (!h->graph_exec) {
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
