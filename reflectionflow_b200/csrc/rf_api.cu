#include <cstdlib>
// rf_api.cu — operator-level C ABI (include/rf_b200.h) over the kernel launchers.
#include <atomic>
#include <cstring>
#include <map>
#include <vector>

#include "../../include/rf_b200.h"
#include "rf_internal.h"

namespace rf {
bool pdl_enabled() {
  // opt-in (RF_PDL=1): the default is plain stream order
  static const bool on = getenv("RF_PDL") && getenv("RF_PDL")[0] == '1';
  return on;
}

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* get_error() { return g_err.c_str(); }
static std::atomic<int64_t> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }

struct ProfRec {
  const char* name;
  double flops, bytes;
  cudaEvent_t e0, e1;
};
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
bool prof_on() { return g_prof_on; }
ProfScope::ProfScope(const char* name, double flops, double bytes, cudaStream_t s)
    : idx(-1), stream(s) {
  if (!g_prof_on) return;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) return;
  ProfRec r{name, flops, bytes, nullptr, nullptr};
  if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
  cudaEventRecord(r.e0, s);
  g_prof.push_back(r);
  idx = static_cast<int>(g_prof.size()) - 1;
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(g_prof[idx].e1, stream);
}
}  // namespace rf

using rf::bf16;
namespace rf {
int resize_u8_launch(const uint8_t* in, int H, int W, uint8_t* tmp, uint8_t* out, int OH, int OW,
                     const int* bx, const int* kx, int ksx, const int* by, const int* ky, int ksy,
                     cudaStream_t stream);
}
namespace rf { void dbg_force_gemm_v1(bool on); }

extern "C" {

// test hook: 1 = the next GEMM launches use tiles at most 128 wide (covers both tile widths at small shapes)
void rf_dbg_force_gemm_v1(int on) { rf::dbg_force_gemm_v1(on != 0); }

// Test hooks over the internal launchers the DiT orchestrator calls (not declared in include/rf_b200.h): the grouped
// GEMM with every epilogue and the fused LoRA fields, the grouped LoRA down-projection, the grouped LayerNorm +
// modulate, the adaLN / embedder LoRA add and the fuse_lora merge.  rf_dbg_gemm_group mirrors rf::GemmGroupArgs
// field by field; rf_dbg_gemm_group_size() lets a binding check its copy of the layout.
struct rf_dbg_gemm_group {
  const void* A; int lda; int M;
  const void* W;
  const void* bias;
  void* out; int ldo;
  const void* addend; int ldadd;
  const void* res; int ldr;
  const void* gate;
  const float* rope_cos;
  const float* rope_sin;
  const void* norm_q;
  const void* norm_k;
  const void* lora_T; int ld_t;
  const void* lora_B;
  int lora_sec_cols;
  int lora_pad;
  float lora_scale[3];
};

size_t rf_dbg_gemm_group_size(void) { return sizeof(rf_dbg_gemm_group); }

static int dbg_groups(int ngroups, const rf_dbg_gemm_group* src, rf::GemmGroupArgs* dst) {
  if (!src || ngroups < 1 || ngroups > 3) {
    rf::set_error("rf_dbg: 1..3 groups");
    return -1;
  }
  memset(dst, 0, 3 * sizeof(rf::GemmGroupArgs));
  for (int i = 0; i < ngroups; ++i) {
    const rf_dbg_gemm_group& s = src[i];
    rf::GemmGroupArgs& d = dst[i];
    d.A = static_cast<const bf16*>(s.A); d.lda = s.lda; d.M = s.M;
    d.W = static_cast<const bf16*>(s.W);
    d.bias = static_cast<const bf16*>(s.bias);
    d.out = static_cast<bf16*>(s.out); d.ldo = s.ldo;
    d.addend = static_cast<const bf16*>(s.addend); d.ldadd = s.ldadd;
    d.res = static_cast<const bf16*>(s.res); d.ldr = s.ldr;
    d.gate = static_cast<const bf16*>(s.gate);
    d.rope_cos = s.rope_cos; d.rope_sin = s.rope_sin;
    d.norm_q = static_cast<const bf16*>(s.norm_q);
    d.norm_k = static_cast<const bf16*>(s.norm_k);
    d.lora_T = static_cast<const bf16*>(s.lora_T); d.ld_t = s.ld_t;
    d.lora_B = static_cast<const bf16*>(s.lora_B);
    d.lora_sec_cols = s.lora_sec_cols;
    d.lora_pad = s.lora_pad;
    for (int k = 0; k < 3; ++k) d.lora_scale[k] = s.lora_scale[k];
  }
  return 0;
}

int rf_dbg_gemm_grouped(int epi, int N, int K, int ngroups, const rf_dbg_gemm_group* g, void* stream) {
  rf::GemmGroupArgs a[3];
  if (int rc = dbg_groups(ngroups, g, a)) return rc;
  return rf::gemm_launch(epi, N, K, ngroups, a, static_cast<cudaStream_t>(stream));
}

int rf_dbg_lora_down_grouped(int K, int NT, int ngroups, const rf_dbg_gemm_group* g, void* stream) {
  rf::GemmGroupArgs a[3];
  if (int rc = dbg_groups(ngroups, g, a)) return rc;
  return rf::lora_down_launch(K, NT, ngroups, a, static_cast<cudaStream_t>(stream));
}

int rf_dbg_ln_modulate_grouped(const void* x, int ldx, void* out, int ldo, int dim, int ngroups, const int* row_end,
                               const void* const* scale, const void* const* shift, void* stream) {
  if (!x || !out || !row_end || !scale || !shift || ngroups < 1 || ngroups > 3) {
    rf::set_error("rf_dbg_ln_modulate_grouped: null operand or not 1..3 groups");
    return -1;
  }
  const bf16* sc[3] = {nullptr, nullptr, nullptr};
  const bf16* sh[3] = {nullptr, nullptr, nullptr};
  for (int i = 0; i < ngroups; ++i) {
    sc[i] = static_cast<const bf16*>(scale[i]);
    sh[i] = static_cast<const bf16*>(shift[i]);
  }
  return rf::ln_modulate_grouped_launch(static_cast<const bf16*>(x), ldx, static_cast<bf16*>(out), ldo, dim, ngroups,
                                        row_end, sc, sh, static_cast<cudaStream_t>(stream));
}

int rf_dbg_add_rows(void* dst, int64_t ldd, const void* src, int lds, int rows, int cols, float scale, void* stream) {
  return rf::add_rows_launch(static_cast<bf16*>(dst), ldd, static_cast<const bf16*>(src), lds, rows, cols, scale,
                             static_cast<cudaStream_t>(stream));
}

int rf_dbg_lora_merge(const void* W, const void* A, const void* B, void* Wm, int N, int K, int R, float scale,
                      void* stream) {
  return rf::lora_merge_launch(static_cast<const bf16*>(W), static_cast<const bf16*>(A), static_cast<const bf16*>(B),
                               static_cast<bf16*>(Wm), N, K, R, scale, static_cast<cudaStream_t>(stream));
}

// the T5 / CLIP attention on the tensor-core path the encoders run (text.cu: small_attn); refuses shapes that path
// does not take instead of falling back to the CUDA-core kernel
int rf_dbg_text_attention(const void* q, const void* k, const void* v, int ld, void* out, int ldo, int B, int S,
                          int heads, const void* bias, float scale, int use_scale, int causal, void* stream) {
  if (!q || !k || !v || !out || B <= 0 || heads <= 0) {
    rf::set_error("rf_dbg_text_attention: null operand or empty problem");
    return -1;
  }
  if (!rf::text_attn_tc_eligible(S, ld, ldo)) {
    rf::set_error("rf_dbg_text_attention: needs 1 <= S <= 512 and 16-byte row pitches");
    return -1;
  }
  return rf::text_attn_tc_launch(static_cast<const bf16*>(q), static_cast<const bf16*>(k), static_cast<const bf16*>(v),
                                 ld, static_cast<bf16*>(out), ldo, B, S, heads, static_cast<const bf16*>(bias), scale,
                                 use_scale, causal, static_cast<cudaStream_t>(stream));
}


const char* rf_last_error(void) { return rf::get_error(); }
int rf_abi_version(void) { return RF_B200_ABI_VERSION; }
int64_t rf_launch_count(void) { return rf::launch_count(); }

int rf_profile_start(void) {
  for (auto& r : rf::g_prof) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  rf::g_prof.clear();
  rf::g_prof_on = true;
  return 0;
}

int rf_profile_stop(char* json_out, int capacity) {
  rf::g_prof_on = false;
  if (cudaDeviceSynchronize() != cudaSuccess) {
    rf::set_error("rf_profile_stop: device synchronize failed");
    return -2;
  }
  struct Agg { int n = 0; double ms = 0, flops = 0, bytes = 0; };
  std::map<std::string, Agg> agg;
  for (auto& r : rf::g_prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    Agg& a = agg[r.name];
    a.n += 1; a.ms += ms; a.flops += r.flops; a.bytes += r.bytes;
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  rf::g_prof.clear();
  std::string js = "{";
  bool first = true;
  for (auto& kv : agg) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s\"%s\": {\"launches\": %d, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}",
             first ? "" : ", ", kv.first.c_str(), kv.second.n, kv.second.ms, kv.second.flops,
             kv.second.bytes);
    js += buf;
    first = false;
  }
  js += "}";
  if (!json_out || capacity <= static_cast<int>(js.size())) {
    rf::set_error("rf_profile_stop: buffer too small");
    return -1;
  }
  memcpy(json_out, js.c_str(), js.size() + 1);
  return 0;
}

int rf_op_linear(int epilogue, int M, int N, int K, const void* x, int ldx, const void* W,
                 const void* bias, void* y, int ldy, const void* addend, int ld_addend,
                 const void* res, int ld_res, const void* gate, const float* rope_cos,
                 const float* rope_sin, const void* norm_q, const void* norm_k, void* stream) {
  if (!x || !W || !y) {
    rf::set_error("rf_op_linear: null operand");
    return -1;
  }
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = static_cast<const bf16*>(x); g.lda = ldx; g.M = M;
  g.W = static_cast<const bf16*>(W);
  g.bias = static_cast<const bf16*>(bias);
  g.out = static_cast<bf16*>(y); g.ldo = ldy;
  g.addend = static_cast<const bf16*>(addend); g.ldadd = ld_addend;
  g.res = static_cast<const bf16*>(res); g.ldr = ld_res;
  g.gate = static_cast<const bf16*>(gate);
  g.rope_cos = rope_cos; g.rope_sin = rope_sin;
  g.norm_q = static_cast<const bf16*>(norm_q);
  g.norm_k = static_cast<const bf16*>(norm_k);
  return rf::gemm_launch(epilogue, N, K, 1, &g, static_cast<cudaStream_t>(stream));
}

size_t rf_op_linear_lora_workspace_bytes(int M) {
  const size_t rows = (static_cast<size_t>(M > 0 ? M : 1) + 127) / 128 * 128;
  return rows * 192 * 2 + 256;
}

int rf_op_linear_lora(int epilogue, int M, int N, int K, const void* x, int ldx, const void* W,
                      const void* bias, void* y, int ldy, const void* lora_A, int t_cols,
                      const void* lora_B, const void* res, int ld_res, const void* gate,
                      const float* rope_cos, const float* rope_sin, const void* norm_q,
                      const void* norm_k, void* workspace, void* stream) {
  if (!x || !W || !y || !lora_A || !lora_B || !workspace) {
    rf::set_error("rf_op_linear_lora: null operand");
    return -1;
  }
  if (t_cols != 64 && t_cols != 192) {
    rf::set_error("rf_op_linear_lora: t_cols must be 64 (one target) or 192 (stacked q|k|v)");
    return -1;
  }
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = static_cast<const bf16*>(x); g.lda = ldx; g.M = M;
  g.W = static_cast<const bf16*>(W);
  g.bias = static_cast<const bf16*>(bias);
  g.out = static_cast<bf16*>(y); g.ldo = ldy;
  g.res = static_cast<const bf16*>(res); g.ldr = ld_res;
  g.gate = static_cast<const bf16*>(gate);
  g.rope_cos = rope_cos; g.rope_sin = rope_sin;
  g.norm_q = static_cast<const bf16*>(norm_q);
  g.norm_k = static_cast<const bf16*>(norm_k);
  if (!rf::gemm_lora_eligible(epilogue, N, K, g)) {
    rf::set_error("rf_op_linear_lora: needs M >= 128, N % 128 == 0 (QKV: N % 384 == 0), K % 64 == 0, "
                  "16-byte aligned pitches, and the GELU / GATE_RES / QKV epilogue");
    return -1;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // workspace = T (bf16 [rows, t_cols])
  bf16* T = static_cast<bf16*>(workspace);
  int rc = rf::lora_down_launch(g.A, ldx, M, K, static_cast<const bf16*>(lora_A), t_cols, T, t_cols, s);
  if (rc) return rc;
  g.lora_T = T; g.ld_t = t_cols;
  g.lora_B = static_cast<const bf16*>(lora_B);
  g.lora_sec_cols = t_cols == 192 ? N / 3 : 0;
  g.lora_pad = 64;
  g.lora_scale[0] = g.lora_scale[1] = g.lora_scale[2] = 1.f;
  return rf::gemm_launch(epilogue, N, K, 1, &g, s);
}

int rf_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out,
                    int n_tok, int heads, int batch, int n_main, int cond_mode, float cond_bias,
                    void* stream) {
  if (!q || !k || !v || !out) {
    rf::set_error("rf_op_attention: null operand");
    return -1;
  }
  rf::AttnArgs a;
  a.q = static_cast<const bf16*>(q); a.k = static_cast<const bf16*>(k);
  a.v = static_cast<const bf16*>(v); a.ld_qkv = ld_qkv;
  a.out = static_cast<bf16*>(out); a.ldo = ld_out;
  a.n_tok = n_tok; a.heads = heads; a.batch = batch;
  a.n_main = n_main; a.cond_mode = cond_mode; a.cond_bias = cond_bias;
  return rf::attention_launch(a, static_cast<cudaStream_t>(stream));
}

int rf_op_ln_modulate(const void* x, int ldx, void* out, int ld_out, int rows, int dim,
                      const void* scale, const void* shift, int rows_per_batch, int mod_stride,
                      void* stream) {
  if (!x || !out || !scale || !shift) {
    rf::set_error("rf_op_ln_modulate: null operand");
    return -1;
  }
  return rf::ln_modulate_launch(static_cast<const bf16*>(x), ldx, static_cast<bf16*>(out), ld_out,
                                rows, dim, static_cast<const bf16*>(scale),
                                static_cast<const bf16*>(shift), rows_per_batch, mod_stride,
                                static_cast<cudaStream_t>(stream));
}

int rf_op_gemv(const void* x, int ldx, int batch, const void* W, const void* bias, void* y, int ldy,
               int N, int K, int act, void* stream) {
  if (!x || !W || !y) {
    rf::set_error("rf_op_gemv: null operand");
    return -1;
  }
  return rf::gemv_launch(static_cast<const bf16*>(x), ldx, batch, static_cast<const bf16*>(W),
                         static_cast<const bf16*>(bias), static_cast<bf16*>(y), ldy, N, K, act,
                         static_cast<cudaStream_t>(stream));
}

int rf_op_timestep_embed(const void* t, float pre_scale, void* out, int batch, void* stream) {
  if (!t || !out) {
    rf::set_error("rf_op_timestep_embed: null operand");
    return -1;
  }
  return rf::timestep_embed_launch(static_cast<const bf16*>(t), nullptr, 1, pre_scale,
                                   static_cast<bf16*>(out), batch,
                                   static_cast<cudaStream_t>(stream));
}

int rf_op_resize_u8(const uint8_t* in_hwc, int H, int W, uint8_t* tmp, uint8_t* out_hwc, int out_h,
                    int out_w, const int* bounds_x, const int* coef_x, int ksize_x, const int* bounds_y,
                    const int* coef_y, int ksize_y, void* stream) {
  if (!in_hwc || !tmp || !out_hwc || !bounds_x || !coef_x || !bounds_y || !coef_y) {
    rf::set_error("rf_op_resize_u8: null operand");
    return -1;
  }
  return rf::resize_u8_launch(in_hwc, H, W, tmp, out_hwc, out_h, out_w, bounds_x, coef_x, ksize_x,
                              bounds_y, coef_y, ksize_y, static_cast<cudaStream_t>(stream));
}

int rf_op_euler_step(void* x, const void* v, const float* sigmas, const int* step, int n,
                     void* stream) {
  if (!x || !v || !sigmas || !step) {
    rf::set_error("rf_op_euler_step: null operand");
    return -1;
  }
  return rf::euler_step_launch(static_cast<bf16*>(x), static_cast<const bf16*>(v), sigmas, step, n,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
