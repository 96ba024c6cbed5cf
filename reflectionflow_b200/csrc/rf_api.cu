#include <cstdlib>
// rf_api.cu — operator-level C ABI (include/rf_b200.h) over the kernel launchers, and the host plumbing the
// handles share (rf_internal.h).
#include <algorithm>
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
static std::atomic<int64_t> g_captures{0};

int require_device(const char* who) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error(std::string(who) + ": no CUDA device (this library has no CPU fallback)");
    return -3;
  }
  return 0;
}

void DeviceAllocs::release(void* p) {
  auto it = std::find(blocks_.begin(), blocks_.end(), p);
  if (it == blocks_.end()) return;
  blocks_.erase(it);
  cudaFree(p);
}
void DeviceAllocs::release_all() {
  for (void* p : blocks_) cudaFree(p);
  blocks_.clear();
}

void WeightTable::add(const std::string& key, bf16* dst, int64_t numel, ConvRepack conv) {
  entries_[key] = Entry{dst, numel, conv, false};
}
int WeightTable::load(const char* who, const char* key, const void* src, int64_t numel) {
  auto it = entries_.find(key);
  if (it == entries_.end()) {
    set_error(std::string(who) + ": unknown key " + key);
    return -4;
  }
  Entry& e = it->second;
  if (e.numel != numel) {
    set_error(std::string(who) + ": size mismatch for " + key + ": got " + std::to_string(numel) + ", want " +
              std::to_string(e.numel));
    return -4;
  }
  const ConvRepack& c = e.conv;
  if (c.taps > 0)
    RF_TRY(conv_repack_launch(static_cast<const bf16*>(src), e.dst, c.cout, c.cin, c.taps, c.cout_pad, c.cin_pad,
                              nullptr));
  else
    RF_CHECK_CUDA(cudaMemcpy(e.dst, src, static_cast<size_t>(numel) * 2, cudaMemcpyDeviceToDevice));
  e.loaded = true;
  return 0;
}
int WeightTable::missing(const char* prefix, const char* what) const {
  int n = 0;
  std::string names;
  const size_t pl = strlen(prefix);
  for (auto& kv : entries_)
    if (!kv.second.loaded && kv.first.compare(0, pl, prefix) == 0) {
      if (n < 8) names += kv.first + " ";
      ++n;
    }
  if (n) set_error(std::string(what) + ": " + names + (n > 8 ? "..." : ""));
  return n;
}

int SideStream::enter(cudaStream_t caller, cudaStream_t* s) {
  if (!stream_) {
    RF_CHECK_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&ev_in_, cudaEventDisableTiming));
    RF_CHECK_CUDA(cudaEventCreateWithFlags(&ev_out_, cudaEventDisableTiming));
  }
  RF_CHECK_CUDA(cudaEventRecord(ev_in_, caller));
  RF_CHECK_CUDA(cudaStreamWaitEvent(stream_, ev_in_, 0));
  *s = stream_;
  return 0;
}
int SideStream::leave(cudaStream_t caller) {
  RF_CHECK_CUDA(cudaEventRecord(ev_out_, stream_));
  RF_CHECK_CUDA(cudaStreamWaitEvent(caller, ev_out_, 0));
  return 0;
}
void SideStream::destroy() {
  if (stream_) cudaStreamDestroy(stream_);
  if (ev_in_) cudaEventDestroy(ev_in_);
  if (ev_out_) cudaEventDestroy(ev_out_);
  stream_ = nullptr;
  ev_in_ = ev_out_ = nullptr;
}

int capture_graph(cudaStream_t s, const char* who, const std::function<int()>& body, cudaGraphExec_t* exec,
                  int64_t* launches) {
  RF_CHECK_CUDA(cudaStreamSynchronize(s));
  g_captures.fetch_add(1, std::memory_order_relaxed);
  const int64_t before = launch_count();
  RF_CHECK_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  int rc = body();
  cudaGraph_t graph = nullptr;
  cudaError_t ce = cudaStreamEndCapture(s, &graph);
  *launches = launch_count() - before;
  count_launch(static_cast<int>(-*launches));  // captured, not executed
  if (rc || ce != cudaSuccess) {
    if (graph) cudaGraphDestroy(graph);
    if (!rc) {
      set_error(std::string(who) + ": graph capture failed: " + cudaGetErrorString(ce));
      rc = -2;
    }
    return rc;
  }
  ce = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) {
    *exec = nullptr;
    set_error(std::string(who) + ": cudaGraphInstantiate: " + cudaGetErrorString(ce));
    return -2;
  }
  return 0;
}

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

// Test hooks over the text encoders' launchers (csrc/text.cu): the same host code rf_t5_encode / rf_clip_encode run,
// on caller-owned buffers.  Layouts: rf_internal.h.
int rf_dbg_text_embed(const int* ids, const void* table, const void* pos, void* out, int T, int S, int D,
                      void* stream) {
  return rf::text_embed_launch(ids, static_cast<const bf16*>(table), static_cast<const bf16*>(pos),
                               static_cast<bf16*>(out), T, S, D, static_cast<cudaStream_t>(stream));
}

int rf_dbg_text_rownorm(const void* x, void* out, int rows, int dim, const void* w, const void* b, float eps, int mode,
                        void* stream) {
  return rf::text_rownorm_launch(static_cast<const bf16*>(x), static_cast<bf16*>(out), rows, dim,
                                 static_cast<const bf16*>(w), static_cast<const bf16*>(b), eps, mode,
                                 static_cast<cudaStream_t>(stream));
}

int rf_dbg_text_ewise(const void* a, const void* b, void* out, int64_t n, int mode, void* stream) {
  return rf::text_ewise_launch(static_cast<const bf16*>(a), static_cast<const bf16*>(b), static_cast<bf16*>(out), n,
                               mode, static_cast<cudaStream_t>(stream));
}

int rf_dbg_text_gather_rows(const void* x, const int* pos, void* out, int B, int S, int D, void* stream) {
  return rf::text_gather_rows_launch(static_cast<const bf16*>(x), pos, static_cast<bf16*>(out), B, S, D,
                                     static_cast<cudaStream_t>(stream));
}

int rf_dbg_t5_gated_gelu(const void* x, int T, int D, const void* wi0, const void* wi1, int F, void* h0, void* h1,
                         void* stream) {
  return rf::t5_gated_gelu(static_cast<const bf16*>(x), T, D, static_cast<const bf16*>(wi0),
                           static_cast<const bf16*>(wi1), F, static_cast<bf16*>(h0), static_cast<bf16*>(h1),
                           static_cast<cudaStream_t>(stream));
}

// Test hooks over the VAE's launchers (csrc/vae.cu, the convolution in csrc/gemm_sm90.cu): the same host code
// rf_vae_decode / rf_vae_encode run, on caller-owned buffers.  Layouts: rf_internal.h.
int rf_dbg_vae_conv(const void* in, const void* weight, const void* bias, void* out, const void* res, const void* ones,
                    int H, int W, int Cin, int Cout, int taps, int stride, void* stream) {
  return rf::conv_launch(static_cast<const bf16*>(in), static_cast<const bf16*>(weight), static_cast<const bf16*>(bias),
                         static_cast<bf16*>(out), static_cast<const bf16*>(res), static_cast<const bf16*>(ones), H, W,
                         Cin, Cout, taps, stride, static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_conv_repack(const void* src, void* dst, int Cout, int Cin, int taps, int Cout_pad, int Cin_pad,
                           void* stream) {
  return rf::conv_repack_launch(static_cast<const bf16*>(src), static_cast<bf16*>(dst), Cout, Cin, taps, Cout_pad,
                                Cin_pad, static_cast<cudaStream_t>(stream));
}

// part: rf_dbg_vae_gn_part_floats() floats; mean_rstd: 64 floats (the 32 group means, then the 32 values of 1 / std)
int rf_dbg_vae_gn_part_floats(void) { return rf::gn_part_floats; }
int rf_dbg_vae_group_norm(const void* x, void* out, int H, int W, int C, const void* gamma, const void* beta, int silu,
                          int in_padded, int out_padded, float* part, float* mean_rstd, void* stream) {
  return rf::group_norm_launch(static_cast<const bf16*>(x), static_cast<bf16*>(out), H, W, C,
                               static_cast<const bf16*>(gamma), static_cast<const bf16*>(beta), silu, in_padded,
                               out_padded, part, mean_rstd, static_cast<cudaStream_t>(stream));
}

// the mid-block attention of a loaded rf_vae handle (encoder 0: decoder.mid_block, 1: encoder.mid_block)
int rf_dbg_vae_mid_attention(rf_vae* h, int encoder, const void* x, void* out, int H, int W, void* stream) {
  return vae_mid_attention(h, encoder, static_cast<const bf16*>(x), static_cast<bf16*>(out), H, W,
                           static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_softmax_rows(void* s, int rows, int n, int valid, float scale, void* stream) {
  return rf::softmax_rows_launch(static_cast<bf16*>(s), rows, n, valid, scale, static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_unpack_latents(const void* packed, void* out, int h, int w, float scaling, float shift, void* stream) {
  return rf::unpack_latents_launch(static_cast<const bf16*>(packed), static_cast<bf16*>(out), h, w, scaling, shift,
                                   static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_upsample2x(const void* x, void* out, int H, int W, int C, void* stream) {
  return rf::upsample2x_launch(static_cast<const bf16*>(x), static_cast<bf16*>(out), H, W, C,
                               static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_repad(const void* x, void* out, int H, int W, int C, int in_padded, int out_padded, void* stream) {
  return rf::repad_launch(static_cast<const bf16*>(x), static_cast<bf16*>(out), H, W, C, in_padded, out_padded,
                          static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_transpose(const void* in, int ld_in, void* out, int rows, int cols, void* stream) {
  return rf::transpose_launch(static_cast<const bf16*>(in), ld_in, static_cast<bf16*>(out), rows, cols,
                              static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_postprocess(const void* x, int H, int W, int C, uint8_t* u8, void* chw, void* stream) {
  return rf::postprocess_launch(static_cast<const bf16*>(x), H, W, C, u8, static_cast<bf16*>(chw),
                                static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_image_to_nhwc(const uint8_t* u8, const void* chw, void* out, int H, int W, void* stream) {
  return rf::image_to_nhwc_launch(u8, static_cast<const bf16*>(chw), static_cast<bf16*>(out), H, W,
                                  static_cast<cudaStream_t>(stream));
}

int rf_dbg_vae_sample_pack(const void* mom, int C, const void* eps, void* packed, int h, int w, float scaling,
                           float shift, void* stream) {
  return rf::sample_pack_launch(static_cast<const bf16*>(mom), C, static_cast<const bf16*>(eps),
                                static_cast<bf16*>(packed), h, w, scaling, shift, static_cast<cudaStream_t>(stream));
}


const char* rf_last_error(void) { return rf::get_error(); }
int rf_abi_version(void) { return RF_B200_ABI_VERSION; }
int64_t rf_launch_count(void) { return rf::launch_count(); }
int64_t rf_graph_capture_count(void) { return rf::g_captures.load(std::memory_order_relaxed); }

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

int rf_op_image_guidance_step(void* x, const void* v_cond, const void* v_uncond, const float* scale,
                              const float* sigmas, const int* step, int n, void* stream) {
  if (!x || !v_cond || !v_uncond || !scale || !sigmas || !step) {
    rf::set_error("rf_op_image_guidance_step: null operand");
    return -1;
  }
  return rf::image_guidance_step_launch(static_cast<bf16*>(x), static_cast<const bf16*>(v_cond),
                                        static_cast<const bf16*>(v_uncond), scale, sigmas, step, n,
                                        static_cast<cudaStream_t>(stream));
}

}  // extern "C"
