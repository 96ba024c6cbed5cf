// rf_internal.h — host-side declarations shared by the kernel translation units and the
// DiT orchestrator.  Nothing here is part of the public C ABI (see include/rf_b200.h).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <string>

namespace rf {

typedef __nv_bfloat16 bf16;

// thread-local error string behind rf_last_error()
void set_error(const std::string& msg);
const char* get_error();
// launch accounting behind rf_launch_count()
void count_launch(int n = 1);
int64_t launch_count();

#define RF_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::rf::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));               \
      return -2;                                                                         \
    }                                                                                    \
  } while (0)

// Launch with programmatic stream serialization (PDL) unless RF_PDL=0: the kernel MUST call
// pdl_wait() (rf_ptx.cuh) before its first global-memory access.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Optional per-launch timing (rf_profile_start/stop): CUDA events around every kernel launch on
// the launching stream, aggregated per kernel name with its algorithmic FLOPs / bytes.
bool prof_on();  // rf_profile_start() is active: per-launch events are being recorded (graphs are bypassed)
struct ProfScope {
  ProfScope(const char* name, double flops, double bytes, cudaStream_t stream);
  ~ProfScope();
  int idx;
  cudaStream_t stream;
};

// Encode a 2-D bf16 row-major tensor map with 128-byte swizzle.
//   rows x cols elements, row pitch ld (elements); box = box_rows x 64 columns.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols = 64);

// 3-D bf16 NHWC image map {C, Wp, Hp} with 128-byte swizzle; box {64, box_x, box_y} elements of the
// traversed (strided) lattice, i.e. the box spans box_x * stride pixels in x.
int make_tmap_3d(CUtensorMap* out, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp,
                 uint32_t box_x, uint32_t box_y, uint32_t stride);

// ---------------------------------------------------------------------------- GEMM
enum GemmEpilogue {
  EPI_BIAS = 0,      // out = bf16(acc + bias)
  EPI_GELU = 1,      // out = bf16(gelu_tanh(bf16(acc + bias)))
  EPI_GATE_RES = 2,  // out = bf16(res + bf16(gate[n] * bf16(acc + bias)))
  EPI_QKV = 3,       // q,k sections: per-head RMSNorm * w, interleaved RoPE; v: bias only
  EPI_SCALE = 4,     // out = bf16(bf16(acc + bias) * lora_scale[0]): peft's scaled low-rank term, unfused
};

// One member of a grouped GEMM: out[M, N] = epi(A[M, K] @ W[N, K]^T).  All groups of a
// launch share N, K and the epilogue kind; they differ in operands (token streams).
struct GemmGroupArgs {
  const bf16* A;   int lda;  int M;
  const bf16* W;             // [N, K] row-major (torch Linear weight layout), ld = K
  const bf16* bias;          // [N] or nullptr
  bf16* out;       int ldo;
  const bf16* addend; int ldadd;   // optional [M, N] term added after the bias rounding (LoRA)
  const bf16* res; int ldr;        // EPI_GATE_RES
  const bf16* gate;                // EPI_GATE_RES: [N]
  const float* rope_cos;           // EPI_QKV: [M, 64] (pair-compact), row index local to group
  const float* rope_sin;
  const bf16* norm_q;              // EPI_QKV: [128]
  const bf16* norm_k;
  // peft's unfused LoRA arithmetic fused into this group's tiles (lora_T != nullptr):
  //   out = epi( bf16( bf16(A W^T + b) + bf16( bf16(T lora_B^T) * lora_scale[s] ) ) ),
  //   T = bf16(A loraA^T) computed beforehand.
  // T: [M, ld_t]; with lora_sec_cols > 0 output section s = n / lora_sec_cols reads T columns
  // [lora_pad s, lora_pad (s + 1)) (stacked q|k|v), else s = 0 and T columns [0, lora_pad); lora_B: [N, lora_pad]
  // (rank zero-padded to lora_pad = 64 or 128: one or two 64-deep low-rank k-blocks).  lora_scale[s] is the
  // fp32 peft scaling of section s (1: the multiply is the identity).  See gemm_lora_eligible.
  // EPI_SCALE reads lora_scale[0] as its output scale.
  const bf16* lora_T; int ld_t;
  const bf16* lora_B;
  int lora_sec_cols;
  int lora_pad;
  float lora_scale[3];
};
int gemm_launch(int epi, int N, int K, int ngroups, const GemmGroupArgs* groups,
                cudaStream_t stream);

// Whether group `a` (without its lora_* fields) can carry the fused LoRA term in gemm_launch.
bool gemm_lora_eligible(int epi, int N, int K, const GemmGroupArgs& a);

// LoRA down-projection of one token stream: T[M, NT] = bf16(X[M, K] @ A[NT, K]^T), NT a multiple of 64,
// on the GEMM kernel above (fp32 accumulation over the whole K, one rounding).
int lora_down_launch(const bf16* X, int ldx, int M, int K, const bf16* A, int NT, bf16* T, int ldT,
                     cudaStream_t stream);
// The same for up to 3 token streams in one launch, each group with its own rows (A, lda, M), its own A factor
// (W: [NT, K]) and its own T (out, ldo): e.g. the text rows with the text stream's factors and the image + condition
// rows with the shared ones.  bias, epilogue and LoRA fields of the groups must be zero.
int lora_down_launch(int K, int NT, int ngroups, const GemmGroupArgs* groups, cudaStream_t stream);

// ---------------------------------------------------------------------------- attention
// Non-causal softmax(Q K^T / sqrt(128)) V over one joint token sequence.
// q, k, v: token-major [n_tok, heads*128] slices of one buffer (see attn_sm90.cu)
struct AttnArgs {
  const bf16* q; const bf16* k; const bf16* v;  // each [n_tok, heads*128] slices, pitch ld_qkv
  int ld_qkv;
  bf16* out; int ldo;                           // [n_tok, heads*128], pitch ldo
  int n_tok; int heads; int batch;              // rows of batch b start at b*n_tok
  int n_main;                                   // tokens [0, n_main) vs [n_main, n_tok) = cond
  int cond_mode;                                // 0 none, 1 additive log-bias, 2 block mask
  float cond_bias;                              // log(c_factor) when cond_mode == 1
};
int attention_launch(const AttnArgs& a, cudaStream_t stream);

// T5 / CLIP self-attention, head_dim 64, S <= 512, on wgmma (text_attn_sm90.cu): eager-attention
// rounding points (scores -> bf16 [* scale -> bf16] [+ bias -> bf16], fp32 softmax -> bf16, PV -> bf16)
bool text_attn_tc_eligible(int S, int ld, int ldo);
int text_attn_tc_launch(const bf16* q, const bf16* k, const bf16* v, int ld, bf16* out, int ldo, int B, int S,
                        int heads, const bf16* bias, float scale, int use_scale, int causal, cudaStream_t stream);

// ---------------------------------------------------------------------------- bandwidth kernels
// out = bf16(bf16(bf16(LN(x)) * bf16(1 + scale)) + shift)   (LN: no affine, eps 1e-6)
//   rows of batch element b (= row / rows_per_batch) use scale/shift + b * mod_stride
int ln_modulate_launch(const bf16* x, int ldx, bf16* out, int ldo, int rows, int dim,
                       const bf16* scale, const bf16* shift, int rows_per_batch, int mod_stride,
                       cudaStream_t stream);
// same, for up to 3 consecutive row ranges of one buffer (token streams), each with its own vectors:
// rows [0, row_end[0]) use (scale[0], shift[0]), rows [row_end[0], row_end[1]) the next, ...
int ln_modulate_grouped_launch(const bf16* x, int ldx, bf16* out, int ldo, int dim, int ngroups,
                               const int* row_end, const bf16* const* scale, const bf16* const* shift,
                               cudaStream_t stream);
// y[n] = bf16(sum_k act(x[k]) * W[n, k] + b[n]) for `batch` input vectors.
//   act: 0 identity, 1 = bf16(silu(x))
int gemv_launch(const bf16* x, int ldx, int batch, const bf16* W, const bf16* bias, bf16* y,
                int ldy, int N, int K, int act, cudaStream_t stream);
// sinusoidal timestep projection (256 channels, flip_sin_to_cos) of a bf16 scalar * 1000
//   t value of batch b = t[b * t_stride + (step ? *step : 0)]
int timestep_embed_launch(const bf16* t, const int* step, int t_stride, float pre_scale, bf16* out,
                          int batch, cudaStream_t stream);
int advance_step_launch(int* step, cudaStream_t stream);
// out = bf16(a + b + c) evaluated left to right with bf16 rounding after each add
int add3_launch(const bf16* a, const bf16* b, const bf16* c, bf16* out, int n,
                cudaStream_t stream);
// x = bf16(float(x) + dt * float(v))
int euler_step_launch(bf16* x, const bf16* v, const float* sigmas, const int* step, int n,
                      cudaStream_t stream);
int copy_rows_launch(const bf16* src, int lds, bf16* dst, int ldd, int rows, int cols,
                     cudaStream_t stream);
// dst[r * ldd + c] = bf16(dst[r * ldd + c] + bf16(src[r * lds + c] * scale)) for r < rows, c < cols
int add_rows_launch(bf16* dst, int64_t ldd, const bf16* src, int lds, int rows, int cols, float scale,
                    cudaStream_t stream);
// Wm[n, k] = bf16(W[n, k] + scale * sum_r B[n, r] A[r, k]) (peft's merged weight; W, Wm [N, K], A [R, K], B [N, R])
int lora_merge_launch(const bf16* W, const bf16* A, const bf16* B, bf16* Wm, int N, int K, int R, float scale,
                      cudaStream_t stream);

}  // namespace rf
