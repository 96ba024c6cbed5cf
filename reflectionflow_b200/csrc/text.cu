// text.cu — T5 encoder (T5-v1.1-XXL shape) and CLIP text encoder on sm_90a, behind rf_text_* (C ABI).
//
// Replaces `pipe.text_encoder_2(ids)[0]` (T5, prompt_embeds [B, 512, 4096]) and
// `pipe.text_encoder(ids).pooler_output` (CLIP-L, pooled [B, 768]) inside diffusers
// FluxPipeline.encode_prompt, called once per candidate at train_flux/flux/generate.py:148-161 (via
// pipeline_tools.py:33-52) — each reflection candidate has its own refined prompt
// (tts/tts_reflectionflow.py:286-294).  Token ids in (tokenizers stay on the host), embeddings out.
//
// All Linear layers run on the wgmma GEMM kernel of this library (fused residual / GELU
// epilogues); the pieces specific to the text encoders are small bandwidth kernels here: T5 RMSNorm,
// affine LayerNorm, embedding gathers, the gated-GELU product, quick-GELU, and a shared-memory
// attention for short sequences with head_dim 64 (T5: additive relative-position bias, no scaling;
// CLIP: causal mask, 1/8 scaling) that keeps the rounding points of the transformers "eager" path:
// scores -> bf16, + bias -> bf16, softmax in fp32 -> bf16, P V -> bf16.
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/rf_b200.h"
#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

__device__ __forceinline__ float warp_sum_t(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_t(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// out[t, :] = table[ids[t], :] (+ pos[t % S, :] in bf16)
__global__ void embed_kernel(const int* __restrict__ ids, const bf16* __restrict__ table,
                             const bf16* __restrict__ pos, bf16* __restrict__ out, int T, int S, int D) {
  const int t = blockIdx.x;
  if (t >= T) return;
  const uint4* src = reinterpret_cast<const uint4*>(table + static_cast<size_t>(ids[t]) * D);
  const uint4* ps = pos ? reinterpret_cast<const uint4*>(pos + static_cast<size_t>(t % S) * D) : nullptr;
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * D);
  for (int i = threadIdx.x; i < D / 8; i += blockDim.x) {
    uint4 u = __ldg(src + i);
    if (ps) {
      const uint4 p = __ldg(ps + i);
      const uint32_t a[4] = {u.x, u.y, u.z, u.w}, b[4] = {p.x, p.y, p.z, p.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 x = unpack_bf16x2(a[q]), y = unpack_bf16x2(b[q]);
        o[q] = pack_bf16x2(x.x + y.x, x.y + y.y);
      }
      u = make_uint4(o[0], o[1], o[2], o[3]);
    }
    dst[i] = u;
  }
}

// T5LayerNorm: y = w * bf16(x * rsqrt(mean(x^2) + eps))   (fp32 statistics, no mean subtraction)
// affine LayerNorm (mode 1): y = bf16((x - mean) * rstd * w + b)
__global__ void __launch_bounds__(256)
rownorm_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int rows, int dim,
               const bf16* __restrict__ w, const bf16* __restrict__ b, float eps, int mode) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * dim);
  const int nch = dim / 8;
  float s = 0.f, q = 0.f;
  for (int i = lane; i < nch; i += 32) {
    const uint4 u = __ldg(xr + i);
    const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(ww[k]);
      s += f.x + f.y;
      q = fmaf(f.x, f.x, q);
      q = fmaf(f.y, f.y, q);
    }
  }
  s = warp_sum_t(s);
  q = warp_sum_t(q);
  float mean = 0.f, rstd;
  if (mode == 0) {
    rstd = __fdiv_rn(1.0f, __fsqrt_rn(q / dim + eps));
  } else {
    mean = s / dim;
    float var = 0.f;  // second pass for the variance (row is L1/L2 resident)
    for (int i = lane; i < nch; i += 32) {
      const uint4 u = __ldg(xr + i);
      const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16x2(ww[k]);
        var = fmaf(f.x - mean, f.x - mean, var);
        var = fmaf(f.y - mean, f.y - mean, var);
      }
    }
    var = warp_sum_t(var) / dim;
    rstd = __fdiv_rn(1.0f, __fsqrt_rn(var + eps));
  }
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * dim);
  for (int i = lane; i < nch; i += 32) {
    const uint4 u = __ldg(xr + i);
    const uint4 uw = __ldg(reinterpret_cast<const uint4*>(w) + i);
    uint4 ub = make_uint4(0, 0, 0, 0);
    if (mode == 1) ub = __ldg(reinterpret_cast<const uint4*>(b) + i);
    const uint32_t xs[4] = {u.x, u.y, u.z, u.w}, ws[4] = {uw.x, uw.y, uw.z, uw.w},
                   bs[4] = {ub.x, ub.y, ub.z, ub.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(xs[k]), g = unpack_bf16x2(ws[k]), bb = unpack_bf16x2(bs[k]);
      float y0, y1;
      if (mode == 0) {
        y0 = __fmul_rn(g.x, bf16_round(__fmul_rn(f.x, rstd)));
        y1 = __fmul_rn(g.y, bf16_round(__fmul_rn(f.y, rstd)));
      } else {
        y0 = (f.x - mean) * rstd * g.x + bb.x;
        y1 = (f.y - mean) * rstd * g.y + bb.y;
      }
      o[k] = pack_bf16x2(y0, y1);
    }
    orow[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// out = bf16(a * b)  (gated-GELU product)   |  mode 1: out = bf16(a * sigmoid(1.702 a)) (quick_gelu)
// (a and out may alias: every thread reads its 8 elements before writing them)
__global__ void ewise_kernel(const bf16* a, const bf16* b, bf16* out, long long n8, int mode) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 ua = reinterpret_cast<const uint4*>(a)[i];
  uint4 ub = make_uint4(0, 0, 0, 0);
  if (mode == 0) ub = reinterpret_cast<const uint4*>(b)[i];
  const uint32_t xs[4] = {ua.x, ua.y, ua.z, ua.w}, ys[4] = {ub.x, ub.y, ub.z, ub.w};
  uint32_t o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 x = unpack_bf16x2(xs[k]), y = unpack_bf16x2(ys[k]);
    if (mode == 0) {
      o[k] = pack_bf16x2(x.x * y.x, x.y * y.y);
    } else {  // x * sigmoid(1.702 x): torch evaluates sigmoid(bf16(1.702 x)) in fp32 and rounds, then multiplies
      const float s0 = bf16_round(1.0f / (1.0f + expf(-bf16_round(1.702f * x.x))));
      const float s1 = bf16_round(1.0f / (1.0f + expf(-bf16_round(1.702f * x.y))));
      o[k] = pack_bf16x2(x.x * s0, x.y * s1);
    }
  }
  reinterpret_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

// Attention for short sequences, head_dim 64.  q/k/v: [B*S, ld] slices (head h at columns h*64),
// out [B*S, ldo].  grid (ceil(S/32), heads, B), 256 threads.  K^T (bf16 pairs of adjacent keys per
// word) and V of the head live in shared memory; each warp owns 4 query rows and register-blocks
// 4 rows x 2 keys (scores) / 4 rows x 2 channels (P V) so that one LDS.32 + one broadcast LDS.128
// feed 8 FMAs.  A lane only ever re-reads the score columns it wrote itself until the P V pass.
//   scores = bf16(q.k) [ = bf16(scores * scale) ] [ = bf16(scores + bias[h, i, j]) ] ; causal: j <= i
//   p = bf16(softmax_fp32(scores)) ; out = bf16(sum_j p_j v_j)
__host__ __device__ inline int small_attn_sp2(int S) { return ((S + 1) / 2) | 1; }  // odd word pitch: conflict-free fill

__global__ void __launch_bounds__(256)
small_attn_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                  int ld, bf16* __restrict__ out, int ldo, int S, const bf16* __restrict__ bias,
                  float scale, int use_scale, int causal) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  const int Sp2 = small_attn_sp2(S);
  float4* sc4 = reinterpret_cast<float4*>(sm_raw);                      // [8 warps][S] x (4 rows)
  float4* q4 = sc4 + 8 * S;                                            // [8 warps][64] x (4 rows)
  uint32_t* vs2 = reinterpret_cast<uint32_t*>(q4 + 8 * 64);            // [S][32] bf16x2
  uint32_t* kt2 = vs2 + S * 32;                                        // [64][Sp2] bf16x2 (keys 2m, 2m+1)
  bf16* ktb = reinterpret_cast<bf16*>(kt2);
  const int h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t base = static_cast<size_t>(b) * S;
  for (int i = threadIdx.x; i < S * 32; i += blockDim.x) {
    const int j = i >> 5, dp = i & 31;
    const uint32_t kk = *reinterpret_cast<const uint32_t*>(k + (base + j) * ld + h * 64 + 2 * dp);
    vs2[i] = *reinterpret_cast<const uint32_t*>(v + (base + j) * ld + h * 64 + 2 * dp);
    reinterpret_cast<uint16_t*>(ktb)[(2 * dp) * (2 * Sp2) + j] = static_cast<uint16_t>(kk & 0xffffu);
    reinterpret_cast<uint16_t*>(ktb)[(2 * dp + 1) * (2 * Sp2) + j] = static_cast<uint16_t>(kk >> 16);
  }
  if (S & 1)  // the odd tail key of each K^T row is read (and discarded): keep it finite
    for (int d = threadIdx.x; d < 64; d += blockDim.x) reinterpret_cast<uint16_t*>(ktb)[d * (2 * Sp2) + S] = 0;
  const int i0 = blockIdx.x * 32 + warp * 4;
  float4* myq = q4 + warp * 64;
  {  // q rows of this warp, interleaved [d][row]
    float qv[4][2];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = min(i0 + r, S - 1);
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q + (base + i) * ld + h * 64 + 2 * lane));
      qv[r][0] = f.x;
      qv[r][1] = f.y;
    }
    myq[2 * lane] = make_float4(qv[0][0], qv[1][0], qv[2][0], qv[3][0]);
    myq[2 * lane + 1] = make_float4(qv[0][1], qv[1][1], qv[2][1], qv[3][1]);
  }
  __syncthreads();
  if (i0 >= S) return;
  float4* my = sc4 + warp * S;
  float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (int kb = 0; kb < S; kb += 64) {
    const int jw = min(kb / 2 + lane, Sp2 - 1);
    float acc[4][2] = {};
#pragma unroll 8
    for (int d = 0; d < 64; ++d) {
      const float2 kk = unpack_bf16x2(kt2[d * Sp2 + jw]);
      const float4 qq = myq[d];
      acc[0][0] = fmaf(qq.x, kk.x, acc[0][0]); acc[0][1] = fmaf(qq.x, kk.y, acc[0][1]);
      acc[1][0] = fmaf(qq.y, kk.x, acc[1][0]); acc[1][1] = fmaf(qq.y, kk.y, acc[1][1]);
      acc[2][0] = fmaf(qq.z, kk.x, acc[2][0]); acc[2][1] = fmaf(qq.z, kk.y, acc[2][1]);
      acc[3][0] = fmaf(qq.w, kk.x, acc[3][0]); acc[3][1] = fmaf(qq.w, kk.y, acc[3][1]);
    }
    const int j0 = kb + 2 * lane;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = j0 + u;
      if (j >= S) break;
      float sv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = min(i0 + r, S - 1);
        float x = bf16_round(acc[r][u]);
        if (use_scale) x = bf16_round(x * scale);
        if (bias) x = bf16_round(x + __bfloat162float(bias[(static_cast<size_t>(h) * S + i) * S + j]));
        if (causal && j > i) x = -INFINITY;
        sv[r] = x;
        mx[r] = fmaxf(mx[r], x);
      }
      my[j] = make_float4(sv[0], sv[1], sv[2], sv[3]);
    }
  }
  float sum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 4; ++r) mx[r] = warp_max_t(mx[r]);
  for (int kb = 0; kb < S; kb += 64)
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = kb + 2 * lane + u;
      if (j >= S) break;
      float4 e = my[j];
      e.x = expf(e.x - mx[0]); e.y = expf(e.y - mx[1]); e.z = expf(e.z - mx[2]); e.w = expf(e.w - mx[3]);
      sum[0] += e.x; sum[1] += e.y; sum[2] += e.z; sum[3] += e.w;
      my[j] = e;
    }
#pragma unroll
  for (int r = 0; r < 4; ++r) sum[r] = 1.0f / warp_sum_t(sum[r]);
  for (int kb = 0; kb < S; kb += 64)
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = kb + 2 * lane + u;
      if (j >= S) break;
      float4 e = my[j];
      my[j] = make_float4(bf16_round(e.x * sum[0]), bf16_round(e.y * sum[1]), bf16_round(e.z * sum[2]),
                          bf16_round(e.w * sum[3]));
    }
  __syncwarp();
  float o[4][2] = {};
#pragma unroll 4
  for (int j = 0; j < S; ++j) {
    const float4 p = my[j];
    const float2 vv = unpack_bf16x2(vs2[j * 32 + lane]);
    o[0][0] = fmaf(p.x, vv.x, o[0][0]); o[0][1] = fmaf(p.x, vv.y, o[0][1]);
    o[1][0] = fmaf(p.y, vv.x, o[1][0]); o[1][1] = fmaf(p.y, vv.y, o[1][1]);
    o[2][0] = fmaf(p.z, vv.x, o[2][0]); o[2][1] = fmaf(p.z, vv.y, o[2][1]);
    o[3][0] = fmaf(p.w, vv.x, o[3][0]); o[3][1] = fmaf(p.w, vv.y, o[3][1]);
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + r;
    if (i < S)
      *reinterpret_cast<uint32_t*>(out + (base + i) * ldo + h * 64 + 2 * lane) = pack_bf16x2(o[r][0], o[r][1]);
  }
}

// pooled[b, :] = hidden[b * S + pos[b], :]
__global__ void gather_rows_kernel(const bf16* __restrict__ x, const int* __restrict__ pos, bf16* __restrict__ out,
                                   int S, int D) {
  const int b = blockIdx.x;
  const bf16* src = x + (static_cast<size_t>(b) * S + pos[b]) * D;
  for (int i = threadIdx.x; i < D; i += blockDim.x) out[static_cast<size_t>(b) * D + i] = src[i];
}

}  // namespace rf

using rf::bf16;

namespace {
struct TSlot { bf16* dst; int64_t numel; bool loaded; };
struct T5Layer { bf16 *qkv, *o, *ln0, *wi0, *wi1, *wo, *ln1; };
struct ClipLayer { bf16 *ln1w, *ln1b, *qkvw, *qkvb, *ow, *ob, *ln2w, *ln2b, *fc1w, *fc1b, *fc2w, *fc2b; };
}  // namespace

struct rf_text {
  rf_text_config cfg;
  std::vector<void*> allocs;
  std::unordered_map<std::string, TSlot> slots;
  // T5
  bf16 *t5_shared = nullptr, *t5_final = nullptr;
  std::vector<T5Layer> t5;
  // CLIP
  bf16 *clip_tok = nullptr, *clip_pos = nullptr, *clip_fw = nullptr, *clip_fb = nullptr;
  std::vector<ClipLayer> clip;
  bf16* ones = nullptr;
  // workspace
  int ws_tokens = 0;
  bf16 *x = nullptr, *xn = nullptr, *qkv = nullptr, *att = nullptr, *h0 = nullptr, *h1 = nullptr;
  int* ids = nullptr;
};

namespace {
#define RF_TRYT(expr)           \
  do {                          \
    int _rc = (expr);           \
    if (_rc != 0) return _rc;   \
  } while (0)

int talloc(rf_text* h, void** p, size_t bytes) {
  RF_CHECK_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  h->allocs.push_back(*p);
  return 0;
}
bf16* take(rf_text* h, int64_t n, int& rc, const std::string& key = "") {
  void* p = nullptr;
  if (talloc(h, &p, static_cast<size_t>(n) * 2)) rc = -2;
  if (!key.empty()) h->slots[key] = {static_cast<bf16*>(p), n, false};
  return static_cast<bf16*>(p);
}
// a slice of a packed matrix registered under its own key
void alias(rf_text* h, const std::string& key, bf16* p, int64_t n) { h->slots[key] = {p, n, false}; }

int rownorm(const bf16* x, bf16* out, int rows, int dim, const bf16* w, const bf16* b, float eps, int mode,
            cudaStream_t s) {
  rf::rownorm_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, out, rows, dim, w, b, eps, mode);
  RF_CHECK_CUDA(cudaGetLastError());
  rf::count_launch();
  return 0;
}
int linear(int epi, const bf16* A, int lda, int M, const bf16* W, const bf16* bias, bf16* out, int ldo, int N,
           int K, const bf16* res, int ldr, const bf16* ones, cudaStream_t s) {
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = A; g.lda = lda; g.M = M; g.W = W; g.bias = bias; g.out = out; g.ldo = ldo;
  g.res = res; g.ldr = ldr; g.gate = ones;
  return rf::gemm_launch(epi, N, K, 1, &g, s);
}
int small_attn(const bf16* q, const bf16* k, const bf16* v, int ld, bf16* out, int ldo, int B, int S, int heads,
               const bf16* bias, float scale, int use_scale, int causal, cudaStream_t s) {
  // tensor-core path (text_attn_sm90.cu); RF_TEXT_ATTN=smem keeps the CUDA-core kernel below for A/B runs
  static const bool force_smem = getenv("RF_TEXT_ATTN") && std::string(getenv("RF_TEXT_ATTN")) == "smem";
  if (!force_smem && rf::text_attn_tc_eligible(S, ld, ldo))
    return rf::text_attn_tc_launch(q, k, v, ld, out, ldo, B, S, heads, bias, scale, use_scale, causal, s);
  const size_t smem = static_cast<size_t>(8) * S * 16 + 8 * 64 * 16 + static_cast<size_t>(S) * 32 * 4 +
                      static_cast<size_t>(64) * rf::small_attn_sp2(S) * 4;
  static bool attr = false;
  if (!attr) {
    RF_CHECK_CUDA(cudaFuncSetAttribute(rf::small_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       220 * 1024));
    attr = true;
  }
  if (smem > 220 * 1024) {
    rf::set_error("small_attn: sequence too long for the shared-memory kernel (S <= 512)");
    return -1;
  }
  dim3 grid((S + 31) / 32, heads, B);
  rf::ProfScope prof("text_attention", 4.0 * B * heads * S * S * 64, 0, s);
  rf::small_attn_kernel<<<grid, 256, smem, s>>>(q, k, v, ld, out, ldo, S, bias, scale, use_scale, causal);
  RF_CHECK_CUDA(cudaGetLastError());
  rf::count_launch();
  return 0;
}
int ensure_ws(rf_text* h, int tokens) {
  if (tokens <= h->ws_tokens) return 0;
  const rf_text_config& c = h->cfg;
  const int D = c.t5_d_model > c.clip_d_model ? c.t5_d_model : c.clip_d_model;
  const int F = c.t5_d_ff > 4 * c.clip_d_model ? c.t5_d_ff : 4 * c.clip_d_model;
  const int QKV = 3 * (c.t5_heads * 64 > c.clip_d_model ? c.t5_heads * 64 : c.clip_d_model);
  void* p;
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * D * 2)); h->x = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * D * 2)); h->xn = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * QKV * 2)); h->qkv = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * D * 2)); h->att = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * F * 2)); h->h0 = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * F * 2)); h->h1 = static_cast<bf16*>(p);
  RF_TRYT(talloc(h, &p, static_cast<size_t>(tokens) * 4)); h->ids = static_cast<int*>(p);
  h->ws_tokens = tokens;
  return 0;
}
int missing(rf_text* h, const char* prefix) {
  int n = 0;
  std::string names;
  const size_t pl = strlen(prefix);
  for (auto& kv : h->slots)
    if (kv.first.compare(0, pl, prefix) == 0 && !kv.second.loaded) {
      if (n < 6) names += kv.first + " ";
      ++n;
    }
  if (n) rf::set_error("missing text-encoder weights: " + names);
  return n;
}
}  // namespace

extern "C" {

int rf_text_create(const rf_text_config* cfg, rf_text** out) {
  if (!cfg || !out) {
    rf::set_error("rf_text_create: null argument");
    return -1;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    rf::set_error("rf_text_create: no CUDA device (this library has no CPU fallback)");
    return -3;
  }
  if (cfg->t5_d_model % 256 || cfg->t5_d_ff % 256 || cfg->clip_d_model % 256 || cfg->t5_d_model > 4096 ||
      cfg->clip_heads * 64 != cfg->clip_d_model) {
    rf::set_error("rf_text_create: unsupported config (widths must be multiples of 256, head_dim 64)");
    return -1;
  }
  rf_text* h = new rf_text();
  h->cfg = *cfg;
  int rc = 0;
  const int D = cfg->t5_d_model, F = cfg->t5_d_ff, I = cfg->t5_heads * 64;
  h->t5_shared = take(h, static_cast<int64_t>(cfg->t5_vocab) * D, rc, "t5.shared.weight");
  h->t5.resize(cfg->t5_layers);
  for (int i = 0; i < cfg->t5_layers; ++i) {
    T5Layer& L = h->t5[i];
    const std::string p = "t5.encoder.block." + std::to_string(i) + ".layer.";
    L.qkv = take(h, static_cast<int64_t>(3) * I * D, rc);
    alias(h, p + "0.SelfAttention.q.weight", L.qkv, static_cast<int64_t>(I) * D);
    alias(h, p + "0.SelfAttention.k.weight", L.qkv + static_cast<int64_t>(I) * D, static_cast<int64_t>(I) * D);
    alias(h, p + "0.SelfAttention.v.weight", L.qkv + static_cast<int64_t>(2) * I * D, static_cast<int64_t>(I) * D);
    L.o = take(h, static_cast<int64_t>(D) * I, rc, p + "0.SelfAttention.o.weight");
    L.ln0 = take(h, D, rc, p + "0.layer_norm.weight");
    L.wi0 = take(h, static_cast<int64_t>(F) * D, rc, p + "1.DenseReluDense.wi_0.weight");
    L.wi1 = take(h, static_cast<int64_t>(F) * D, rc, p + "1.DenseReluDense.wi_1.weight");
    L.wo = take(h, static_cast<int64_t>(D) * F, rc, p + "1.DenseReluDense.wo.weight");
    L.ln1 = take(h, D, rc, p + "1.layer_norm.weight");
  }
  h->t5_final = take(h, D, rc, "t5.encoder.final_layer_norm.weight");
  const int C = cfg->clip_d_model;
  h->clip_tok = take(h, static_cast<int64_t>(cfg->clip_vocab) * C, rc, "clip.text_model.embeddings.token_embedding.weight");
  h->clip_pos = take(h, static_cast<int64_t>(cfg->clip_max_pos) * C, rc, "clip.text_model.embeddings.position_embedding.weight");
  h->clip.resize(cfg->clip_layers);
  for (int i = 0; i < cfg->clip_layers; ++i) {
    ClipLayer& L = h->clip[i];
    const std::string p = "clip.text_model.encoder.layers." + std::to_string(i) + ".";
    L.ln1w = take(h, C, rc, p + "layer_norm1.weight");
    L.ln1b = take(h, C, rc, p + "layer_norm1.bias");
    L.qkvw = take(h, static_cast<int64_t>(3) * C * C, rc);
    L.qkvb = take(h, 3 * C, rc);
    const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      alias(h, p + "self_attn." + nm[j] + ".weight", L.qkvw + static_cast<int64_t>(j) * C * C, static_cast<int64_t>(C) * C);
      alias(h, p + "self_attn." + nm[j] + ".bias", L.qkvb + j * C, C);
    }
    L.ow = take(h, static_cast<int64_t>(C) * C, rc, p + "self_attn.out_proj.weight");
    L.ob = take(h, C, rc, p + "self_attn.out_proj.bias");
    L.ln2w = take(h, C, rc, p + "layer_norm2.weight");
    L.ln2b = take(h, C, rc, p + "layer_norm2.bias");
    L.fc1w = take(h, static_cast<int64_t>(4) * C * C, rc, p + "mlp.fc1.weight");
    L.fc1b = take(h, 4 * C, rc, p + "mlp.fc1.bias");
    L.fc2w = take(h, static_cast<int64_t>(4) * C * C, rc, p + "mlp.fc2.weight");
    L.fc2b = take(h, C, rc, p + "mlp.fc2.bias");
  }
  h->clip_fw = take(h, C, rc, "clip.text_model.final_layer_norm.weight");
  h->clip_fb = take(h, C, rc, "clip.text_model.final_layer_norm.bias");
  h->ones = take(h, 4096, rc);
  if (!rc) {
    std::vector<uint16_t> one(4096, 0x3F80);
    if (cudaMemcpy(h->ones, one.data(), 8192, cudaMemcpyHostToDevice) != cudaSuccess) rc = -2;
  }
  if (rc) {
    rf_text_destroy(h);
    return rc;
  }
  *out = h;
  return 0;
}

void rf_text_destroy(rf_text* h) {
  if (!h) return;
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

int rf_text_load_weight(rf_text* h, const char* key, const void* src, int64_t numel) {
  if (!h || !key || !src) {
    rf::set_error("rf_text_load_weight: null argument");
    return -1;
  }
  auto it = h->slots.find(key);
  if (it == h->slots.end()) {
    rf::set_error(std::string("rf_text_load_weight: unknown key ") + key);
    return -4;
  }
  if (it->second.numel != numel) {
    rf::set_error(std::string("rf_text_load_weight: size mismatch for ") + key + ": got " +
                  std::to_string(numel) + ", want " + std::to_string(it->second.numel));
    return -4;
  }
  RF_CHECK_CUDA(cudaMemcpy(it->second.dst, src, static_cast<size_t>(numel) * 2, cudaMemcpyDeviceToDevice));
  it->second.loaded = true;
  return 0;
}

int rf_text_missing_weights(rf_text* h, const char* prefix) { return h ? missing(h, prefix ? prefix : "") : -1; }

int rf_t5_encode(rf_text* h, const int* ids, int batch, int seq, const void* position_bias, void* out,
                 void* stream) {
  if (!h || !ids || !position_bias || !out || batch <= 0 || seq <= 0) {
    rf::set_error("rf_t5_encode: bad argument");
    return -1;
  }
  if (missing(h, "t5.") != 0) return -4;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const rf_text_config& c = h->cfg;
  const int D = c.t5_d_model, F = c.t5_d_ff, I = c.t5_heads * 64, T = batch * seq;
  RF_TRYT(ensure_ws(h, T));
  bf16* xo = static_cast<bf16*>(out);  // residual stream lives in the caller's output buffer
  rf::embed_kernel<<<T, 128, 0, s>>>(ids, h->t5_shared, nullptr, xo, T, seq, D);
  RF_CHECK_CUDA(cudaGetLastError());
  rf::count_launch();
  for (int i = 0; i < c.t5_layers; ++i) {
    const T5Layer& L = h->t5[i];
    RF_TRYT(rownorm(xo, h->xn, T, D, L.ln0, nullptr, c.t5_eps, 0, s));
    RF_TRYT(linear(rf::EPI_BIAS, h->xn, D, T, L.qkv, nullptr, h->qkv, 3 * I, 3 * I, D, nullptr, 0, nullptr, s));
    RF_TRYT(small_attn(h->qkv, h->qkv + I, h->qkv + 2 * I, 3 * I, h->att, I, batch, seq, c.t5_heads,
                       static_cast<const bf16*>(position_bias), 1.0f, 0, 0, s));
    RF_TRYT(linear(rf::EPI_GATE_RES, h->att, I, T, L.o, nullptr, xo, D, D, I, xo, D, h->ones, s));
    RF_TRYT(rownorm(xo, h->xn, T, D, L.ln1, nullptr, c.t5_eps, 0, s));
    RF_TRYT(linear(rf::EPI_GELU, h->xn, D, T, L.wi0, nullptr, h->h0, F, F, D, nullptr, 0, nullptr, s));
    RF_TRYT(linear(rf::EPI_BIAS, h->xn, D, T, L.wi1, nullptr, h->h1, F, F, D, nullptr, 0, nullptr, s));
    const long long n8 = static_cast<long long>(T) * F / 8;
    rf::ewise_kernel<<<static_cast<int>((n8 + 255) / 256), 256, 0, s>>>(h->h0, h->h1, h->h0, n8, 0);
    RF_CHECK_CUDA(cudaGetLastError());
    rf::count_launch();
    RF_TRYT(linear(rf::EPI_GATE_RES, h->h0, F, T, L.wo, nullptr, xo, D, D, F, xo, D, h->ones, s));
  }
  RF_TRYT(rownorm(xo, h->xn, T, D, h->t5_final, nullptr, c.t5_eps, 0, s));
  RF_CHECK_CUDA(cudaMemcpyAsync(xo, h->xn, static_cast<size_t>(T) * D * 2, cudaMemcpyDeviceToDevice, s));
  return 0;
}

int rf_clip_encode(rf_text* h, const int* ids, const int* eos_pos, int batch, int seq, void* pooled_out,
                   void* hidden_out, void* stream) {
  if (!h || !ids || !eos_pos || !pooled_out || batch <= 0 || seq <= 0 || seq > h->cfg.clip_max_pos) {
    rf::set_error("rf_clip_encode: bad argument");
    return -1;
  }
  if (missing(h, "clip.") != 0) return -4;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const rf_text_config& c = h->cfg;
  const int C = c.clip_d_model, T = batch * seq;
  RF_TRYT(ensure_ws(h, T));
  bf16* x = h->x;
  rf::embed_kernel<<<T, 128, 0, s>>>(ids, h->clip_tok, h->clip_pos, x, T, seq, C);
  RF_CHECK_CUDA(cudaGetLastError());
  rf::count_launch();
  for (int i = 0; i < c.clip_layers; ++i) {
    const ClipLayer& L = h->clip[i];
    RF_TRYT(rownorm(x, h->xn, T, C, L.ln1w, L.ln1b, 1e-5f, 1, s));
    RF_TRYT(linear(rf::EPI_BIAS, h->xn, C, T, L.qkvw, L.qkvb, h->qkv, 3 * C, 3 * C, C, nullptr, 0, nullptr, s));
    RF_TRYT(small_attn(h->qkv, h->qkv + C, h->qkv + 2 * C, 3 * C, h->att, C, batch, seq, c.clip_heads, nullptr,
                       0.125f, 1, 1, s));
    RF_TRYT(linear(rf::EPI_GATE_RES, h->att, C, T, L.ow, L.ob, x, C, C, C, x, C, h->ones, s));
    RF_TRYT(rownorm(x, h->xn, T, C, L.ln2w, L.ln2b, 1e-5f, 1, s));
    RF_TRYT(linear(rf::EPI_BIAS, h->xn, C, T, L.fc1w, L.fc1b, h->h0, 4 * C, 4 * C, C, nullptr, 0, nullptr, s));
    const long long n8 = static_cast<long long>(T) * 4 * C / 8;
    rf::ewise_kernel<<<static_cast<int>((n8 + 255) / 256), 256, 0, s>>>(h->h0, nullptr, h->h0, n8, 1);
    RF_CHECK_CUDA(cudaGetLastError());
    rf::count_launch();
    RF_TRYT(linear(rf::EPI_GATE_RES, h->h0, 4 * C, T, L.fc2w, L.fc2b, x, C, C, 4 * C, x, C, h->ones, s));
  }
  RF_TRYT(rownorm(x, h->xn, T, C, h->clip_fw, h->clip_fb, 1e-5f, 1, s));
  if (hidden_out)
    RF_CHECK_CUDA(cudaMemcpyAsync(hidden_out, h->xn, static_cast<size_t>(T) * C * 2, cudaMemcpyDeviceToDevice, s));
  rf::gather_rows_kernel<<<batch, 128, 0, s>>>(h->xn, eos_pos, static_cast<bf16*>(pooled_out), seq, C);
  RF_CHECK_CUDA(cudaGetLastError());
  rf::count_launch();
  return 0;
}

}  // extern "C"
