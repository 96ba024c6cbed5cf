// text_attn_sm90.cu — T5 / CLIP self-attention (head_dim 64, S <= 512) on the tensor cores (sm_90a).
//
//   scores = bf16(q k^T) [ = bf16(scores * scale) ] [ = bf16(scores + bias[h, i, j]) ] ; causal: j <= i
//   p      = bf16(softmax_fp32(scores)) ;  out = bf16(p v)
//
// the rounding points of transformers' eager attention in bf16 (T5Attention.forward: no scaling, additive
// relative-position bias; CLIPAttention: scaling, causal mask) — the text encoders diffusers' encode_prompt runs
// for every candidate prompt (train_flux/flux/generate.py:148-161).
//
// One CTA = one warpgroup = 64 query rows of one head; Q, every K and every V block of the head are loaded by
// TMA once.  The score rows are produced 128 keys at a time by wgmma (K = 64) and walked three times: round +
// bias + mask + max (the rounded bf16 scores are parked in shared memory, each thread reading back only what it
// wrote), exp + sum, and normalise -> bf16 P, which is the register A operand of O = P V (V read MN-major).
// Probabilities are normalised BEFORE the bf16 rounding and before P V, exactly like the eager reference (an
// online-softmax kernel would round un-normalised P).
#include <cuda.h>

#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

static constexpr int kTaThreads = 128;
static constexpr int kTaQBox = 64 * 64 * 2;    // [64 query rows x 64 cols] bf16 = 8 KB
static constexpr int kTaBox = 128 * 64 * 2;    // [128 key rows x 64 cols] bf16 = 16 KB
static constexpr int kTaMaxBlocks = 4;         // S <= 512
static constexpr int kTaPark = kTaThreads * kTaMaxBlocks * 32 * 4;  // packed bf16 scores, 64 KB
static constexpr int kTaSmem = kTaQBox + 2 * kTaMaxBlocks * kTaBox + kTaPark + 1024 + 64;

struct alignas(64) TextAttnParams {
  CUtensorMap tmQ, tmK, tmV;
  bf16* out;
  const bf16* bias;  // [heads, S, S] or nullptr
  int ldo, S, nb, use_scale, causal, bias_vec;
  float scale;
};

__global__ void __launch_bounds__(kTaThreads, 1) text_attn_kernel(const __grid_constant__ TextAttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kTaQBox;
  uint8_t* sV = sK + kTaMaxBlocks * kTaBox;
  uint32_t* park = reinterpret_cast<uint32_t*>(sV + kTaMaxBlocks * kTaBox);
  uint64_t* ld_bar = reinterpret_cast<uint64_t*>(park + kTaPark / 4);

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int wq = tid >> 5;
  const int cq = 2 * (lane & 3);
  const int q0 = blockIdx.x * 64;
  const int h = blockIdx.y;
  const int base = blockIdx.z * p.S;
  const int S = p.S, nb = p.nb;

  if (tid == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    mbar_init(ld_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(ld_bar, kTaQBox + 2 * nb * kTaBox);
    tma_load_2d(sQ, &p.tmQ, ld_bar, h * 64, base + q0);
    for (int b = 0; b < nb; ++b) {
      tma_load_2d(sK + b * kTaBox, &p.tmK, ld_bar, h * 64, base + b * 128);
      tma_load_2d(sV + b * kTaBox, &p.tmV, ld_bar, h * 64, base + b * 128);
    }
  }

  // this thread: query rows r0 + {0, 8} of the tile, keys 8 jj + cq + {0, 1} of every 128-key block
  const int r0 = q0 + wq * 16 + (lane >> 2);
  int row_c[2];
  const bf16* brow[2];
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = r0 + 8 * h2;
    row_c[h2] = row < S ? row : S - 1;
    brow[h2] = p.bias ? p.bias + (static_cast<size_t>(h) * S + row_c[h2]) * S : nullptr;
  }
  // parked pair i of key block c lives at park[(c * 32 + i) * 128 + tid]: pair i = 2 jj + h2
  auto park_at = [&](int c, int i) -> uint32_t& { return park[(c * 32 + i) * kTaThreads + tid]; };
  mbar_wait(ld_bar, 0);

  // ---- pass 1: the reference's score roundings, mask, running max
  float mx[2] = {-INFINITY, -INFINITY};
  const uint64_t qdesc = make_wgmma_desc(smem_u32(sQ), 16, 1024);
#pragma unroll 1
  for (int c = 0; c < nb; ++c) {
    float acc[64];
    const uint64_t kdesc = make_wgmma_desc(smem_u32(sK + c * kTaBox), 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n128(acc, qdesc + 2 * k, kdesc + 2 * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int j = c * 128 + 8 * jj + cq;
        float bv0 = 0.f, bv1 = 0.f;
        if (brow[h2] != nullptr) {
          if (p.bias_vec && j + 1 < S) {
            const float2 bb = unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(brow[h2] + j)));
            bv0 = bb.x;
            bv1 = bb.y;
          } else {
            if (j < S) bv0 = __bfloat162float(brow[h2][j]);
            if (j + 1 < S) bv1 = __bfloat162float(brow[h2][j + 1]);
          }
        }
        float x[2] = {acc[4 * jj + 2 * h2], acc[4 * jj + 2 * h2 + 1]};
        const float bv[2] = {bv0, bv1};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float y = bf16_round(x[e]);
          if (p.use_scale) y = bf16_round(y * p.scale);
          if (brow[h2] != nullptr) y = bf16_round(y + bv[e]);
          if (j + e >= S || (p.causal && j + e > row_c[h2])) y = -INFINITY;
          mx[h2] = fmaxf(mx[h2], y);
          x[e] = y;
        }
        park_at(c, 2 * jj + h2) = pack_bf16x2(x[0], x[1]);  // exact: the values are bf16 already
      }
    }
  }
  // ---- pass 2: row sums of e = exp(x - max)
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 1));
    mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 2));
  }
#pragma unroll 1
  for (int c = 0; c < nb; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float2 x = unpack_bf16x2(park_at(c, i));
      sum[i & 1] += expf(x.x - mx[i & 1]) + expf(x.y - mx[i & 1]);
    }
  float inv[2];
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    sum[h2] += __shfl_xor_sync(0xffffffffu, sum[h2], 1);
    sum[h2] += __shfl_xor_sync(0xffffffffu, sum[h2], 2);
    inv[h2] = 1.0f / sum[h2];
  }
  // ---- pass 3: p = bf16(e / sum) as the A fragments of O = P V, 128 keys (8 k-steps) at a time
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint32_t aV = smem_u32(sV);
#pragma unroll 1
  for (int c = 0; c < nb; ++c) {
    uint32_t pa[8][4];
#pragma unroll
    for (int kb = 0; kb < 8; ++kb)
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // a[q] = pair 4 kb + q (key blocks 2 kb, 2 kb + 1; rows +0 / +8)
        const float2 x = unpack_bf16x2(park_at(c, 4 * kb + q));
        pa[kb][q] = pack_bf16x2(expf(x.x - mx[q & 1]) * inv[q & 1], expf(x.y - mx[q & 1]) * inv[q & 1]);
      }
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 8; ++kb)  // 16 keys per step: V advances 16 rows x 128 B
      wgmma_rs_n64_tb(o, pa[kb], make_wgmma_desc(aV + c * kTaBox + kb * 2048, kTaBox, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
  }
  // ---- epilogue: O -> bf16 -> token-major output
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = r0 + 8 * h2;
    if (row < S) {
      bf16* dst = p.out + static_cast<size_t>(base + row) * p.ldo + h * 64 + cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h2], o[4 * jj + 2 * h2 + 1]);
    }
  }
}

bool text_attn_tc_eligible(int S, int ld, int ldo) {
  return S >= 1 && S <= 512 && (ld * 2) % 16 == 0 && (ldo * 2) % 16 == 0;
}

int text_attn_tc_launch(const bf16* q, const bf16* k, const bf16* v, int ld, bf16* out, int ldo, int B, int S,
                        int heads, const bf16* bias, float scale, int use_scale, int causal, cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    RF_CHECK_CUDA(cudaFuncSetAttribute(text_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTaSmem));
    attr = true;
  }
  TextAttnParams p;
  memset(&p, 0, sizeof(p));
  const uint64_t rows = static_cast<uint64_t>(B) * S, cols = static_cast<uint64_t>(heads) * 64;
  int rc = make_tmap_2d(&p.tmQ, q, rows, cols, ld, 64);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmK, k, rows, cols, ld, 128);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmV, v, rows, cols, ld, 128);
  if (rc) return rc;
  p.out = out;
  p.bias = bias;
  p.ldo = ldo;
  p.S = S;
  p.nb = (S + 127) / 128;
  p.use_scale = use_scale;
  p.causal = causal;
  p.scale = scale;
  p.bias_vec = (S % 8 == 0 && (reinterpret_cast<uintptr_t>(bias) & 15) == 0) ? 1 : 0;
  dim3 grid((S + 63) / 64, heads, B);
  ProfScope prof("text_attention", 4.0 * B * heads * static_cast<double>(S) * S * 64, 0, stream);
  RF_CHECK_CUDA(launch_pdl(text_attn_kernel, grid, dim3(kTaThreads), kTaSmem, stream, p));
  count_launch();
  return 0;
}

}  // namespace rf
