// attn_sm90.cu — non-causal joint attention for sm_90a (H100), head_dim 128.
//
//   O = softmax(Q K^T / sqrt(128)) V        over the joint [txt | img | cond] token sequence
//
// Replaces F.scaled_dot_product_attention at train_flux/flux/block.py:123-125 and the
// torch.cat / transpose traffic around it (block.py:31-33,70-72,102-104,126-128): Q, K, V are
// read by TMA straight out of the token-major [n_tok, heads*128] buffers the QKV GEMM epilogue
// wrote, and O is written token-major so it is the A operand of the out-projection GEMM.
//
// One CTA = one 128-row query tile of one head:
//   warpgroup 0      TMA producer: Q once, then K_j / V_j through a 2-stage ring
//   warpgroups 1, 2  query rows [0, 64) / [64, 128): S = Q K^T by wgmma (both operands from shared
//                    memory), online softmax in registers (log2 domain), P packed to bf16 in registers
//                    and O += P V by wgmma with P as the register A operand (V read MN-major)
// A masked (q tile, kv tile) pair of cond_mode 2 is skipped: its P would be 0.  When n_main % 128 != 0 the query
// tile and the kv tile that hold the split take the cond_mode 2 mask / cond_mode 1 bias per element instead.
#include <cuda.h>

#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

static constexpr int kAttnThreads = 384;
static constexpr int kTile = 128;
static constexpr int kHalfBytes = kTile * 128;     // one [128 x 64] bf16 box = 16 KB
static constexpr int kTileBytes = 2 * kHalfBytes;  // [128 x 128] bf16 = 32 KB
static constexpr int kKVStages = 2;
static constexpr int kAttnSmem = (1 + 2 * kKVStages) * kTileBytes + 1024 + 256;

struct alignas(64) AttnParamsDev {
  CUtensorMap tmQ, tmK, tmV;
  bf16* out;
  int ldo, n_tok, heads, batch, q_tiles, kv_tiles;
  int n_main, cond_mode;
  float scale_log2;  // log2(e) / sqrt(128)
  float bias_log2;   // log2(e) * cond_bias
  float bias_raw;    // cond_bias * sqrt(128): the same bias added to a raw score (split tiles)
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_kernel(const __grid_constant__ AttnParamsDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kTileBytes;            // kKVStages tiles
  uint8_t* sV = sK + kKVStages * kTileBytes;  // kKVStages tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kKVStages * kTileBytes);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;    // [2]
  uint64_t* v_full = bars + 3;    // [2]
  uint64_t* kv_empty = bars + 5;  // [2]

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  // q tile fastest so that all CTAs of one head run together (its K/V stay in L2)
  int bid = blockIdx.x;
  const int qt = bid % p.q_tiles;
  bid /= p.q_tiles;
  const int head = bid % p.heads;
  const int b = bid / p.heads;
  const int row_base = b * p.n_tok;
  const int q0 = qt * kTile;
  const int col0 = head * 128;
  const int n_kv = p.kv_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < kKVStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);  // one arrive per math warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, kTileBytes);
      tma_load_2d(sQ, &p.tmQ, q_full, col0, row_base + q0);
      tma_load_2d(sQ + kHalfBytes, &p.tmQ, q_full, col0 + 64, row_base + q0);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j & 1;
        mbar_wait(&kv_empty[st], ((j >> 1) & 1) ^ 1);
        uint8_t* kd = sK + st * kTileBytes;
        uint8_t* vd = sV + st * kTileBytes;
        mbar_arrive_expect_tx(&k_full[st], kTileBytes);
        tma_load_2d(kd, &p.tmK, &k_full[st], col0, row_base + j * kTile);
        tma_load_2d(kd + kHalfBytes, &p.tmK, &k_full[st], col0 + 64, row_base + j * kTile);
        mbar_arrive_expect_tx(&v_full[st], kTileBytes);
        tma_load_2d(vd, &p.tmV, &v_full[st], col0, row_base + j * kTile);
        tma_load_2d(vd + kHalfBytes, &p.tmV, &v_full[st], col0 + 64, row_base + j * kTile);
      }
    }
    return;
  }

  // ===================== softmax / MMA warpgroups =====================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3;
  const int cq = 2 * (lane & 3);
  const bool q_is_cond = (p.cond_mode != 0) && (q0 >= p.n_main);
  // the query tile holding the split row n_main (n_main % 128 != 0): rows on both sides of it
  const bool q_straddle = (p.cond_mode != 0) && q0 < p.n_main && p.n_main < q0 + kTile;
  const int row0 = q0 + cw * 64 + wq * 16 + (lane >> 2);  // this thread's query rows: row0, row0 + 8
  const uint32_t aQ = smem_u32(sQ) + cw * 64 * 128, aK = smem_u32(sK), aV = smem_u32(sV);

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running row max, log2-scaled units
  float l_run[2] = {0.f, 0.f};              // this thread's share of the row sums
  auto release = [&](int st) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  };
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    const bool cross = (p.cond_mode != 0) && ((j * kTile >= p.n_main) != q_is_cond);
    // a pair with the split inside its query or its key range takes the mask / bias per element
    const bool split = q_straddle || ((p.cond_mode != 0) && j * kTile < p.n_main && p.n_main < (j + 1) * kTile);
    mbar_wait(&k_full[st], ph);
    if (p.cond_mode == 2 && cross && !split) {  // fully masked tile: P = 0, statistics untouched
      mbar_wait(&v_full[st], ph);
      release(st);
      continue;
    }
    const float bias = (p.cond_mode == 1 && cross && !split) ? p.bias_log2 : 0.f;
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t off = (kk >> 2) * kHalfBytes + (kk & 3) * 32;
      wgmma_ss_n128(s, make_wgmma_desc(aQ + off, 16, 1024),
                    make_wgmma_desc(aK + st * kTileBytes + off, 16, 1024), kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);

    // keys past n_tok (last, partial tile): TMA zero-filled them; mask their scores
    const int kv_valid = p.n_tok - j * kTile;
    if (kv_valid < kTile) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * jj + cq + e >= kv_valid) {
            s[4 * jj + e] = -INFINITY;
            s[4 * jj + 2 + e] = -INFINITY;
          }
    }
    if (split) {
      // per element: -inf where cond_mode 2 masks the pair, + cond_bias (in units of the raw score) where
      // cond_mode 1 biases it; the statistics below then run with no tile bias
      const int kc = p.n_main - j * kTile - cq;  // key column 8 jj + e is a condition key iff 8 jj + e >= kc
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const bool rc = row0 + 8 * h2 >= p.n_main;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if ((8 * jj + e >= kc) != rc) {
              float& v = s[4 * jj + 2 * h2 + e];
              v = p.cond_mode == 2 ? -INFINITY : v + p.bias_raw;
            }
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2)
        mx[h2] = fmaxf(mx[h2], fmaxf(s[4 * jj + 2 * h2], s[4 * jj + 2 * h2 + 1]));
    float neg_m[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 1));
      mx[h2] = fmaxf(mx[h2], __shfl_xor_sync(0xffffffffu, mx[h2], 2));
      const float m_new = fmaxf(m_run[h2], fmaf(mx[h2], p.scale_log2, bias));
      // split pairs only: a row whose keys so far are all masked keeps max -inf but exponentiates against 0
      // (-inf - -inf would be NaN); its P, O and row sum stay 0
      const float m_use = (split && m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = ex2_approx(m_run[h2] - m_use);  // 0 on the first tile
      m_run[h2] = m_new;
      l_run[h2] *= alpha;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        o[4 * jj + 2 * h2] *= alpha;
        o[4 * jj + 2 * h2 + 1] *= alpha;
      }
      neg_m[h2] = bias - m_use;
    }
    // P = exp2(s * scale + bias - m), packed into the A fragments of the 8 k-steps of P V
    uint32_t pa[8][4];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const float e0 = ex2_approx(fmaf(s[4 * jj + 2 * h2], p.scale_log2, neg_m[h2]));
        const float e1 = ex2_approx(fmaf(s[4 * jj + 2 * h2 + 1], p.scale_log2, neg_m[h2]));
        l_run[h2] += e0 + e1;
        pa[jj >> 1][(jj & 1) * 2 + h2] = pack_bf16x2(e0, e1);
      }

    mbar_wait(&v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      // 16 kv rows per k-step (16 x 128 B); the two 64-column halves of V are 16 KB apart
      wgmma_rs_n128_tb(o, pa[kk], make_wgmma_desc(aV + st * kTileBytes + kk * 2048, kHalfBytes, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    release(st);
  }

  // ---- epilogue: O / l -> bf16 -> HBM (token-major)
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    float l = l_run[h2];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = l > 0.f ? __fdiv_rn(1.0f, l) : 0.f;
    const int row = q0 + cw * 64 + wq * 16 + (lane >> 2) + 8 * h2;
    if (row < p.n_tok) {
      bf16* orow = p.out + static_cast<size_t>(row_base + row) * p.ldo + col0 + cq;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj) =
            pack_bf16x2(o[4 * jj + 2 * h2] * inv_l, o[4 * jj + 2 * h2 + 1] * inv_l);
    }
  }
}

int attention_init() {
  static bool attr_set = false;
  if (!attr_set) {
    RF_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kAttnSmem));
    attr_set = true;
  }
  return 0;
}

int attention_launch(const AttnArgs& a, cudaStream_t stream) {
  if (a.n_tok <= 0 || a.heads <= 0 || a.batch <= 0) {
    set_error("attention_launch: empty problem");
    return -1;
  }
  if (a.cond_mode != 0 && (a.n_main <= 0 || a.n_main >= a.n_tok)) {
    set_error("attention_launch: cond split must lie inside (0, n_tok)");
    return -1;
  }
  if (a.batch > 1 && a.n_tok % kTile != 0) {
    set_error("attention_launch: batched call needs n_tok % 128 == 0");
    return -1;
  }
  if ((a.ldo & 1) || (reinterpret_cast<uintptr_t>(a.out) & 3)) {
    set_error("attention_launch: output pitch / base must be 4-byte aligned");
    return -1;
  }
  // cond_bias = -inf (condition_scale 0: the reference's bias log 0) gives the cross pairs a weight of exactly 0, the
  // cond_mode 2 mask.  Run it as cond_mode 2: a whole cross tile under a -inf tile bias would take -inf - -inf = NaN.
  const int cond_mode = (a.cond_mode == 1 && a.cond_bias == -INFINITY) ? 2 : a.cond_mode;
  AttnParamsDev p;
  memset(&p, 0, sizeof(p));
  const uint64_t rows = static_cast<uint64_t>(a.n_tok) * a.batch;
  const uint64_t cols = static_cast<uint64_t>(a.heads) * 128;
  int rc = make_tmap_2d(&p.tmQ, a.q, rows, cols, a.ld_qkv, kTile);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmK, a.k, rows, cols, a.ld_qkv, kTile);
  if (rc) return rc;
  rc = make_tmap_2d(&p.tmV, a.v, rows, cols, a.ld_qkv, kTile);
  if (rc) return rc;
  p.out = a.out;
  p.ldo = a.ldo;
  p.n_tok = a.n_tok;
  p.heads = a.heads;
  p.batch = a.batch;
  p.q_tiles = (a.n_tok + kTile - 1) / kTile;
  p.kv_tiles = (a.n_tok + kTile - 1) / kTile;
  p.n_main = cond_mode ? a.n_main : a.n_tok;
  p.cond_mode = cond_mode;
  const float kLog2e = 1.4426950408889634f;
  p.scale_log2 = kLog2e * 0.08838834764831845f;  // 1/sqrt(128)
  p.bias_log2 = kLog2e * a.cond_bias;
  p.bias_raw = a.cond_bias * 11.313708498984761f;  // sqrt(128)
  if (int rc = attention_init()) return rc;
  const int grid = p.q_tiles * a.heads * a.batch;
  // algorithmic FLOPs: QK^T and PV only (4 * n^2 * 128 per head); bytes: q,k,v read + o written
  const double n = a.n_tok;
  ProfScope prof("attention", 4.0 * n * n * 128.0 * a.heads * a.batch,
                 2.0 * 4.0 * n * 128.0 * a.heads * a.batch, stream);
  RF_CHECK_CUDA(launch_pdl(attn_kernel, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, p));
  count_launch();
  return 0;
}

}  // namespace rf
