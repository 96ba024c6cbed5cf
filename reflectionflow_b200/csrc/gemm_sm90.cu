// gemm_sm90.cu — persistent, warp-specialised bf16 GEMM for sm_90a (H100).
//
//   out[M, N] = epilogue( A[M, K] @ W[N, K]^T )        (torch.nn.Linear weight layout)
//
// Replaces every nn.Linear call site on the reference's DiT hot path
// (train_flux/flux/block.py:27-29,46-48,81-83,148-154,252-259,296,320-328;
//  train_flux/flux/transformer.py:92-93,115,244) together with the element-wise work the
// reference runs after it (bias, GELU-tanh, gate*y + residual, per-head RMSNorm + RoPE), the LoRA
// down-projection and fused up-projection of the condition tokens, and the VAE convolutions
// (implicit GEMM over zero-ringed NHWC images).
//
// Structure (one CTA per SM, persistent over 128 x BN output tiles):
//   warpgroup 0      TMA producer : cp.async.bulk.tensor 128B-swizzled A/W k-blocks -> smem ring
//   warpgroups 1, 2  math         : wgmma m64nBNk16 on rows [0, 64) / [64, 128) of the tile, fp32
//                                   accumulators in registers, fused epilogue straight to HBM
// The producer runs ahead through the ring, so the next tile's operands load under the epilogue.
#include <cuda.h>

#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

static constexpr int BM = 128;
static constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
static constexpr int kGemmThreads = 384;
static constexpr int kMathWarps = 8;
static constexpr int kMaxGroups = 3;

struct alignas(64) GemmGroupDev {
  CUtensorMap tmA;
  CUtensorMap tmB;
  // fused peft LoRA (kLora kernels): T = bf16(x A^T) [M, 64 per section] and the B factor [N, 64];
  // a tile in column section s = n0 / lora_sec_cols reads T columns [64 s, 64 s + 64)
  CUtensorMap tmT, tmLB;
  const bf16* bias;
  bf16* out;
  const bf16* addend;
  const bf16* res;
  const bf16* gate;
  const float* rope_cos;
  const float* rope_sin;
  const bf16* norm_q;
  const bf16* norm_k;
  int M, ldo, ldadd, ldr;
  int m_tiles, tile_begin, lora_sec_cols;
  // implicit-GEMM convolution over zero-ringed NHWC images (conv_w > 0; tmA is a 3-D map {C, W+2, H+2},
  // out / res are [(H+2)(W+2), N]): an M tile is conv_by rows x conv_bx columns of OUTPUT pixels
  // (bx * by = 128); tap (ky, kx) of a k-block reads input pixels (s*y + ky + s-1, s*x + kx + s-1)
  int conv_w, conv_taps, conv_cin_blocks, conv_bx, conv_by, conv_stride;
};

struct alignas(64) GemmParamsDev {
  GemmGroupDev g[kMaxGroups];
  int ngroups, N, K, n_tiles, total_tiles, num_kb, band;
};

template <int BN>
struct GemmCfg {
  static constexpr int kStageBytesA = BM * BK * 2;
  static constexpr int kStageBytesB = BN * BK * 2;
  static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
  static constexpr int kStages = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);  // 192 KB of ring
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct TileCoord {
  int g, m0, n0;  // m0: first row (group-local), n0: first column
};
// Tiles run m-major inside bands of `band` n-tiles: a band's W slice stays L2-resident while every
// m tile of the group streams past it.
template <int BN>
__device__ __forceinline__ TileCoord decode_tile(const GemmParamsDev& p, int t) {
  int g = 0;
#pragma unroll
  for (int i = 1; i < kMaxGroups; ++i)
    if (i < p.ngroups && t >= p.g[i].tile_begin) g = i;
  const int local = t - p.g[g].tile_begin;
  const int mt = p.g[g].m_tiles, nt = p.n_tiles, band = p.band;
  const int full = nt / band;
  const int full_tiles = full * mt * band;
  int m, n;
  if (local < full_tiles) {
    const int per = mt * band;
    const int sc = local / per, r = local - sc * per;
    m = r / band;
    n = sc * band + (r - m * band);
  } else {
    const int rem = nt - full * band;
    const int r = local - full_tiles;
    m = r / rem;
    n = full * band + (r - m * rem);
  }
  return TileCoord{g, m * BM, n * BN};
}

struct PixTile { int x0, y0; };
__device__ __forceinline__ PixTile pix_tile(const GemmGroupDev& G, int m0) {
  const int mt = m0 >> 7;                // 128-pixel tile index
  const int xt = G.conv_w / G.conv_bx;   // tiles per image row
  const int ty = mt / xt;
  return PixTile{(mt - ty * xt) * G.conv_bx, ty * G.conv_by};
}

__device__ __forceinline__ float2 ld_bf16x2(const bf16* p) {
  return unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(p)));
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (BN == 256) wgmma_ss_n256(d, a, b, scale_d);
  else if constexpr (BN == 128) wgmma_ss_n128(d, a, b, scale_d);
  else wgmma_ss_n64(d, a, b, scale_d);
}

template <int BN, int EPI, bool kLora>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ GemmParamsDev p) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int g = 0; g < p.ngroups; ++g) {
      tma_prefetch_desc(&p.g[g].tmA);
      tma_prefetch_desc(&p.g[g].tmB);
      if constexpr (kLora) {
        tma_prefetch_desc(&p.g[g].tmT);
        tma_prefetch_desc(&p.g[g].tmLB);
      }
    }
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kMathWarps);  // one arrive per math warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // PDL: the prologue above overlapped the previous kernel's tail

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        const TileCoord tc = decode_tile<BN>(p, t);
        const GemmGroupDev& G = p.g[tc.g];
        PixTile pt{0, 0};
        if (G.conv_w != 0) pt = pix_tile(G, tc.m0);
        for (int kb = kLora ? -1 : 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kStageBytesA;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (kLora && kb < 0) {  // the low-rank k-block first: T rows, B factor rows of the tile
            const int tcol = G.lora_sec_cols > 0 ? (tc.n0 / G.lora_sec_cols) * 64 : 0;
            tma_load_2d(sa, &G.tmT, &full_bar[stage], tcol, tc.m0);
            tma_load_2d(sb, &G.tmLB, &full_bar[stage], 0, tc.n0);
          } else {
            if (G.conv_w != 0) {
              const int tap = kb / G.conv_cin_blocks;
              const int c0 = (kb - tap * G.conv_cin_blocks) * BK;
              const int ky = G.conv_taps == 9 ? tap / 3 : 1, kx = G.conv_taps == 9 ? tap % 3 : 1;
              const int sft = G.conv_stride - 1;
              tma_load_3d(sa, &G.tmA, &full_bar[stage], c0, G.conv_stride * pt.x0 + kx + sft,
                          G.conv_stride * pt.y0 + ky + sft);
            } else {
              tma_load_2d(sa, &G.tmA, &full_bar[stage], kb * BK, tc.m0);
            }
            tma_load_2d(sb, &G.tmB, &full_bar[stage], kb * BK, tc.n0);
          }
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== math warpgroups =====================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                 // rows [64 cw, 64 cw + 64) of the tile
  const int wq = (threadIdx.x >> 5) & 3;  // warp inside the warpgroup
  const int cq = 2 * (lane & 3);          // first of this thread's two columns in every 8-column block
  int stage = 0;
  uint32_t phase = 0;
  auto release = [&](int s) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  };
  auto a_desc = [&](int s) {
    return make_wgmma_desc(smem_u32(smem + s * Cfg::kStageBytes) + cw * 64 * 128, 16, 1024);
  };
  auto b_desc = [&](int s) {
    return make_wgmma_desc(smem_u32(smem + s * Cfg::kStageBytes + Cfg::kStageBytesA), 16, 1024);
  };

  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileCoord tc = decode_tile<BN>(p, t);
    const GemmGroupDev& G = p.g[tc.g];

    // bf16(L) of the low-rank term, packed pairs in accumulator order (kLora)
    uint32_t lpk[kLora ? BN / 4 : 1];
    if constexpr (kLora) {
      float accl[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) accl[i] = 0.f;
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) wgmma_tile<BN>(accl, a_desc(stage) + 2 * k, b_desc(stage) + 2 * k, k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(accl);
      release(stage);
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
#pragma unroll
      for (int i = 0; i < BN / 4; ++i) lpk[i] = pack_bf16x2(accl[2 * i], accl[2 * i + 1]);
    }

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        // +32 B per 16-element k-step inside the 128 B swizzle row (encoded >> 4)
        wgmma_tile<BN>(acc, a_desc(stage) + 2 * k, b_desc(stage) + 2 * k, (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have read their slot
      if (prev >= 0) release(prev);
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (prev >= 0) release(prev);

    // ===================== epilogue: registers -> fused math -> HBM =====================
    // this thread: rows r_loc + {0, 8} of the tile, columns 8 j + cq + {0, 1}
    const int r_loc = cw * 64 + wq * 16 + (lane >> 2);
    int orow[2];
    bool ok[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const int rl = r_loc + 8 * h2;
      if (G.conv_w != 0) {
        const PixTile pt = pix_tile(G, tc.m0);
        const int x = pt.x0 + rl % G.conv_bx, y = pt.y0 + rl / G.conv_bx;
        orow[h2] = (y + 1) * (G.conv_w + 2) + x + 1;
        ok[h2] = true;
      } else {
        orow[h2] = tc.m0 + rl;
        ok[h2] = orow[h2] < G.M;
      }
    }
    // v = bf16(acc + bias) [ = bf16(v + addend) ] [ = bf16(v + bf16(L)) ]: the rounding points of
    // nn.Linear (+ peft's unfused LoRA term) in bf16
    auto linear_round = [&](int j, int h2, float& v0, float& v1) {
      const int col = tc.n0 + 8 * j + cq;
      v0 = acc[4 * j + 2 * h2];
      v1 = acc[4 * j + 2 * h2 + 1];
      if (G.bias != nullptr) {
        const float2 b = ld_bf16x2(G.bias + col);
        v0 += b.x;
        v1 += b.y;
      }
      bf16_round2(v0, v1);
      if (G.addend != nullptr && ok[h2]) {
        const float2 a = ld_bf16x2(G.addend + static_cast<size_t>(orow[h2]) * G.ldadd + col);
        v0 += a.x;
        v1 += a.y;
        bf16_round2(v0, v1);
      }
      if constexpr (kLora) {
        const float2 l = unpack_bf16x2(lpk[2 * j + h2]);
        v0 += l.x;
        v1 += l.y;
        bf16_round2(v0, v1);
      }
    };
    auto store = [&](int j, int h2, float v0, float v1) {
      if (ok[h2])
        *reinterpret_cast<uint32_t*>(G.out + static_cast<size_t>(orow[h2]) * G.ldo + tc.n0 + 8 * j + cq) =
            pack_bf16x2(v0, v1);
    };

    if constexpr (EPI == EPI_QKV) {
      // Column space is [q | k | v] x heads x 128.  A head never straddles a tile (BN % 128 == 0);
      // a row of one head lives in the 4 lanes of a quad.
      const int inner = p.N / 3;
#pragma unroll
      for (int hc = 0; hc < BN / 128; ++hc) {
        const int col_h = tc.n0 + hc * 128;
        const int section = col_h / inner;  // 0 q, 1 k, 2 v
        float v[2][32];
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) linear_round(hc * 16 + jj, h2, v[h2][2 * jj], v[h2][2 * jj + 1]);
        if (section != 2) {
          const bf16* nw = (section == 0) ? G.norm_q : G.norm_k;
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) ss = __fmaf_rn(v[h2][i], v[h2][i], ss);
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            const float var = __fdiv_rn(ss, 128.0f);
            const float rinv = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, 1e-6f)));
            const int rr = ok[h2] ? orow[h2] : 0;
            const float* cosr = G.rope_cos + static_cast<size_t>(rr) * 64;
            const float* sinr = G.rope_sin + static_cast<size_t>(rr) * 64;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
              const int ch = 8 * jj + cq;  // column inside the head; (ch, ch + 1) is one RoPE pair
              const float2 w = ld_bf16x2(nw + ch);
              float y0 = __fmul_rn(v[h2][2 * jj], rinv), y1 = __fmul_rn(v[h2][2 * jj + 1], rinv);
              bf16_round2(y0, y1);  // RMSNorm -> bf16
              y0 = __fmul_rn(y0, w.x);
              y1 = __fmul_rn(y1, w.y);
              bf16_round2(y0, y1);  // * weight -> bf16
              // interleaved-pair RoPE, fp32, one rounding at the pack
              const float cs = __ldg(cosr + (ch >> 1)), sn = __ldg(sinr + (ch >> 1));
              v[h2][2 * jj] = __fadd_rn(__fmul_rn(y0, cs), __fmul_rn(-y1, sn));
              v[h2][2 * jj + 1] = __fadd_rn(__fmul_rn(y1, cs), __fmul_rn(y0, sn));
            }
          }
        }
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) store(hc * 16 + jj, h2, v[h2][2 * jj], v[h2][2 * jj + 1]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = tc.n0 + 8 * j + cq;
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          float v0, v1;
          linear_round(j, h2, v0, v1);
          if constexpr (EPI == EPI_GELU) {
            v0 = gelu_tanh(v0);
            v1 = gelu_tanh(v1);
          }
          if constexpr (EPI == EPI_GATE_RES) {
            if (ok[h2]) {
              const float2 gt = ld_bf16x2(G.gate + col);
              const float2 r = ld_bf16x2(G.res + static_cast<size_t>(orow[h2]) * G.ldr + col);
              float g0 = __fmul_rn(gt.x, v0), g1 = __fmul_rn(gt.y, v1);
              bf16_round2(g0, g1);
              v0 = __fadd_rn(r.x, g0);
              v1 = __fadd_rn(r.y, g1);
            }
          }
          store(j, h2, v0, v1);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------ host
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e =
      cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return -3;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0) {
    set_error("make_tmap_2d: base/pitch must be 16-byte aligned");
    return -1;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed, CUresult=" + std::to_string(static_cast<int>(r)));
    return -3;
  }
  return 0;
}

int make_tmap_3d(CUtensorMap* out, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp,
                 uint32_t box_x, uint32_t box_y, uint32_t stride) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return -3;
  }
  cuuint64_t gdim[3] = {C, Wp, Hp};
  cuuint64_t gstride[2] = {C * 2, Wp * C * 2};
  cuuint32_t box[3] = {64, box_x * stride, box_y * stride};
  cuuint32_t estr[3] = {1, stride, stride};
  if (box[1] > 256 || box[2] > 256) {
    set_error("make_tmap_3d: box dimension exceeds 256");
    return -1;
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstride,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(3d) failed, CUresult=" + std::to_string(static_cast<int>(r)));
    return -3;
  }
  return 0;
}

static int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

template <int BN, int EPI, bool LORA>
static int set_attr() {
  static bool attr_set = false;
  if (!attr_set) {
    RF_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<BN, EPI, LORA>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       GemmCfg<BN>::kSmemBytes));
    attr_set = true;
  }
  return 0;
}

int gemm_init() {
  int rc = 0;
  rc |= set_attr<256, EPI_BIAS, false>(); rc |= set_attr<256, EPI_GELU, false>();
  rc |= set_attr<256, EPI_GATE_RES, false>(); rc |= set_attr<256, EPI_QKV, false>();
  rc |= set_attr<128, EPI_BIAS, false>(); rc |= set_attr<128, EPI_GELU, false>();
  rc |= set_attr<128, EPI_GATE_RES, false>(); rc |= set_attr<128, EPI_QKV, false>();
  rc |= set_attr<64, EPI_BIAS, false>(); rc |= set_attr<64, EPI_GELU, false>();
  rc |= set_attr<64, EPI_GATE_RES, false>();
  rc |= set_attr<128, EPI_GELU, true>(); rc |= set_attr<128, EPI_GATE_RES, true>();
  rc |= set_attr<128, EPI_QKV, true>();
  return rc ? -2 : 0;
}

static thread_local int g_reserve_sms = 0;
int gemm_reserve_sms(int sms) {
  const int prev = g_reserve_sms;
  g_reserve_sms = sms < 0 ? 0 : sms;
  return prev;
}
// persistent grid: one CTA per SM, minus the reserved ones when the tiles still take the same number of
// waves; max_ctas > 0 caps it (the LoRA down-projection that runs beside another GEMM)
static int grid_ctas(int tiles, int max_ctas) {
  int ctas = num_sms();
  const int fewer = ctas - g_reserve_sms;
  if (g_reserve_sms > 0 && fewer > 0 && (tiles + fewer - 1) / fewer == (tiles + ctas - 1) / ctas) ctas = fewer;
  if (max_ctas > 0 && ctas > max_ctas) ctas = max_ctas;
  if (ctas > tiles) ctas = tiles;
  return ctas;
}

template <int BN, int EPI, bool LORA>
static int launch_cfg(GemmParamsDev& p, int max_ctas, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  if (int rc = set_attr<BN, EPI, LORA>()) return rc;
  const int grid = grid_ctas(p.total_tiles, max_ctas);
  double rows = 0;
  for (int g = 0; g < p.ngroups; ++g) rows += p.g[g].M;
  static const char* kNames[4] = {"gemm_bias", "gemm_gelu", "gemm_gate_res", "gemm_qkv_rms_rope"};
  const bool conv = p.g[0].conv_w != 0;
  const char* name = conv ? (EPI == EPI_GATE_RES ? "conv_res" : "conv_bias") : kNames[EPI];
  // algorithmic FLOPs: 2 M N K; algorithmic bytes: A (each pixel once for a convolution) + W + out once
  ProfScope prof(name, 2.0 * rows * p.N * p.K,
                 2.0 * (rows * p.K / (conv ? p.g[0].conv_taps : 1) +
                        static_cast<double>(p.ngroups) * p.N * p.K + rows * p.N),
                 stream);
  RF_CHECK_CUDA(launch_pdl(gemm_kernel<BN, EPI, LORA>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes,
                           stream, p));
  count_launch();
  return 0;
}

template <int BN>
static int launch_bn(int epi, GemmParamsDev& p, int max_ctas, cudaStream_t stream) {
  switch (epi) {
    case EPI_BIAS: return launch_cfg<BN, EPI_BIAS, false>(p, max_ctas, stream);
    case EPI_GELU: return launch_cfg<BN, EPI_GELU, false>(p, max_ctas, stream);
    case EPI_GATE_RES: return launch_cfg<BN, EPI_GATE_RES, false>(p, max_ctas, stream);
    case EPI_QKV:
      if constexpr (BN >= 128) return launch_cfg<BN, EPI_QKV, false>(p, max_ctas, stream);
      break;
    default: break;
  }
  set_error("gemm_launch: epilogue not available for this tile width");
  return -1;
}

// m-major raster inside bands of n tiles: up to 12 n tiles one band covers N, so every A row block is
// read once; wider outputs (QKV, MLP-in) use bands of 4 so the band's W slice stays in L2
static void set_raster(GemmParamsDev& p) { p.band = p.n_tiles <= 12 ? p.n_tiles : 4; }

static bool g_narrow_tiles = false;
void dbg_force_gemm_v1(bool on) { g_narrow_tiles = on; }

static int gemm_launch_impl(int epi, int N, int K, int ngroups, const GemmGroupArgs* groups, int max_ctas,
                            cudaStream_t stream) {
  if (ngroups < 1 || ngroups > kMaxGroups) {
    set_error("gemm_launch: ngroups must be 1..3");
    return -1;
  }
  if (K % BK != 0 || K <= 0) {
    set_error("gemm_launch: K must be a positive multiple of 64");
    return -1;
  }
  int bn = (N % 256 == 0) ? 256 : (N % 128 == 0 ? 128 : (N % 64 == 0 ? 64 : 0));
  if (bn == 0) {
    set_error("gemm_launch: N must be a multiple of 64");
    return -1;
  }
  if (epi == EPI_QKV && (bn < 128 || N % 384 != 0)) {
    set_error("gemm_launch: EPI_QKV needs N = 3 * heads * 128");
    return -1;
  }
  // 256-wide tiles halve the W traffic per FLOP; narrower ones when 256-wide tiles would leave SMs idle
  if (bn == 256) {
    int tiles256 = 0;
    for (int g = 0; g < ngroups; ++g) tiles256 += (groups[g].M + BM - 1) / BM * (N / 256);
    if (g_narrow_tiles || tiles256 < num_sms()) bn = 128;
  }
  GemmParamsDev p;
  memset(&p, 0, sizeof(p));
  p.ngroups = ngroups;
  p.N = N;
  p.K = K;
  p.n_tiles = N / bn;
  p.num_kb = K / BK;
  set_raster(p);
  int tiles = 0;
  for (int g = 0; g < ngroups; ++g) {
    const GemmGroupArgs& a = groups[g];
    GemmGroupDev& d = p.g[g];
    if (a.M <= 0) {
      set_error("gemm_launch: empty group");
      return -1;
    }
    if ((a.ldo & 1) || (reinterpret_cast<uintptr_t>(a.out) & 3)) {
      set_error("gemm_launch: output pitch / base must be 4-byte aligned");
      return -1;
    }
    int rc = make_tmap_2d(&d.tmA, a.A, a.M, K, a.lda, BM);
    if (rc) return rc;
    rc = make_tmap_2d(&d.tmB, a.W, N, K, K, bn);
    if (rc) return rc;
    d.bias = a.bias; d.out = a.out; d.addend = a.addend; d.res = a.res; d.gate = a.gate;
    d.rope_cos = a.rope_cos; d.rope_sin = a.rope_sin; d.norm_q = a.norm_q; d.norm_k = a.norm_k;
    d.M = a.M; d.ldo = a.ldo; d.ldadd = a.ldadd; d.ldr = a.ldr;
    d.m_tiles = (a.M + BM - 1) / BM;
    d.tile_begin = tiles;
    tiles += d.m_tiles * p.n_tiles;
    if (epi == EPI_GATE_RES && (a.res == nullptr || a.gate == nullptr)) {
      set_error("gemm_launch: EPI_GATE_RES needs res and gate");
      return -1;
    }
    if (epi == EPI_QKV && (!a.rope_cos || !a.rope_sin || !a.norm_q || !a.norm_k)) {
      set_error("gemm_launch: EPI_QKV needs rope tables and norm weights");
      return -1;
    }
  }
  p.total_tiles = tiles;
  switch (bn) {
    case 256: return launch_bn<256>(epi, p, max_ctas, stream);
    case 128: return launch_bn<128>(epi, p, max_ctas, stream);
    default: return launch_bn<64>(epi, p, max_ctas, stream);
  }
}

int gemm_launch(int epi, int N, int K, int ngroups, const GemmGroupArgs* groups, cudaStream_t stream) {
  return gemm_launch_impl(epi, N, K, ngroups, groups, 0, stream);
}

// ---- LoRA down-projection: T[M, NT] = bf16(X[M, K] @ A[NT, K]^T), an EPI_BIAS GEMM without bias
static GemmGroupArgs lora_down_args(const bf16* X, int ldx, int M, const bf16* A, bf16* T, int ldT) {
  GemmGroupArgs g;
  memset(&g, 0, sizeof(g));
  g.A = X; g.lda = ldx; g.M = M; g.W = A; g.out = T; g.ldo = ldT;
  return g;
}
int lora_down_launch(const bf16* X, int ldx, int M, int K, const bf16* A, int NT, bf16* T, int ldT,
                     cudaStream_t stream) {
  const GemmGroupArgs g = lora_down_args(X, ldx, M, A, T, ldT);
  return gemm_launch_impl(EPI_BIAS, NT, K, 1, &g, 0, stream);
}
int lora_down_side_launch(const bf16* X, int ldx, int M, int K, const bf16* A, int NT, bf16* T, int ldT,
                          cudaStream_t stream) {
  const GemmGroupArgs g = lora_down_args(X, ldx, M, A, T, ldT);
  return gemm_launch_impl(EPI_BIAS, NT, K, 1, &g, kLoraSideCtas, stream);
}

// ---- one token stream with peft LoRA fused: out = epi(bf16(bf16(A W^T + b) + bf16(T B^T)))
bool gemm2_lora_eligible(int epi, int N, int K, const GemmGroupArgs& a) {
  if (epi != EPI_GELU && epi != EPI_GATE_RES && epi != EPI_QKV) return false;
  if (N % 128 != 0 || K % BK != 0 || a.M < 128 || a.addend != nullptr) return false;
  if (epi == EPI_QKV && N % 384 != 0) return false;
  if ((a.ldo * 2) % 16 != 0 || (reinterpret_cast<uintptr_t>(a.out) & 15)) return false;
  if (epi == EPI_GATE_RES && ((a.ldr * 2) % 16 != 0 || (reinterpret_cast<uintptr_t>(a.res) & 15))) return false;
  return true;
}
int gemm2_lora_launch(int epi, int N, int K, const GemmGroupArgs& a, const bf16* T, int ldT,
                      const bf16* loraB, int sec_cols, cudaStream_t stream) {
  constexpr int bn = 128;  // two fp32 accumulators (base + low-rank) per thread
  GemmParamsDev p;
  memset(&p, 0, sizeof(p));
  p.ngroups = 1;
  p.N = N;
  p.K = K;
  p.n_tiles = N / bn;
  p.num_kb = K / BK;
  set_raster(p);
  GemmGroupDev& d = p.g[0];
  int rc = make_tmap_2d(&d.tmA, a.A, a.M, K, a.lda, BM);
  if (rc) return rc;
  rc = make_tmap_2d(&d.tmB, a.W, N, K, K, bn);
  if (rc) return rc;
  const int t_cols = sec_cols > 0 ? (N / sec_cols) * 64 : 64;
  rc = make_tmap_2d(&d.tmT, T, a.M, t_cols, ldT, BM);
  if (rc) return rc;
  rc = make_tmap_2d(&d.tmLB, loraB, N, 64, 64, bn);
  if (rc) return rc;
  if (epi == EPI_GATE_RES && (a.res == nullptr || a.gate == nullptr)) {
    set_error("gemm2_lora_launch: EPI_GATE_RES needs res and gate");
    return -1;
  }
  if (epi == EPI_QKV && (!a.rope_cos || !a.rope_sin || !a.norm_q || !a.norm_k)) {
    set_error("gemm2_lora_launch: EPI_QKV needs rope tables and norm weights");
    return -1;
  }
  d.bias = a.bias; d.out = a.out; d.addend = nullptr; d.res = a.res; d.gate = a.gate;
  d.rope_cos = a.rope_cos; d.rope_sin = a.rope_sin; d.norm_q = a.norm_q; d.norm_k = a.norm_k;
  d.M = a.M; d.ldo = a.ldo; d.ldadd = 0; d.ldr = a.ldr;
  d.lora_sec_cols = sec_cols;
  d.m_tiles = (a.M + BM - 1) / BM;
  d.tile_begin = 0;
  p.total_tiles = d.m_tiles * p.n_tiles;
  switch (epi) {
    case EPI_GELU: return launch_cfg<bn, EPI_GELU, true>(p, 0, stream);
    case EPI_GATE_RES: return launch_cfg<bn, EPI_GATE_RES, true>(p, 0, stream);
    case EPI_QKV: return launch_cfg<bn, EPI_QKV, true>(p, 0, stream);
    default: break;
  }
  set_error("gemm2_lora_launch: unsupported epilogue");
  return -1;
}

// 3x3 (taps = 9) or 1x1 (taps = 1) convolution, stride 1 (zero padding 1) or stride 2 (diffusers
// Downsample2D: pad right/bottom by one, no other padding), NHWC bf16 images with a one-pixel zero
// ring: in [(Hin+2)(Win+2), Cin], out [(H+2)(W+2), Cout] (interior written, ring untouched), weights
// [Cout, taps * Cin] (tap-major K), optional residual res (same geometry as out) added after the bias
// rounding (ResnetBlock2D: x + conv2(...)).  H, W are the OUTPUT size; Hin = stride * H.
// Needs: Cin % 64 == 0, Cout % 128 == 0, W a power of two >= 8 (or a multiple of 128), H % (128/bx) == 0.
int conv_launch(const bf16* in, const bf16* weight, const bf16* bias, bf16* out, const bf16* res,
                const bf16* ones, int H, int W, int Cin, int Cout, int taps, int stride,
                cudaStream_t stream) {
  const int bx = W >= 128 ? 128 : W;
  const int by = 128 / bx;
  if (Cin % 64 != 0 || Cout % 128 != 0 || (taps != 9 && taps != 1) || (stride != 1 && stride != 2) ||
      W % bx != 0 || 128 % bx != 0 || H % by != 0) {
    set_error("conv_launch: unsupported geometry (Cin % 64, Cout % 128, W = 2^k or multiple of 128, "
              "H divisible by 128 / min(W, 128))");
    return -1;
  }
  const int bn = (Cout % 256 == 0) ? 256 : 128;
  GemmParamsDev p;
  memset(&p, 0, sizeof(p));
  p.ngroups = 1;
  p.N = Cout;
  p.K = taps * Cin;
  p.n_tiles = Cout / bn;
  p.num_kb = p.K / BK;
  p.band = p.n_tiles;
  GemmGroupDev& d = p.g[0];
  const int Hin = stride * H, Win = stride * W;
  int rc = make_tmap_3d(&d.tmA, in, Cin, Win + 2, Hin + 2, bx, by, stride);
  if (rc) return rc;
  rc = make_tmap_2d(&d.tmB, weight, Cout, p.K, p.K, bn);
  if (rc) return rc;
  d.bias = bias;
  d.out = out;
  d.ldo = Cout;
  d.res = res;
  d.ldr = Cout;
  d.gate = ones;  // residual epilogue = bf16(res + bf16(1 * y))
  d.M = H * W;
  d.m_tiles = d.M / BM;
  d.conv_w = W;
  d.conv_taps = taps;
  d.conv_cin_blocks = Cin / BK;
  d.conv_bx = bx;
  d.conv_by = by;
  d.conv_stride = stride;
  p.total_tiles = d.m_tiles * p.n_tiles;
  const int epi = res ? EPI_GATE_RES : EPI_BIAS;
  return bn == 256 ? launch_bn<256>(epi, p, 0, stream) : launch_bn<128>(epi, p, 0, stream);
}

}  // namespace rf
