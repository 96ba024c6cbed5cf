// elementwise.cu — the HBM-bound kernels of the DiT step (sm_90a).
//
//   ln_modulate   : LayerNorm(no affine, eps 1e-6) + adaLN scale/shift in one pass over the
//                   hidden state; writes the bf16 A operand of the next GEMM.
//                   (diffusers AdaLayerNormZero / ZeroSingle / Continuous bodies; reference call
//                   sites train_flux/flux/block.py:186,191,201,232-247,295,299 and
//                   transformer.py:243)
//   gemv          : every adaLN modulation Linear of all 57 blocks in ONE launch per step
//                   (M = batch <= 8 rows against ~1.06 M weight rows; pure weight streaming),
//                   also the small time/guidance/text embedder MLPs (transformer.py:102-114)
//   timestep_embed: sinusoidal projection (diffusers Timesteps(256, flip_sin_to_cos=True))
//   euler_step    : FlowMatchEulerDiscreteScheduler.step (generate.py:276)
// All of them keep the reference's bf16 rounding points (SURVEY.md Appendix A).
#include <cstring>

#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------- ln_modulate
// one warp per row; dim <= 3072 and dim % 256 == 0 (each lane owns dim/256 16-byte chunks)
static constexpr int kLnMaxChunks = 12;

struct LnGroups {  // up to 3 row ranges (token streams) of one joint buffer, each with its own adaLN vectors
  int row_end[3];
  const bf16* scale[3];
  const bf16* shift[3];
  int ngroups;
};

__global__ void __launch_bounds__(256, 3)
ln_modulate_kernel(const bf16* __restrict__ x, int ldx, bf16* __restrict__ out, int ldo, int rows,
                   int dim, const __grid_constant__ LnGroups G, int rows_per_batch, int mod_stride) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const int nch = dim >> 8;  // 16-byte chunks per lane
  for (int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps_total) {
  const int b = row / rows_per_batch;
  int gi = 0;
  if (G.ngroups > 1 && row >= G.row_end[0]) gi = 1;
  if (G.ngroups > 2 && row >= G.row_end[1]) gi = 2;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * ldx);
  const uint4* sc = reinterpret_cast<const uint4*>(G.scale[gi] + static_cast<size_t>(b) * mod_stride);
  const uint4* sh = reinterpret_cast<const uint4*>(G.shift[gi] + static_cast<size_t>(b) * mod_stride);
  // the row stays in registers as packed bf16 (48 regs) so that 32 warps/SM are resident
  uint4 raw[kLnMaxChunks];
#pragma unroll
  for (int i = 0; i < kLnMaxChunks; ++i)
    if (i < nch) raw[i] = __ldg(xr + lane + 32 * i);
  // element pairs (IEEE round-to-nearest like the scalar forms), unpacked from bf16x2 once
  float2 s2 = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < kLnMaxChunks; ++i) {
    if (i < nch) {
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) s2 = fadd2(s2, unpack_bf16x2(w[q]));
    }
  }
  const float mean = warp_sum(s2.x + s2.y) / static_cast<float>(dim);
  const float2 nmean = make_float2(-mean, -mean);
  float2 q2 = make_float2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < kLnMaxChunks; ++i) {
    if (i < nch) {
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 d = fadd2(unpack_bf16x2(w[q]), nmean);
        q2 = ffma2(d, d, q2);
      }
    }
  }
  const float var = warp_sum(q2.x + q2.y) / static_cast<float>(dim);
  const float rstd = __fdiv_rn(1.0f, __fsqrt_rn(var + 1e-6f));
  const float2 rstd2 = make_float2(rstd, rstd);
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * ldo);
#pragma unroll
  for (int i = 0; i < kLnMaxChunks; ++i) {
    if (i < nch) {
      const uint4 us = __ldg(sc + lane + 32 * i), uh = __ldg(sh + lane + 32 * i);
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
      const uint32_t su[4] = {us.x, us.y, us.z, us.w};
      const uint32_t hu[4] = {uh.x, uh.y, uh.z, uh.w};
      uint32_t ou[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float2 y = fmul2(fadd2(unpack_bf16x2(w[q]), nmean), rstd2);   // LayerNorm
        bf16_round2(y.x, y.y);                                                      //   -> bf16
        float2 t = fadd2(unpack_bf16x2(su[q]), make_float2(1.0f, 1.0f));      // (1 + scale)
        bf16_round2(t.x, t.y);                                                      //   -> bf16
        y = fmul2(y, t);
        bf16_round2(y.x, y.y);                                                      //   -> bf16
        const float2 o = fadd2(y, unpack_bf16x2(hu[q]));                      // + shift -> bf16 at the pack
        ou[q] = pack_bf16x2(o.x, o.y);
      }
      orow[lane + 32 * i] = make_uint4(ou[0], ou[1], ou[2], ou[3]);
    }
  }
  }  // row loop
}

static int ln_launch_common(const bf16* x, int ldx, bf16* out, int ldo, int rows, int dim, const LnGroups& G,
                            int rows_per_batch, int mod_stride, cudaStream_t stream) {
  if (dim % 256 != 0 || dim > 256 * kLnMaxChunks || dim <= 0) {
    set_error("ln_modulate: dim must be a multiple of 256, <= 3072");
    return -1;
  }
  if (rows <= 0) return 0;
  // one warp per row, rows dealt round-robin to a grid that is at most one resident wave
  // (3 blocks x 8 warps per SM): no block-granular tail
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  int blocks = (rows + 7) / 8;
  if (blocks > sms * 3) blocks = sms * 3;
  ProfScope prof("ln_modulate", 0.0, 4.0 * rows * dim, stream);
  RF_CHECK_CUDA(launch_pdl(ln_modulate_kernel, dim3(blocks), dim3(256), 0, stream, x, ldx, out, ldo, rows, dim, G,
                           rows_per_batch > 0 ? rows_per_batch : rows, mod_stride));
  count_launch();
  return 0;
}

// grouped form: rows [0, row_end[0]) use (scale[0], shift[0]), [row_end[0], row_end[1]) the next ...
int ln_modulate_grouped_launch(const bf16* x, int ldx, bf16* out, int ldo, int dim, int ngroups,
                               const int* row_end, const bf16* const* scale, const bf16* const* shift,
                               cudaStream_t stream) {
  if (ngroups < 1 || ngroups > 3) {
    set_error("ln_modulate: 1..3 row groups");
    return -1;
  }
  LnGroups G;
  memset(&G, 0, sizeof(G));
  G.ngroups = ngroups;
  for (int i = 0; i < ngroups; ++i) {
    G.row_end[i] = row_end[i];
    G.scale[i] = scale[i];
    G.shift[i] = shift[i];
  }
  return ln_launch_common(x, ldx, out, ldo, row_end[ngroups - 1], dim, G, 0, 0, stream);
}

int ln_modulate_launch(const bf16* x, int ldx, bf16* out, int ldo, int rows, int dim,
                       const bf16* scale, const bf16* shift, int rows_per_batch, int mod_stride,
                       cudaStream_t stream) {
  LnGroups G;
  memset(&G, 0, sizeof(G));
  G.ngroups = 1;
  G.row_end[0] = rows;
  G.scale[0] = scale;
  G.shift[0] = shift;
  return ln_launch_common(x, ldx, out, ldo, rows, dim, G, rows_per_batch, mod_stride, stream);
}

// ------------------------------------------------------------------------- gemv
// y[b, n] = bf16( sum_k act(x[b, k]) * W[n, k] + bias[n] ),  act = identity | bf16(silu)
template <int NB>
__global__ void __launch_bounds__(256)
gemv_kernel(const bf16* __restrict__ x, int ldx, const bf16* __restrict__ W,
            const bf16* __restrict__ bias, bf16* __restrict__ y, int ldy, int N, int K, int act) {
  extern __shared__ float xs[];  // [NB][K]
  pdl_launch_dependents();
  pdl_wait();
  for (int i = threadIdx.x; i < NB * K; i += blockDim.x) {
    const int b = i / K, k = i - b * K;
    float v = __bfloat162float(x[static_cast<size_t>(b) * ldx + k]);
    if (act == 1) v = bf16_round(__fdiv_rn(v, 1.0f + expf(-v)));  // silu in fp32 -> bf16
    xs[i] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const int kchunks = K >> 3;  // 16-byte chunks per row
  for (int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < N; n += warps_total) {
    const uint4* wr = reinterpret_cast<const uint4*>(W + static_cast<size_t>(n) * K);
    float acc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[b] = 0.f;
    for (int c0 = lane; c0 < kchunks; c0 += 128) {
      uint4 u[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = c0 + 32 * q;
        u[q] = (c < kchunks) ? __ldg(wr + c) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = c0 + 32 * q;
        if (c < kchunks) {
          float2 w0 = unpack_bf16x2(u[q].x), w1 = unpack_bf16x2(u[q].y),
                 w2 = unpack_bf16x2(u[q].z), w3 = unpack_bf16x2(u[q].w);
#pragma unroll
          for (int b = 0; b < NB; ++b) {
            const float4* xp = reinterpret_cast<const float4*>(xs + b * K + c * 8);
            float4 xa = xp[0], xb = xp[1];
            acc[b] = fmaf(w0.x, xa.x, acc[b]); acc[b] = fmaf(w0.y, xa.y, acc[b]);
            acc[b] = fmaf(w1.x, xa.z, acc[b]); acc[b] = fmaf(w1.y, xa.w, acc[b]);
            acc[b] = fmaf(w2.x, xb.x, acc[b]); acc[b] = fmaf(w2.y, xb.y, acc[b]);
            acc[b] = fmaf(w3.x, xb.z, acc[b]); acc[b] = fmaf(w3.y, xb.w, acc[b]);
          }
        }
      }
    }
    const float bv = bias ? __bfloat162float(bias[n]) : 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float s = warp_sum(acc[b]);
      if (lane == 0) y[static_cast<size_t>(b) * ldy + n] = __float2bfloat16_rn(s + bv);
    }
  }
}

template <int NB>
static int gemv_set_attr() {
  static bool attr_set = false;
  if (!attr_set) {
    RF_CHECK_CUDA(cudaFuncSetAttribute(gemv_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       NB * 4096 * 4));
    attr_set = true;
  }
  return 0;
}
int gemv_init() {
  return (gemv_set_attr<1>() | gemv_set_attr<2>() | gemv_set_attr<4>() | gemv_set_attr<8>()) ? -2 : 0;
}

template <int NB>
static int gemv_launch_nb(const bf16* x, int ldx, const bf16* W, const bf16* bias, bf16* y,
                          int ldy, int N, int K, int act, cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(NB) * K * sizeof(float);
  if (int rc = gemv_set_attr<NB>()) return rc;
  int blocks = (N + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  ProfScope prof("gemv", 2.0 * NB * N * K, 2.0 * N * K, stream);
  RF_CHECK_CUDA(launch_pdl(gemv_kernel<NB>, dim3(blocks), dim3(256), smem, stream, x, ldx, W, bias, y, ldy, N, K, act));
  count_launch();
  return 0;
}

int gemv_launch(const bf16* x, int ldx, int batch, const bf16* W, const bf16* bias, bf16* y,
                int ldy, int N, int K, int act, cudaStream_t stream) {
  if (K % 8 != 0 || K <= 0 || K > 4096) {
    set_error("gemv: K must be a multiple of 8, <= 4096");
    return -1;
  }
  int done = 0;
  while (done < batch) {
    const int left = batch - done;
    const bf16* xb = x + static_cast<size_t>(done) * ldx;
    bf16* yb = y + static_cast<size_t>(done) * ldy;
    int rc, step;
    if (left >= 8) { rc = gemv_launch_nb<8>(xb, ldx, W, bias, yb, ldy, N, K, act, stream); step = 8; }
    else if (left >= 4) { rc = gemv_launch_nb<4>(xb, ldx, W, bias, yb, ldy, N, K, act, stream); step = 4; }
    else if (left >= 2) { rc = gemv_launch_nb<2>(xb, ldx, W, bias, yb, ldy, N, K, act, stream); step = 2; }
    else { rc = gemv_launch_nb<1>(xb, ldx, W, bias, yb, ldy, N, K, act, stream); step = 1; }
    if (rc) return rc;
    done += step;
  }
  return 0;
}

// ------------------------------------------------------------------------- timestep embedding
// out[b, 0:128] = cos(t_b * f_i), out[b, 128:256] = sin(t_b * f_i), f_i = exp(-ln(1e4) * i / 128)
// with t_b = bf16(t_in[b] * pre_scale) — the "* 1000" the reference applies in bf16
// (train_flux/flux/transformer.py:95,98).
__global__ void timestep_embed_kernel(const bf16* __restrict__ t, const int* __restrict__ step,
                                      int t_stride, float pre_scale, bf16* __restrict__ out,
                                      int batch) {
  const int b = blockIdx.x;
  const int i = threadIdx.x;  // 0..127
  if (b >= batch || i >= 128) return;
  const int idx = step ? *step : 0;
  const float tv = bf16_round(__fmul_rn(__bfloat162float(t[static_cast<size_t>(b) * t_stride + idx]),
                                        pre_scale));
  const float expo = __fdiv_rn(__fmul_rn(-9.210340371976184f, static_cast<float>(i)), 128.0f);
  const float f = expf(expo);
  const float arg = __fmul_rn(tv, f);
  out[static_cast<size_t>(b) * 256 + i] = __float2bfloat16_rn(cosf(arg));
  out[static_cast<size_t>(b) * 256 + 128 + i] = __float2bfloat16_rn(sinf(arg));
}

int timestep_embed_launch(const bf16* t, const int* step, int t_stride, float pre_scale, bf16* out,
                          int batch, cudaStream_t stream) {
  timestep_embed_kernel<<<batch, 128, 0, stream>>>(t, step, t_stride, pre_scale, out, batch);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------- small elementwise
__global__ void add3_kernel(const bf16* a, const bf16* b, const bf16* c, bf16* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = bf16_round(__bfloat162float(a[i]) + __bfloat162float(b[i]));
  out[i] = __float2bfloat16_rn(s + __bfloat162float(c[i]));
}
int add3_launch(const bf16* a, const bf16* b, const bf16* c, bf16* out, int n,
                cudaStream_t stream) {
  add3_kernel<<<(n + 255) / 256, 256, 0, stream>>>(a, b, c, out, n);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// x_{i+1} = bf16( float(x_i) + (sigma_{i+1} - sigma_i) * float(v) )
__global__ void euler_step_kernel(bf16* __restrict__ x, const bf16* __restrict__ v,
                                  const float* __restrict__ sigmas, const int* __restrict__ step,
                                  int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= n) return;
  const int s = *step;
  const float dt = __fsub_rn(sigmas[s + 1], sigmas[s]);
  uint4 ux = *reinterpret_cast<const uint4*>(x + i);
  uint4 uv = __ldg(reinterpret_cast<const uint4*>(v + i));
  uint32_t xs[4] = {ux.x, ux.y, ux.z, ux.w}, vs[4] = {uv.x, uv.y, uv.z, uv.w}, os[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float2 xf = unpack_bf16x2(xs[q]), vf = unpack_bf16x2(vs[q]);
    os[q] = pack_bf16x2(__fadd_rn(xf.x, __fmul_rn(dt, vf.x)), __fadd_rn(xf.y, __fmul_rn(dt, vf.y)));
  }
  *reinterpret_cast<uint4*>(x + i) = make_uint4(os[0], os[1], os[2], os[3]);
}
int euler_step_launch(bf16* x, const bf16* v, const float* sigmas, const int* step, int n,
                      cudaStream_t stream) {
  if (n % 8 != 0) {
    set_error("euler_step: n must be a multiple of 8");
    return -1;
  }
  const int threads = n / 8;
  RF_CHECK_CUDA(launch_pdl(euler_step_kernel, dim3((threads + 255) / 256), dim3(256), 0, stream, x, v, sigmas, step, n));
  count_launch();
  return 0;
}

// image classifier-free guidance (generate.py:270) then the Euler step above:
//   v = bf16( u + bf16( s * bf16(c - u) ) )   — torch's bf16 ops with the Python scalar s taken as fp32
//   x = bf16( float(x) + (sigma_{i+1} - sigma_i) * float(v) )
__global__ void image_guidance_step_kernel(bf16* __restrict__ x, const bf16* __restrict__ vc,
                                           const bf16* __restrict__ vu, const float* __restrict__ scale,
                                           const float* __restrict__ sigmas, const int* __restrict__ step, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= n) return;
  const int s = *step;
  const float dt = __fsub_rn(sigmas[s + 1], sigmas[s]);
  const float g = *scale;
  uint4 ux = *reinterpret_cast<const uint4*>(x + i);
  uint4 uc = __ldg(reinterpret_cast<const uint4*>(vc + i));
  uint4 uu = __ldg(reinterpret_cast<const uint4*>(vu + i));
  uint32_t xs[4] = {ux.x, ux.y, ux.z, ux.w}, cs[4] = {uc.x, uc.y, uc.z, uc.w}, us[4] = {uu.x, uu.y, uu.z, uu.w};
  uint32_t os[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float2 xf = unpack_bf16x2(xs[q]), cf = unpack_bf16x2(cs[q]), uf = unpack_bf16x2(us[q]);
    float v[2], xo[2];
    const float c2[2] = {cf.x, cf.y}, u2[2] = {uf.x, uf.y}, x2[2] = {xf.x, xf.y};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float d = bf16_round(__fsub_rn(c2[e], u2[e]));
      v[e] = bf16_round(__fadd_rn(u2[e], bf16_round(__fmul_rn(g, d))));
      xo[e] = __fadd_rn(x2[e], __fmul_rn(dt, v[e]));
    }
    os[q] = pack_bf16x2(xo[0], xo[1]);
  }
  *reinterpret_cast<uint4*>(x + i) = make_uint4(os[0], os[1], os[2], os[3]);
}
int image_guidance_step_launch(bf16* x, const bf16* v_cond, const bf16* v_uncond, const float* scale,
                               const float* sigmas, const int* step, int n, cudaStream_t stream) {
  if (n % 8 != 0) {
    set_error("image_guidance_step: n must be a multiple of 8");
    return -1;
  }
  const int threads = n / 8;
  RF_CHECK_CUDA(launch_pdl(image_guidance_step_kernel, dim3((threads + 255) / 256), dim3(256), 0, stream, x, v_cond,
                           v_uncond, scale, sigmas, step, n));
  count_launch();
  return 0;
}

__global__ void copy_rows_kernel(const bf16* __restrict__ src, int lds, bf16* __restrict__ dst,
                                 int ldd, int rows, int chunks_per_row) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(rows) * chunks_per_row;
  if (idx >= total) return;
  const int r = static_cast<int>(idx / chunks_per_row);
  const int c = static_cast<int>(idx - static_cast<long long>(r) * chunks_per_row);
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(r) * lds) + c;
  uint4* d = reinterpret_cast<uint4*>(dst + static_cast<size_t>(r) * ldd) + c;
  *d = __ldg(s);
}
int copy_rows_launch(const bf16* src, int lds, bf16* dst, int ldd, int rows, int cols,
                     cudaStream_t stream) {
  if (cols % 8 != 0) {
    set_error("copy_rows: cols must be a multiple of 8");
    return -1;
  }
  const long long total = static_cast<long long>(rows) * (cols / 8);
  if (total == 0) return 0;
  copy_rows_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, stream>>>(src, lds, dst, ldd,
                                                                             rows, cols / 8);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------- PIL-compatible resize
// Pillow ImagingResample, uint8: out = clip8((2^21 + sum_k pix_k * coeff_k) >> 22), horizontal pass
// into a uint8 intermediate, then vertical pass (tables from reflectionflow_b200/resize.py).
__global__ void resize_h_kernel(const uint8_t* __restrict__ in, int H, int W, uint8_t* __restrict__ out,
                                int OW, const int* __restrict__ bounds, const int* __restrict__ coef,
                                int ksize) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(H) * OW) return;
  const int y = static_cast<int>(i / OW), xx = static_cast<int>(i - static_cast<long long>(y) * OW);
  const int x0 = bounds[2 * xx], n = bounds[2 * xx + 1];
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  const uint8_t* row = in + (static_cast<size_t>(y) * W + x0) * 3;
  for (int k = 0; k < n; ++k) {
    const int c = coef[xx * ksize + k];
    a0 += row[3 * k] * c; a1 += row[3 * k + 1] * c; a2 += row[3 * k + 2] * c;
  }
  uint8_t* o = out + i * 3;
  o[0] = static_cast<uint8_t>(min(max(a0 >> 22, 0), 255));
  o[1] = static_cast<uint8_t>(min(max(a1 >> 22, 0), 255));
  o[2] = static_cast<uint8_t>(min(max(a2 >> 22, 0), 255));
}
__global__ void resize_v_kernel(const uint8_t* __restrict__ in, int H, int W, uint8_t* __restrict__ out,
                                int OH, const int* __restrict__ bounds, const int* __restrict__ coef,
                                int ksize) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(OH) * W) return;
  const int yy = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<long long>(yy) * W);
  const int y0 = bounds[2 * yy], n = bounds[2 * yy + 1];
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int k = 0; k < n; ++k) {
    const int c = coef[yy * ksize + k];
    const uint8_t* px = in + (static_cast<size_t>(y0 + k) * W + x) * 3;
    a0 += px[0] * c; a1 += px[1] * c; a2 += px[2] * c;
  }
  uint8_t* o = out + i * 3;
  o[0] = static_cast<uint8_t>(min(max(a0 >> 22, 0), 255));
  o[1] = static_cast<uint8_t>(min(max(a1 >> 22, 0), 255));
  o[2] = static_cast<uint8_t>(min(max(a2 >> 22, 0), 255));
}
int resize_u8_launch(const uint8_t* in, int H, int W, uint8_t* tmp, uint8_t* out, int OH, int OW,
                     const int* bx, const int* kx, int ksx, const int* by, const int* ky, int ksy,
                     cudaStream_t stream) {
  const long long n1 = static_cast<long long>(H) * OW, n2 = static_cast<long long>(OH) * OW;
  resize_h_kernel<<<static_cast<int>((n1 + 255) / 256), 256, 0, stream>>>(in, H, W, tmp, OW, bx, kx, ksx);
  RF_CHECK_CUDA(cudaGetLastError());
  resize_v_kernel<<<static_cast<int>((n2 + 255) / 256), 256, 0, stream>>>(tmp, H, OW, out, OH, by, ky, ksy);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return 0;
}

}  // namespace rf
