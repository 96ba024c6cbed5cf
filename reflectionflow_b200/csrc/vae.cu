// vae.cu — FLUX VAE decoder (diffusers AutoencoderKL.decode) on sm_90a, behind rf_vae_* (C ABI).
//
// Replaces `vae.decode(latents / scaling + shift)` + `image_processor.postprocess` at
// train_flux/flux/generate.py:302-307 (and diffusers FluxPipeline.__call__'s tail): packed latents
// [n, 64] in, uint8 HWC image (or bf16 CHW tensor) out, everything in between on the device.
//
// Layout: activations are NHWC bf16 with a one-pixel zero ring, flattened to [(H+2)(W+2), C], so a
// 3x3 convolution is an implicit GEMM whose A tile for tap (dy, dx) is just a row-shifted TMA box
// of the same tensor (gemm_sm90.cu, conv mode: wgmma, bias / residual fused in
// the epilogue).  GroupNorm(32)+SiLU, nearest 2x upsampling, the latent unpack and the uint8
// post-process are bandwidth kernels here.  The mid-block self-attention (16384 tokens, one head of
// 512) runs as QK^T GEMM -> row softmax -> PV GEMM on the same GEMM kernel.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/rf_b200.h"
#include "rf_internal.h"
#include "rf_ptx.cuh"

namespace rf {

// ------------------------------------------------------------------ weight repack
// torch conv weight [Cout, Cin, kh, kw] -> [Cout_pad, (kh*kw) * Cin_pad], tap-major K, zero padded
__global__ void repack_conv_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int Cout,
                                   int Cin, int taps, int Cin_pad, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int K = taps * Cin_pad;
  const int co = static_cast<int>(i / K);
  const int r = static_cast<int>(i - static_cast<long long>(co) * K);
  const int tap = r / Cin_pad, ci = r - tap * Cin_pad;
  bf16 v = __float2bfloat16_rn(0.f);
  if (co < Cout && ci < Cin) v = src[(static_cast<size_t>(co) * Cin + ci) * taps + tap];
  dst[i] = v;
}

// ------------------------------------------------------------------ latents -> padded NHWC
// packed [ (h/2)(w/2), 64 ] -> z[c, y, x] (FluxPipeline._unpack_latents) -> bf16(bf16(z / s) + shift)
// -> padded NHWC [(h+2)(w+2), 64] with channels 16..63 zero.
__global__ void unpack_latents_kernel(const bf16* __restrict__ packed, bf16* __restrict__ out, int h,
                                      int w, float scaling, float shift) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // pixel * 16 + c
  if (idx >= h * w * 16) return;
  const int c = idx & 15, pix = idx >> 4;
  const int y = pix / w, x = pix - y * w;
  const int tok = (y >> 1) * (w >> 1) + (x >> 1);
  const int ch = c * 4 + (y & 1) * 2 + (x & 1);
  const float v = __bfloat162float(packed[static_cast<size_t>(tok) * 64 + ch]);
  const float z = bf16_round(__fdiv_rn(v, scaling));
  out[(static_cast<size_t>(y + 1) * (w + 2) + x + 1) * 64 + c] = __float2bfloat16_rn(z + shift);
}

// ------------------------------------------------------------------ GroupNorm(32)
// stats over the interior of a padded NHWC tensor; one (sum, sumsq) pair per 4-channel subgroup.
// Deterministic (no atomics): fixed-order reduction inside the block, one partial row per block,
// partial rows summed in block order by the finalize kernel — a run-to-run difference in the last
// bit of a mean could flip a bf16 rounding downstream and with it a candidate's score.
// The sums are of x - p, p = the group's first channel at the first interior pixel: E[x^2] - E[x]^2 from fp32 sums
// of x itself loses (mean / std)^2 of the variance's bits (2.9e-3 relative error of 1 / std at mean / std = 128 and
// 1024^2 pixels); shifted by a sample of the group, the sums hold the spread around that sample instead.
__global__ void __launch_bounds__(256)
gn_stats_kernel(const bf16* __restrict__ x, int H, int W, int C, int padded, float* __restrict__ part) {
  __shared__ float sm[256][4];
  const int nsub = C >> 2, oct = C >> 3;
  const int pix_per_iter = blockDim.x / oct;
  const int my_oct = threadIdx.x % oct, my_p = threadIdx.x / oct;
  const int npix = H * W;  // <= 2^22 for every supported image size: 32-bit index arithmetic, a shift when W = 2^k
  const int wshift = (W & (W - 1)) == 0 ? __ffs(W) - 1 : -1;
  float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
  if (my_p < pix_per_iter) {
    const int cpg = C / 32;
    const bf16* first = x + (padded ? static_cast<size_t>(W + 3) : 0) * C;
    const float p0 = __bfloat162float(first[(my_oct * 8) / cpg * cpg]);
    const float p1 = __bfloat162float(first[(my_oct * 8 + 4) / cpg * cpg]);
    for (int p = blockIdx.x * pix_per_iter + my_p; p < npix; p += gridDim.x * pix_per_iter) {
      const int y = wshift >= 0 ? (p >> wshift) : (p / W), xx = p - y * W;
      const size_t row = padded ? static_cast<size_t>(y + 1) * (W + 2) + xx + 1 : static_cast<size_t>(p);
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + row * C) + my_oct);
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
                   d = unpack_bf16x2(u.w);
      const float a0 = a.x - p0, a1 = a.y - p0, b0 = b.x - p0, b1 = b.y - p0;
      const float c0 = c.x - p1, c1 = c.y - p1, d0 = d.x - p1, d1 = d.y - p1;
      s0 += a0 + a1 + b0 + b1;
      q0 += a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1;
      s1 += c0 + c1 + d0 + d1;
      q1 += c0 * c0 + c1 * c1 + d0 * d0 + d1 * d1;
    }
  }
  sm[threadIdx.x][0] = s0; sm[threadIdx.x][1] = q0; sm[threadIdx.x][2] = s1; sm[threadIdx.x][3] = q1;
  __syncthreads();
  if (threadIdx.x < nsub) {  // subgroup sg = 2 * octet + half
    const int o = threadIdx.x >> 1, hf = threadIdx.x & 1;
    float s = 0.f, q = 0.f;
    for (int pp = 0; pp < pix_per_iter; ++pp) {
      s += sm[pp * oct + o][2 * hf];
      q += sm[pp * oct + o][2 * hf + 1];
    }
    part[static_cast<size_t>(blockIdx.x) * 2 * nsub + threadIdx.x] = s;
    part[static_cast<size_t>(blockIdx.x) * 2 * nsub + nsub + threadIdx.x] = q;
  }
}
// one warp per group: lane l sums partials l, l + 32, ... in double, then a fixed shuffle tree (deterministic).
// (One thread per group walked 592 x C/128 dependent loads: 10-45 us per norm, 30 norms per decode.)
// The partials are sums of x - p (gn_stats_kernel); the finalize reads the same p and adds it back to the mean.
__global__ void __launch_bounds__(1024)
gn_finalize_kernel(const float* __restrict__ part, int nblocks, int C, double count, const bf16* __restrict__ x,
                   int W, int padded, float* __restrict__ mean_rstd) {
  const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;  // 32 groups
  const int nsub = C >> 2, per = nsub / 32;
  double s = 0, q = 0;
  for (int k = lane; k < nblocks * per; k += 32) {
    const int b = k / per, i = k - b * per;
    s += static_cast<double>(part[static_cast<size_t>(b) * 2 * nsub + g * per + i]);
    q += static_cast<double>(part[static_cast<size_t>(b) * 2 * nsub + nsub + g * per + i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) {
    const double pivot = __bfloat162float(x[(padded ? static_cast<size_t>(W + 3) : 0) * C + g * (C / 32)]);
    const double n = count * (C / 32);
    const double d = s / n;
    double var = q / n - d * d;
    if (var < 0) var = 0;
    mean_rstd[g] = static_cast<float>(pivot + d);
    mean_rstd[32 + g] = static_cast<float>(1.0 / sqrt(var + 1e-6));
  }
}
// y = [silu] bf16( (x - mean) * rstd * gamma + beta ), padded NHWC in -> padded or compact NHWC out
// One CTA walks image rows (grid.x) and a slice of each row (grid.y): a row's W pixels are contiguous in both the
// padded and the compact layout, so there is no per-element index arithmetic (the first version spent two 64-bit
// divisions per 8 channels and ran at 1.6 TB/s); the thread's 8 channels, their gamma / beta and group statistics are
// fixed over the whole loop (blockDim.x is a multiple of C / 8) and live in registers.
__global__ void __launch_bounds__(256)
gn_apply_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int H, int W, int C,
                const float* __restrict__ mean_rstd, const bf16* __restrict__ gamma,
                const bf16* __restrict__ beta, int silu, int in_padded, int out_padded) {
  const int oct = C >> 3;  // 16-byte vectors per pixel: 16, 32 or 64
  const int cpg = C / 32;
  const int o = threadIdx.x % oct;
  float g[8], b[8], mu[8], rs[8];
  {
    const uint4 ug = __ldg(reinterpret_cast<const uint4*>(gamma) + o);
    const uint4 ub = __ldg(reinterpret_cast<const uint4*>(beta) + o);
    const uint32_t gs[4] = {ug.x, ug.y, ug.z, ug.w}, bs[4] = {ub.x, ub.y, ub.z, ub.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 gv = unpack_bf16x2(gs[q]), bv = unpack_bf16x2(bs[q]);
      g[2 * q] = gv.x; g[2 * q + 1] = gv.y;
      b[2 * q] = bv.x; b[2 * q + 1] = bv.y;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int grp = (o * 8 + 2 * q + e) / cpg;
        mu[2 * q + e] = mean_rstd[grp];
        rs[2 * q + e] = mean_rstd[32 + grp];
      }
    }
  }
  const int row_vecs = W * oct;
  const int stride = blockDim.x * gridDim.y;
  for (int y = blockIdx.x; y < H; y += gridDim.x) {
    const size_t prow = static_cast<size_t>(y + 1) * (W + 2) + 1;
    const uint4* src = reinterpret_cast<const uint4*>(x + (in_padded ? prow : static_cast<size_t>(y) * W) * C);
    uint4* dst = reinterpret_cast<uint4*>(out + (out_padded ? prow : static_cast<size_t>(y) * W) * C);
    for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < row_vecs; j += stride) {
      const uint4 u = __ldg(src + j);
      const uint32_t xs[4] = {u.x, u.y, u.z, u.w};
      uint32_t os[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 xv = unpack_bf16x2(xs[q]);
        float y0 = bf16_round((xv.x - mu[2 * q]) * rs[2 * q] * g[2 * q] + b[2 * q]);
        float y1 = bf16_round((xv.y - mu[2 * q + 1]) * rs[2 * q + 1] * g[2 * q + 1] + b[2 * q + 1]);
        if (silu) {  // x * sigmoid(x); bf16 output: approximate exp / reciprocal are > 1e4 x finer than its rounding
          y0 = __fdividef(y0, 1.0f + __expf(-y0));
          y1 = __fdividef(y1, 1.0f + __expf(-y1));
        }
        os[q] = pack_bf16x2(y0, y1);
      }
      dst[j] = make_uint4(os[0], os[1], os[2], os[3]);
    }
  }
}

// nearest 2x: padded [(H+2)(W+2), C] -> padded [(2H+2)(2W+2), C]
__global__ void upsample2x_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int H, int W,
                                  int C) {
  const int oct = C >> 3;
  const long long total = static_cast<long long>(2 * H) * (2 * W) * oct;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / oct;
    const int o = static_cast<int>(i - p * oct);
    const int y = static_cast<int>(p / (2 * W)), xx = static_cast<int>(p - static_cast<long long>(y) * 2 * W);
    const size_t irow = static_cast<size_t>((y >> 1) + 1) * (W + 2) + (xx >> 1) + 1;
    const size_t orow = static_cast<size_t>(y + 1) * (2 * W + 2) + xx + 1;
    *(reinterpret_cast<uint4*>(out + orow * C) + o) = __ldg(reinterpret_cast<const uint4*>(x + irow * C) + o);
  }
}
// padded <-> compact row copies (mid-block attention works on a compact [HW, C] token matrix)
__global__ void repad_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int H, int W, int C,
                             int in_padded, int out_padded) {
  const int oct = C >> 3;
  const long long total = static_cast<long long>(H) * W * oct;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / oct;
    const int o = static_cast<int>(i - p * oct);
    const int y = static_cast<int>(p / W), xx = static_cast<int>(p - static_cast<long long>(y) * W);
    const size_t prow = static_cast<size_t>(y + 1) * (W + 2) + xx + 1;
    const size_t irow = in_padded ? prow : static_cast<size_t>(p);
    const size_t orow = out_padded ? prow : static_cast<size_t>(p);
    *(reinterpret_cast<uint4*>(out + orow * C) + o) = __ldg(reinterpret_cast<const uint4*>(x + irow * C) + o);
  }
}
// in-place row softmax of a bf16 score matrix: p = softmax(s * scale) (fp32 math, bf16 out).  Rows have n
// columns (n % 8 == 0); the keys [valid, n) are padding: probability 0, outside the max and the row sum.
__global__ void __launch_bounds__(256)
softmax_rows_kernel(bf16* __restrict__ s, int n, int valid, float scale) {
  __shared__ float red[8];
  bf16* row = s + static_cast<size_t>(blockIdx.x) * n;
  const float sl = scale * 1.4426950408889634f;
  // padded columns read as -inf: exp2(-inf) = 0 leaves the max and the sum exactly as without them
  auto load = [&](int i, float (&v)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 f = unpack_bf16x2(w[q]);
      v[2 * q] = i + 2 * q < valid ? f.x : -INFINITY;
      v[2 * q + 1] = i + 2 * q + 1 < valid ? f.y : -INFINITY;
    }
  };
  float mx = -INFINITY;
  for (int i = threadIdx.x * 8; i < n; i += blockDim.x * 8) {
    float v[8];
    load(i, v);
    mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])), fmaxf(fmaxf(v[4], v[5]), fmaxf(v[6], v[7]))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x * 8; i < n; i += blockDim.x * 8) {
    float v[8];
    load(i, v);
#pragma unroll
    for (int q = 0; q < 4; ++q) sum += exp2f((v[2 * q] - mx) * sl) + exp2f((v[2 * q + 1] - mx) * sl);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x * 8; i < n; i += blockDim.x * 8) {
    float v[8];
    load(i, v);
    uint32_t o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      o[q] = pack_bf16x2(exp2f((v[2 * q] - mx) * sl) * inv, exp2f((v[2 * q + 1] - mx) * sl) * inv);
    *reinterpret_cast<uint4*>(row + i) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
// out[c, r] = in[r, c]  (V^T for the PV GEMM), in: [rows, ld_in] slice of cols [0, cols)
__global__ void transpose_kernel(const bf16* __restrict__ in, int ld_in, bf16* __restrict__ out,
                                 int rows, int cols) {
  __shared__ bf16 tile[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y)
    tile[j][threadIdx.x] = in[static_cast<size_t>(r0 + j) * ld_in + c0 + threadIdx.x];
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y)
    out[static_cast<size_t>(c0 + j) * rows + r0 + threadIdx.x] = tile[threadIdx.x][j];
}
// padded NHWC [.., C] (first 3 channels) -> uint8 HWC  (VaeImageProcessor.postprocess) and/or bf16 CHW
__global__ void postprocess_kernel(const bf16* __restrict__ x, int H, int W, int C,
                                   uint8_t* __restrict__ u8, bf16* __restrict__ chw) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(H) * W) return;
  const int y = static_cast<int>(i / W), xx = static_cast<int>(i - static_cast<long long>(y) * W);
  const bf16* px = x + (static_cast<size_t>(y + 1) * (W + 2) + xx + 1) * C;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __bfloat162float(px[c]);
    if (chw) chw[(static_cast<size_t>(c) * H + y) * W + xx] = px[c];
    if (u8) {
      float t = bf16_round(v * 0.5f);  // image / 2 (bf16) + 0.5 (bf16), clamp, * 255, round-half-even
      t = bf16_round(t + 0.5f);
      t = fminf(fmaxf(t, 0.f), 1.f);
      u8[i * 3 + c] = static_cast<uint8_t>(rintf(t * 255.0f));
    }
  }
}

// image -> padded NHWC [(H+2)(W+2), 64] (3 real channels): VaeImageProcessor.preprocess
// (uint8 / 255 -> 2x - 1 in fp32, then .to(bf16)); `chw` (bf16 [3,H,W] already in [-1,1]) is the
// alternative input
__global__ void image_to_nhwc_kernel(const uint8_t* __restrict__ u8, const bf16* __restrict__ chw,
                                     bf16* __restrict__ out, int H, int W) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(H) * W) return;
  const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<long long>(y) * W);
  bf16* px = out + (static_cast<size_t>(y + 1) * (W + 2) + x + 1) * 64;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (u8) {
      const float v = static_cast<float>(u8[i * 3 + c]) / 255.0f;
      px[c] = __float2bfloat16_rn(2.0f * v - 1.0f);
    } else {
      px[c] = chw[(static_cast<size_t>(c) * H + y) * W + x];
    }
  }
}
// moments (padded NHWC, channels 0..15 mean, 16..31 logvar) -> posterior sample -> (z - shift) * scale
// -> FluxPipeline._pack_latents layout [(h/2)(w/2), 64].  eps: bf16 [16, h, w] or NULL (mode).
// Rounding points of diffusers DiagonalGaussianDistribution + pipeline_tools.py:10-14 in bf16.
__global__ void sample_pack_kernel(const bf16* __restrict__ mom, int C, const bf16* __restrict__ eps,
                                   bf16* __restrict__ packed, int h, int w, float scaling, float shift) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // pixel * 16 + c
  if (idx >= h * w * 16) return;
  const int c = idx & 15, pix = idx >> 4;
  const int y = pix / w, x = pix - y * w;
  const bf16* px = mom + (static_cast<size_t>(y + 1) * (w + 2) + x + 1) * C;
  const float mean = __bfloat162float(px[c]);
  float z = mean;
  if (eps) {
    float lv = fminf(fmaxf(__bfloat162float(px[16 + c]), -30.0f), 20.0f);
    const float sd = bf16_round(expf(bf16_round(0.5f * lv)));
    const float e = __bfloat162float(eps[(static_cast<size_t>(c) * h + y) * w + x]);
    z = bf16_round(mean + bf16_round(sd * e));
  }
  z = bf16_round(z - shift);
  z = bf16_round(z * scaling);
  const int tok = (y >> 1) * (w >> 1) + (x >> 1);
  const int ch = c * 4 + (y & 1) * 2 + (x & 1);
  packed[static_cast<size_t>(tok) * 64 + ch] = __float2bfloat16_rn(z);
}

// ------------------------------------------------------------------ launchers (rf_internal.h)
static int grid_for(long long work, int threads = 256) {
  long long b = (work + threads - 1) / threads;
  if (b > 132 * 16) b = 132 * 16;
  return static_cast<int>(b < 1 ? 1 : b);
}

int conv_repack_launch(const bf16* src, bf16* dst, int Cout, int Cin, int taps, int Cout_pad, int Cin_pad,
                       cudaStream_t stream) {
  const long long total = static_cast<long long>(Cout_pad) * taps * Cin_pad;
  repack_conv_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, stream>>>(src, dst, Cout, Cin, taps, Cin_pad,
                                                                                total);
  RF_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int group_norm_launch(const bf16* x, bf16* out, int H, int W, int C, const bf16* gamma, const bf16* beta, int silu,
                      int in_padded, int out_padded, float* part, float* mean_rstd, cudaStream_t s) {
  if (C % 128 != 0 || 256 % (C / 8) != 0) {
    set_error("group_norm: channels must be 128, 256 or 512");
    return -1;
  }
  {
    ProfScope prof("vae_gn_stats", 0, 2.0 * H * W * C, s);
    gn_stats_kernel<<<kGnBlocks, 256, 0, s>>>(x, H, W, C, in_padded, part);
  }
  RF_CHECK_CUDA(cudaGetLastError());
  gn_finalize_kernel<<<1, 1024, 0, s>>>(part, kGnBlocks, C, static_cast<double>(H) * W, x, W, in_padded, mean_rstd);
  {
    ProfScope prof("vae_gn_apply", 0, 4.0 * H * W * C, s);
    // rows x row slices: ~16 CTAs per SM in flight, every thread >= 1 vector of its row slice
    const int rows = H < 132 * 16 ? H : 132 * 16;
    int slices = (132 * 16 + rows - 1) / rows;
    const int max_slices = (W * (C / 8) + 255) / 256;
    if (slices > max_slices) slices = max_slices;
    gn_apply_kernel<<<dim3(rows, slices), 256, 0, s>>>(x, out, H, W, C, mean_rstd, gamma, beta, silu, in_padded,
                                                      out_padded);
  }
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch(3);
  return 0;
}

int unpack_latents_launch(const bf16* packed, bf16* out, int h, int w, float scaling, float shift,
                          cudaStream_t s) {
  unpack_latents_kernel<<<(h * w * 16 + 255) / 256, 256, 0, s>>>(packed, out, h, w, scaling, shift);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int upsample2x_launch(const bf16* x, bf16* out, int H, int W, int C, cudaStream_t s) {
  {
    ProfScope prof("vae_upsample", 0, 10.0 * H * W * C, s);
    upsample2x_kernel<<<grid_for(static_cast<long long>(4) * H * W * (C / 8)), 256, 0, s>>>(x, out, H, W, C);
  }
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int repad_launch(const bf16* x, bf16* out, int H, int W, int C, int in_padded, int out_padded, cudaStream_t s) {
  repad_kernel<<<grid_for(static_cast<long long>(H) * W * (C / 8)), 256, 0, s>>>(x, out, H, W, C, in_padded,
                                                                                out_padded);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int softmax_rows_launch(bf16* S, int rows, int n, int valid, float scale, cudaStream_t s) {
  {
    ProfScope prof("vae_softmax", 0, 4.0 * rows * n, s);
    softmax_rows_kernel<<<rows, 256, 0, s>>>(S, n, valid, scale);
  }
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int transpose_launch(const bf16* in, int ld_in, bf16* out, int rows, int cols, cudaStream_t s) {
  dim3 tg(cols / 32, rows / 32), tb(32, 8);
  transpose_kernel<<<tg, tb, 0, s>>>(in, ld_in, out, rows, cols);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int postprocess_launch(const bf16* x, int H, int W, int C, uint8_t* u8, bf16* chw, cudaStream_t s) {
  postprocess_kernel<<<static_cast<int>((static_cast<long long>(H) * W + 255) / 256), 256, 0, s>>>(x, H, W, C, u8,
                                                                                                 chw);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int image_to_nhwc_launch(const uint8_t* u8, const bf16* chw, bf16* out, int H, int W, cudaStream_t s) {
  image_to_nhwc_kernel<<<static_cast<int>((static_cast<long long>(H) * W + 255) / 256), 256, 0, s>>>(u8, chw, out,
                                                                                                   H, W);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int sample_pack_launch(const bf16* mom, int C, const bf16* eps, bf16* packed, int h, int w, float scaling,
                       float shift, cudaStream_t s) {
  sample_pack_kernel<<<(h * w * 16 + 255) / 256, 256, 0, s>>>(mom, C, eps, packed, h, w, scaling, shift);
  RF_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace rf

using rf::bf16;

namespace {
struct ConvW {
  bf16* w = nullptr;   // repacked [Cout_pad, taps * Cin_pad]
  bf16* b = nullptr;   // [Cout_pad]
  int cin = 0, cout = 0, cin_pad = 0, cout_pad = 0, taps = 9;
};
struct Norm {
  bf16 *g = nullptr, *b = nullptr;
  int c = 0;
};
struct Resnet {
  Norm n1, n2;
  ConvW c1, c2, sc;
  bool has_sc = false;
};
struct LinearW {
  bf16 *w = nullptr, *b = nullptr;
};
}  // namespace

struct MidBlock {
  Resnet res[2];
  Norm attn_gn;
  LinearW attn_qkv, attn_out;  // to_q|to_k|to_v stacked [1536, 512]
};

struct rf_vae {
  rf::DeviceAllocs mem;     // weights, GroupNorm scratch, ones: live until destroy
  rf::DeviceAllocs ws_mem;  // the size-dependent workspace below
  rf::WeightTable weights;
  ConvW conv_in, conv_out;
  Norm norm_out;
  MidBlock mid;
  Resnet up[4][3];
  ConvW upconv[3];
  // encoder
  ConvW e_conv_in, e_conv_out;
  Norm e_norm_out;
  MidBlock e_mid;
  Resnet down[4][2];
  ConvW downconv[3];
  bf16* ones = nullptr;
  // workspace (sized for max_hw at first decode)
  int ws_h = 0, ws_w = 0;
  bf16* buf[4] = {nullptr, nullptr, nullptr, nullptr};
  long long tag[4] = {-1, -1, -1, -1};  // geometry (H, W, C) whose zero ring is currently valid
  bf16 *tok = nullptr, *tokx = nullptr, *qkv = nullptr, *S = nullptr, *vt = nullptr, *ao = nullptr, *ay = nullptr;
  float* gn_acc = nullptr;  // [kGnBlocks][2 * C/4] block partials
  float* gn_mr = nullptr;
  // ---- captured graphs: one decode / encode = ~150 launches whose tensor maps are encoded on the host, which made
  // the call host-bound (22 ms for 16 ms of kernels at 1024x1024).  The launch sequence of a geometry is captured
  // once on the side stream against staging buffers and replayed; RF_VAE_GRAPH=0 and profiling runs stay eager.
  struct Graph {
    int kind, height, width;            // kind 0 decode, 1 encode
    float scale, shift;
    int flags;                          // decode: 1 = u8 out, 2 = bf16 out; encode: 1 = u8 in, 2 = bf16 in, 4 = eps
    cudaGraphExec_t exec;
    long long tag_end[4];
    int64_t launches;
  };
  std::vector<Graph> graphs;
  rf::SideStream side;
  uint8_t* g_u8 = nullptr;              // [H, W, 3] image staging (decode output / encode input)
  bf16* g_chw = nullptr;                // [3, H, W]
  bf16* g_lat = nullptr;                // packed latents [(H/16)(W/16), 64]
  bf16* g_eps = nullptr;                // [16, H/8, W/8]
};

namespace {

int make_conv(rf_vae* h, ConvW& c, const std::string& key, int cin, int cout, int taps) {
  c.cin = cin; c.cout = cout; c.taps = taps;
  c.cin_pad = (cin + 63) / 64 * 64;
  c.cout_pad = (cout + 127) / 128 * 128;
  RF_TRY(h->mem.alloc(&c.w, static_cast<size_t>(c.cout_pad) * taps * c.cin_pad));
  RF_TRY(h->mem.alloc(&c.b, c.cout_pad));
  RF_CHECK_CUDA(cudaMemset(c.b, 0, static_cast<size_t>(c.cout_pad) * 2));
  h->weights.add(key + ".weight", c.w, static_cast<int64_t>(cout) * cin * taps,
                 rf::ConvRepack{cout, cin, taps, c.cout_pad, c.cin_pad});
  h->weights.add(key + ".bias", c.b, cout);
  return 0;
}
int make_norm(rf_vae* h, Norm& n, const std::string& key, int c) {
  n.c = c;
  RF_TRY(h->mem.alloc(&n.g, c));
  RF_TRY(h->mem.alloc(&n.b, c));
  h->weights.add(key + ".weight", n.g, c);
  h->weights.add(key + ".bias", n.b, c);
  return 0;
}
int make_resnet(rf_vae* h, Resnet& r, const std::string& key, int cin, int cout) {
  RF_TRY(make_norm(h, r.n1, key + ".norm1", cin));
  RF_TRY(make_conv(h, r.c1, key + ".conv1", cin, cout, 9));
  RF_TRY(make_norm(h, r.n2, key + ".norm2", cout));
  RF_TRY(make_conv(h, r.c2, key + ".conv2", cout, cout, 9));
  r.has_sc = cin != cout;
  if (r.has_sc) RF_TRY(make_conv(h, r.sc, key + ".conv_shortcut", cin, cout, 1));
  return 0;
}

int make_mid(rf_vae* h, MidBlock& m, const std::string& key) {
  RF_TRY(make_resnet(h, m.res[0], key + ".resnets.0", 512, 512));
  RF_TRY(make_resnet(h, m.res[1], key + ".resnets.1", 512, 512));
  RF_TRY(make_norm(h, m.attn_gn, key + ".attentions.0.group_norm", 512));
  RF_TRY(h->mem.alloc(&m.attn_qkv.w, static_cast<size_t>(1536) * 512));
  RF_TRY(h->mem.alloc(&m.attn_qkv.b, 1536));
  RF_TRY(h->mem.alloc(&m.attn_out.w, static_cast<size_t>(512) * 512));
  RF_TRY(h->mem.alloc(&m.attn_out.b, 512));
  const std::string a = key + ".attentions.0.";
  const char* nm[3] = {"to_q", "to_k", "to_v"};
  for (int j = 0; j < 3; ++j) {  // row slices of the stacked q | k | v projection
    h->weights.add(a + nm[j] + ".weight", m.attn_qkv.w + j * 512 * 512, 512 * 512);
    h->weights.add(a + nm[j] + ".bias", m.attn_qkv.b + j * 512, 512);
  }
  h->weights.add(a + "to_out.0.weight", m.attn_out.w, 512 * 512);
  h->weights.add(a + "to_out.0.bias", m.attn_out.b, 512);
  return 0;
}

size_t padded_elems(int H, int W, int C) { return static_cast<size_t>(H + 2) * (W + 2) * C; }
// keys of the mid-block attention, padded to whole 128-row tiles (the S GEMM's N, the PV GEMM's K)
int padded_tokens(int H, int W) { return (H * W + 127) / 128 * 128; }

int group_norm(rf_vae* h, const bf16* x, bf16* out, int H, int W, const Norm& n, int silu,
               int in_padded, int out_padded, cudaStream_t s) {
  return rf::group_norm_launch(x, out, H, W, n.c, n.g, n.b, silu, in_padded, out_padded, h->gn_acc, h->gn_mr, s);
}
int conv(rf_vae* h, const ConvW& c, const bf16* in, bf16* out, const bf16* res, int H, int W,
         cudaStream_t s) {
  return rf::conv_launch(in, c.w, c.b, out, res, h->ones, H, W, c.cin_pad, c.cout_pad, c.taps, 1, s);
}

void drop_graphs(rf_vae* h) {
  for (auto& g : h->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
}

// Every workspace size grows with the image height and width, so a workspace for (ws_h, ws_w) serves any
// image that fits inside both.  A larger request grows it to the larger of each side (a 1024x1024 call after a
// 768x1344 one makes room for 1024x1344), so alternating shapes allocate once, and frees the old one.
int ensure_workspace(rf_vae* h, int H, int W) {  // H, W: output image size
  if (h->ws_h >= H && h->ws_w >= W && h->buf[0]) return 0;
  drop_graphs(h);  // they reference the old workspace
  if (H < h->ws_h) H = h->ws_h;
  if (W < h->ws_w) W = h->ws_w;
  if (h->buf[0]) RF_CHECK_CUDA(cudaDeviceSynchronize());  // work still queued on the old buffers
  h->ws_mem.release_all();
  h->ws_h = h->ws_w = 0;  // stays 0 if an allocation below fails: the next call starts over
  for (int i = 0; i < 4; ++i) h->tag[i] = -1;
  const int lh = H / 8, lw = W / 8;
  rf::DeviceAllocs& m = h->ws_mem;
  RF_TRY(m.alloc(&h->g_u8, static_cast<size_t>(H) * W * 3));
  RF_TRY(m.alloc(&h->g_chw, static_cast<size_t>(H) * W * 3));
  RF_TRY(m.alloc(&h->g_lat, static_cast<size_t>(H / 16) * (W / 16) * 64));
  RF_TRY(m.alloc(&h->g_eps, static_cast<size_t>(lh) * lw * 16));
  // largest padded tensor: full resolution x 256 channels (input of up_blocks.2's upsampler conv)
  for (int i = 0; i < 4; ++i) RF_TRY(m.alloc(&h->buf[i], padded_elems(H, W, 256)));
  // mid-block attention (decoder at H/8 x W/8; the encoder's is the same size): qkv, the staged K (ay) and V^T
  // run to the padded key count
  const size_t ntok = static_cast<size_t>(lh) * lw, npad = padded_tokens(lh, lw);
  RF_TRY(m.alloc(&h->tok, ntok * 512));
  RF_TRY(m.alloc(&h->tokx, ntok * 512));
  RF_TRY(m.alloc(&h->qkv, npad * 1536));
  RF_TRY(m.alloc(&h->S, ntok * npad));
  RF_TRY(m.alloc(&h->vt, npad * 512));
  RF_TRY(m.alloc(&h->ao, ntok * 512));
  RF_TRY(m.alloc(&h->ay, npad * 512));
  if (!h->gn_acc) {
    RF_TRY(h->mem.alloc(&h->gn_acc, rf::gn_part_floats));
    RF_TRY(h->mem.alloc(&h->gn_mr, 64));
  }
  h->ws_h = H; h->ws_w = W;
  return 0;
}

// Every writer touches interior pixels only; a buffer's one-pixel zero ring has to be re-established
// whenever the geometry of what it holds changes.
int prep(rf_vae* h, int i, int H, int W, int C, cudaStream_t s) {
  const long long tag = (static_cast<long long>(H) << 40) | (static_cast<long long>(W) << 20) | C;
  if (h->tag[i] == tag) return 0;
  RF_CHECK_CUDA(cudaMemsetAsync(h->buf[i], 0, padded_elems(H, W, C) * 2, s));
  h->tag[i] = tag;
  return 0;
}
// ResnetBlock2D: buf[x] -> buf[out], scratch buf[t1], buf[t2]
int resnet(rf_vae* h, const Resnet& r, int x, int out, int t1, int t2, int H, int W, cudaStream_t s) {
  const int cin = r.c1.cin_pad, cout = r.c1.cout_pad;
  RF_TRY(prep(h, t1, H, W, cin, s));
  RF_TRY(group_norm(h, h->buf[x], h->buf[t1], H, W, r.n1, 1, 1, 1, s));
  RF_TRY(prep(h, t2, H, W, cout, s));
  RF_TRY(conv(h, r.c1, h->buf[t1], h->buf[t2], nullptr, H, W, s));
  RF_TRY(prep(h, t1, H, W, cout, s));
  RF_TRY(group_norm(h, h->buf[t2], h->buf[t1], H, W, r.n2, 1, 1, 1, s));
  RF_TRY(prep(h, out, H, W, cout, s));
  const bf16* shortcut = h->buf[x];
  if (r.has_sc) {
    RF_TRY(conv(h, r.sc, h->buf[x], h->buf[out], nullptr, H, W, s));  // 1x1 shortcut, into `out`
    shortcut = h->buf[out];
  }
  // out = shortcut + conv2(t1): each residual box is read before the same box is stored (in place ok)
  return conv(h, r.c2, h->buf[t1], h->buf[out], shortcut, H, W, s);
}

// The mid-block's self-attention over H*W tokens (1 head x 512): x (padded) -> out (padded, interior only).
// The keys run to npad = padded_tokens(H, W): K / V rows [ntok, npad) are zero and the softmax gives them
// probability 0, so the padding changes no result.  With ntok % 128 == 0 there is no padding.
int mid_attention(rf_vae* h, const MidBlock& m, const bf16* x, bf16* out, int H, int W, cudaStream_t s) {
  const int ntok = H * W, npad = padded_tokens(H, W);
  RF_TRY(rf::group_norm_launch(x, h->tok, H, W, 512, m.attn_gn.g, m.attn_gn.b, 0, 1, 0, h->gn_acc, h->gn_mr,
                                s));  // compact tokens
  RF_TRY(rf::repad_launch(x, h->tokx, H, W, 512, 1, 0, s));
  rf::GemmGroupArgs g;
  memset(&g, 0, sizeof(g));  // q | k | v
  g.A = h->tok; g.lda = 512; g.M = ntok; g.W = m.attn_qkv.w; g.bias = m.attn_qkv.b;
  g.out = h->qkv; g.ldo = 1536;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, 1536, 512, 1, &g, s));
  // q | k | v rows of the padding keys (the GEMM writes rows [0, ntok) only)
  if (npad > ntok)
    RF_CHECK_CUDA(cudaMemsetAsync(h->qkv + static_cast<size_t>(ntok) * 1536, 0,
                                  static_cast<size_t>(npad - ntok) * 1536 * 2, s));
  // the GEMM's W operand is [N, K] with pitch K: stage K compactly (ay is free until the out-proj)
  RF_CHECK_CUDA(cudaMemcpy2DAsync(h->ay, 512 * 2, h->qkv + 512, 1536 * 2, 512 * 2, npad,
                                  cudaMemcpyDeviceToDevice, s));
  memset(&g, 0, sizeof(g));  // S = Q K^T  [ntok, npad]
  g.A = h->qkv; g.lda = 1536; g.M = ntok; g.W = h->ay; g.out = h->S; g.ldo = npad;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, npad, 512, 1, &g, s));
  RF_TRY(rf::softmax_rows_launch(h->S, ntok, npad, ntok, 1.0f / sqrtf(512.0f), s));
  RF_TRY(rf::transpose_launch(h->qkv + 1024, 1536, h->vt, npad, 512, s));  // V^T [512, npad]
  memset(&g, 0, sizeof(g));  // O = P V
  g.A = h->S; g.lda = npad; g.M = ntok; g.W = h->vt; g.out = h->ao; g.ldo = 512;
  RF_TRY(rf::gemm_launch(rf::EPI_BIAS, 512, npad, 1, &g, s));
  memset(&g, 0, sizeof(g));  // y = x + to_out(O)
  g.A = h->ao; g.lda = 512; g.M = ntok; g.W = m.attn_out.w; g.bias = m.attn_out.b;
  g.out = h->ay; g.ldo = 512; g.res = h->tokx; g.ldr = 512; g.gate = h->ones;
  RF_TRY(rf::gemm_launch(rf::EPI_GATE_RES, 512, 512, 1, &g, s));
  return rf::repad_launch(h->ay, out, H, W, 512, 0, 1, s);
}

// UNetMidBlock2D: resnet, self-attention, resnet.  buf[x] -> buf[x].
int mid_block(rf_vae* h, const MidBlock& m, int& x, int& y, int t1, int t2, int H, int W, cudaStream_t s) {
  RF_TRY(resnet(h, m.res[0], x, y, t1, t2, H, W, s));
  std::swap(x, y);
  RF_TRY(prep(h, y, H, W, 512, s));
  RF_TRY(mid_attention(h, m, h->buf[x], h->buf[y], H, W, s));
  std::swap(x, y);
  RF_TRY(resnet(h, m.res[1], x, y, t1, t2, H, W, s));
  std::swap(x, y);
  return 0;
}

// Any image whose sides are multiples of 16 (one latent token = 16 x 16 pixels), as diffusers' FLUX pipeline
// accepts.  The cap keeps pixel indices in 32 bits; well below it the workspace (the mid-block's
// (H/8 * W/8)^2 score matrix) outgrows the device, and ensure_workspace reports the failed allocation.
int check_size(const char* fn, int height, int width) {
  if (height % 16 != 0 || width % 16 != 0 || height < 16 || width < 16 || height > 16384 || width > 16384) {
    rf::set_error(std::string(fn) + ": height and width must be multiples of 16 in [16, 16384], got " +
                  std::to_string(height) + "x" + std::to_string(width));
    return -1;
  }
  return 0;
}

bool use_graphs() {
  const char* e = getenv("RF_VAE_GRAPH");
  return !(e && atoi(e) == 0) && !rf::prof_on();
}
// replay the graph of (kind, geometry, factors, flags), capturing `body` first if it does not exist yet.  The
// capture starts from "no zero ring valid", so a replay re-establishes every ring it relies on, whatever ran before.
int run_graph(rf_vae* h, int kind, int height, int width, float scale, float shift, int flags, cudaStream_t s,
              const std::function<int()>& body) {
  rf_vae::Graph* g = nullptr;
  for (auto& c : h->graphs)
    if (c.kind == kind && c.height == height && c.width == width && c.scale == scale && c.shift == shift &&
        c.flags == flags)
      g = &c;
  if (!g) {
    for (int i = 0; i < 4; ++i) h->tag[i] = -1;
    rf_vae::Graph ng{kind, height, width, scale, shift, flags, nullptr, {0, 0, 0, 0}, 0};
    const int rc = rf::capture_graph(s, "rf_vae", body, &ng.exec, &ng.launches);
    if (rc) {
      for (int i = 0; i < 4; ++i) h->tag[i] = -1;
      return rc;
    }
    for (int i = 0; i < 4; ++i) ng.tag_end[i] = h->tag[i];
    if (h->graphs.size() >= 8) {  // a handful of geometries in practice (decode 1024, encode 512)
      if (h->graphs.front().exec) cudaGraphExecDestroy(h->graphs.front().exec);
      h->graphs.erase(h->graphs.begin());
    }
    h->graphs.push_back(ng);
    g = &h->graphs.back();
  }
  RF_CHECK_CUDA(cudaGraphLaunch(g->exec, s));
  rf::count_launch(static_cast<int>(g->launches));
  for (int i = 0; i < 4; ++i) h->tag[i] = g->tag_end[i];
  return 0;
}

}  // namespace

extern "C" {

static int decode_body(rf_vae* h, const void* packed_latents, int height, int width, float scaling_factor,
                       float shift_factor, uint8_t* out_u8_hwc, void* out_bf16_chw, cudaStream_t s);
static int encode_body(rf_vae* h, const uint8_t* image_u8_hwc, const void* image_bf16_chw, int height, int width,
                       const void* eps_bf16_chw, float scaling_factor, float shift_factor, void* packed_out,
                       cudaStream_t s);

int rf_vae_create(rf_vae** out) {
  if (!out) {
    rf::set_error("rf_vae_create: null argument");
    return -1;
  }
  RF_TRY(rf::require_device("rf_vae_create"));
  rf_vae* h = new rf_vae();
  int rc = 0;
  auto chk = [&](int r) { if (r && !rc) rc = r; };
  chk(make_conv(h, h->conv_in, "decoder.conv_in", 16, 512, 9));
  chk(make_mid(h, h->mid, "decoder.mid_block"));
  const int chans[4] = {512, 512, 256, 128};
  int prev = 512;
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 3; ++j)
      chk(make_resnet(h, h->up[i][j],
                      "decoder.up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                      j == 0 ? prev : chans[i], chans[i]));
    if (i < 3)
      chk(make_conv(h, h->upconv[i], "decoder.up_blocks." + std::to_string(i) + ".upsamplers.0.conv",
                    chans[i], chans[i], 9));
    prev = chans[i];
  }
  chk(make_norm(h, h->norm_out, "decoder.conv_norm_out", 128));
  chk(make_conv(h, h->conv_out, "decoder.conv_out", 128, 3, 9));
  // ---- encoder (diffusers Encoder: conv_in, 4 down blocks x 2 resnets, mid block, norm, conv_out)
  chk(make_conv(h, h->e_conv_in, "encoder.conv_in", 3, 128, 9));
  {
    const int ech[4] = {128, 256, 512, 512};
    int ep = 128;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j)
        chk(make_resnet(h, h->down[i][j],
                        "encoder.down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j),
                        j == 0 ? ep : ech[i], ech[i]));
      if (i < 3)
        chk(make_conv(h, h->downconv[i],
                      "encoder.down_blocks." + std::to_string(i) + ".downsamplers.0.conv", ech[i], ech[i], 9));
      ep = ech[i];
    }
  }
  chk(make_mid(h, h->e_mid, "encoder.mid_block"));
  chk(make_norm(h, h->e_norm_out, "encoder.conv_norm_out", 512));
  chk(make_conv(h, h->e_conv_out, "encoder.conv_out", 512, 32, 9));
  chk(h->mem.alloc(&h->ones, 512));
  const std::vector<uint16_t> one(512, 0x3F80);
  if (!rc && cudaMemcpy(h->ones, one.data(), 1024, cudaMemcpyHostToDevice) != cudaSuccess) rc = -2;
  if (rc) {
    rf_vae_destroy(h);
    return rc;
  }
  *out = h;
  return 0;
}

void rf_vae_destroy(rf_vae* h) {
  if (!h) return;
  drop_graphs(h);
  h->side.destroy();
  h->ws_mem.release_all();
  h->mem.release_all();
  delete h;
}

int rf_vae_load_weight(rf_vae* h, const char* key, const void* src, int64_t numel) {
  if (!h || !key || !src) {
    rf::set_error("rf_vae_load_weight: null argument");
    return -1;
  }
  RF_TRY(h->weights.load("rf_vae_load_weight", key, src, numel));
  RF_CHECK_CUDA(cudaDeviceSynchronize());
  return 0;
}

int rf_vae_decode(rf_vae* h, const void* packed_latents, int height, int width, float scaling_factor,
                  float shift_factor, uint8_t* out_u8_hwc, void* out_bf16_chw, void* stream) {
  if (!h || !packed_latents || (!out_u8_hwc && !out_bf16_chw)) {
    rf::set_error("rf_vae_decode: null argument");
    return -1;
  }
  RF_TRY(check_size("rf_vae_decode", height, width));
  RF_TRY(ensure_workspace(h, height, width));
  if (h->weights.missing("decoder.", "missing VAE weights") != 0) return -4;
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  if (!use_graphs()) return decode_body(h, packed_latents, height, width, scaling_factor, shift_factor, out_u8_hwc,
                                        out_bf16_chw, caller);
  cudaStream_t s = nullptr;
  RF_TRY(h->side.enter(caller, &s));
  const size_t lat_bytes = static_cast<size_t>(height / 16) * (width / 16) * 64 * 2;
  RF_CHECK_CUDA(cudaMemcpyAsync(h->g_lat, packed_latents, lat_bytes, cudaMemcpyDeviceToDevice, s));
  const int flags = (out_u8_hwc ? 1 : 0) | (out_bf16_chw ? 2 : 0);
  RF_TRY(run_graph(h, 0, height, width, scaling_factor, shift_factor, flags, s, [&]() {
    return decode_body(h, h->g_lat, height, width, scaling_factor, shift_factor, out_u8_hwc ? h->g_u8 : nullptr,
                       out_bf16_chw ? h->g_chw : nullptr, s);
  }));
  const size_t px = static_cast<size_t>(height) * width * 3;
  if (out_u8_hwc) RF_CHECK_CUDA(cudaMemcpyAsync(out_u8_hwc, h->g_u8, px, cudaMemcpyDeviceToDevice, s));
  if (out_bf16_chw) RF_CHECK_CUDA(cudaMemcpyAsync(out_bf16_chw, h->g_chw, px * 2, cudaMemcpyDeviceToDevice, s));
  return h->side.leave(caller);
}

static int decode_body(rf_vae* h, const void* packed_latents, int height, int width, float scaling_factor,
                       float shift_factor, uint8_t* out_u8_hwc, void* out_bf16_chw, cudaStream_t s) {
  int H = height / 8, W = width / 8;
  int x = 0, y = 1;
  const int t1 = 2, t2 = 3;
  // ---- latents -> NHWC (16 real channels of 64), conv_in
  RF_TRY(prep(h, x, H, W, 64, s));
  RF_TRY(rf::unpack_latents_launch(static_cast<const bf16*>(packed_latents), h->buf[x], H, W, scaling_factor,
                                   shift_factor, s));
  RF_TRY(prep(h, y, H, W, 512, s));
  RF_TRY(conv(h, h->conv_in, h->buf[x], h->buf[y], nullptr, H, W, s));
  std::swap(x, y);
  RF_TRY(mid_block(h, h->mid, x, y, t1, t2, H, W, s));  // result back in buf[x]
  // ---- up blocks: 3 resnets each, nearest 2x + conv between them
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 3; ++j) {
      RF_TRY(resnet(h, h->up[i][j], x, y, t1, t2, H, W, s));
      std::swap(x, y);
    }
    if (i < 3) {
      const int C = h->upconv[i].cin_pad;
      RF_TRY(prep(h, y, 2 * H, 2 * W, C, s));
      RF_TRY(rf::upsample2x_launch(h->buf[x], h->buf[y], H, W, C, s));
      H *= 2;
      W *= 2;
      RF_TRY(prep(h, x, H, W, C, s));
      RF_TRY(conv(h, h->upconv[i], h->buf[y], h->buf[x], nullptr, H, W, s));
    }
  }
  // ---- norm_out + SiLU + conv_out (3 channels padded to 128) + post-process
  RF_TRY(prep(h, t1, H, W, 128, s));
  RF_TRY(group_norm(h, h->buf[x], h->buf[t1], H, W, h->norm_out, 1, 1, 1, s));
  RF_TRY(prep(h, y, H, W, 128, s));
  RF_TRY(conv(h, h->conv_out, h->buf[t1], h->buf[y], nullptr, H, W, s));
  return rf::postprocess_launch(h->buf[y], H, W, 128, out_u8_hwc, static_cast<bf16*>(out_bf16_chw), s);
}

int rf_vae_missing_weights(rf_vae* h) { return h ? h->weights.missing("", "missing VAE weights") : -1; }

}  // extern "C"

int vae_mid_attention(rf_vae* h, int encoder, const bf16* x, bf16* out, int H, int W, cudaStream_t s) {
  if (!h || !x || !out || H < 1 || W < 1 || H > 2048 || W > 2048) {
    rf::set_error("vae_mid_attention: null argument or latent size outside [1, 2048]");
    return -1;
  }
  if (h->weights.missing(encoder ? "encoder.mid_block.attentions." : "decoder.mid_block.attentions.",
                         "missing VAE weights") != 0)
    return -4;
  RF_TRY(ensure_workspace(h, 8 * H, 8 * W));
  return mid_attention(h, encoder ? h->e_mid : h->mid, x, out, H, W, s);
}

extern "C" {

/* image [H, W, 3] uint8 (or bf16 CHW in [-1, 1]) -> packed condition latents [(H/16)(W/16), 64]:
 * preprocess, encoder, posterior sample with caller-provided eps (NULL = mode), (z - shift) * scale,
 * pack.  Replaces encode_images() of train_flux/flux/pipeline_tools.py:7-30. */
int rf_vae_encode(rf_vae* h, const uint8_t* image_u8_hwc, const void* image_bf16_chw, int height,
                  int width, const void* eps_bf16_chw, float scaling_factor, float shift_factor,
                  void* packed_out, void* stream) {
  if (!h || (!image_u8_hwc && !image_bf16_chw) || !packed_out) {
    rf::set_error("rf_vae_encode: null argument");
    return -1;
  }
  RF_TRY(check_size("rf_vae_encode", height, width));
  RF_TRY(ensure_workspace(h, height, width));
  if (h->weights.missing("encoder.", "missing VAE weights") != 0) return -4;
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  if (!use_graphs()) return encode_body(h, image_u8_hwc, image_bf16_chw, height, width, eps_bf16_chw, scaling_factor,
                                        shift_factor, packed_out, caller);
  cudaStream_t s = nullptr;
  RF_TRY(h->side.enter(caller, &s));
  const size_t px = static_cast<size_t>(height) * width * 3;
  if (image_u8_hwc) RF_CHECK_CUDA(cudaMemcpyAsync(h->g_u8, image_u8_hwc, px, cudaMemcpyDeviceToDevice, s));
  else RF_CHECK_CUDA(cudaMemcpyAsync(h->g_chw, image_bf16_chw, px * 2, cudaMemcpyDeviceToDevice, s));
  const size_t eps_bytes = static_cast<size_t>(height / 8) * (width / 8) * 16 * 2;
  if (eps_bf16_chw) RF_CHECK_CUDA(cudaMemcpyAsync(h->g_eps, eps_bf16_chw, eps_bytes, cudaMemcpyDeviceToDevice, s));
  const int flags = (image_u8_hwc ? 1 : 2) | (eps_bf16_chw ? 4 : 0);
  RF_TRY(run_graph(h, 1, height, width, scaling_factor, shift_factor, flags, s, [&]() {
    return encode_body(h, image_u8_hwc ? h->g_u8 : nullptr, image_u8_hwc ? nullptr : h->g_chw, height, width,
                       eps_bf16_chw ? h->g_eps : nullptr, scaling_factor, shift_factor, h->g_lat, s);
  }));
  RF_CHECK_CUDA(cudaMemcpyAsync(packed_out, h->g_lat, static_cast<size_t>(height / 16) * (width / 16) * 64 * 2,
                                cudaMemcpyDeviceToDevice, s));
  return h->side.leave(caller);
}

static int encode_body(rf_vae* h, const uint8_t* image_u8_hwc, const void* image_bf16_chw, int height, int width,
                       const void* eps_bf16_chw, float scaling_factor, float shift_factor, void* packed_out,
                       cudaStream_t s) {
  int H = height, W = width;
  int x = 0, y = 1;
  const int t1 = 2, t2 = 3;
  RF_TRY(prep(h, x, H, W, 64, s));
  RF_TRY(rf::image_to_nhwc_launch(image_u8_hwc, static_cast<const bf16*>(image_bf16_chw), h->buf[x], H, W, s));
  RF_TRY(prep(h, y, H, W, 128, s));
  RF_TRY(conv(h, h->e_conv_in, h->buf[x], h->buf[y], nullptr, H, W, s));
  std::swap(x, y);
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 2; ++j) {
      RF_TRY(resnet(h, h->down[i][j], x, y, t1, t2, H, W, s));
      std::swap(x, y);
    }
    if (i < 3) {  // Downsample2D: pad (0,1,0,1) + conv3x3 stride 2 == strided taps over the zero ring
      const ConvW& c = h->downconv[i];
      H /= 2;
      W /= 2;
      RF_TRY(prep(h, y, H, W, c.cout_pad, s));
      RF_TRY(rf::conv_launch(h->buf[x], c.w, c.b, h->buf[y], nullptr, h->ones, H, W, c.cin_pad,
                             c.cout_pad, 9, 2, s));
      std::swap(x, y);
    }
  }
  RF_TRY(mid_block(h, h->e_mid, x, y, t1, t2, H, W, s));
  RF_TRY(prep(h, t1, H, W, 512, s));
  RF_TRY(group_norm(h, h->buf[x], h->buf[t1], H, W, h->e_norm_out, 1, 1, 1, s));
  RF_TRY(prep(h, y, H, W, 128, s));
  RF_TRY(conv(h, h->e_conv_out, h->buf[t1], h->buf[y], nullptr, H, W, s));  // 32 moments (of 128)
  return rf::sample_pack_launch(h->buf[y], 128, static_cast<const bf16*>(eps_bf16_chw),
                                static_cast<bf16*>(packed_out), H, W, scaling_factor, shift_factor, s);
}

}  // extern "C"
