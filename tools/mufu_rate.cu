// dev tool: MUFU.EX2 issue rate per SM sub-partition as a function of resident warps, and the
// softmax-like instruction mix (2 FFMA + 2 MUFU + 2 FADD + F2FP per 2 elements).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mufu_rate mufu_rate.cu && ./mufu_rate
#include <cstdio>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float ex2(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
template <int MODE>
__global__ void k(float* out, long long* cyc, int iters) {
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = -0.001f * (threadIdx.x + i);
  float2 acc = make_float2(0.f, 0.f);
  unsigned pk = 0;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    if (MODE == 0) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = ex2(v[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 16; i += 2) {
        float2 x = ffma2(make_float2(v[i], v[i + 1]), make_float2(0.999f, 0.999f), make_float2(-0.01f, -0.01f));
        float2 e; e.x = ex2(x.x); e.y = ex2(x.y);
        acc = fadd2(acc, e);
        __nv_bfloat162 b = __floats2bfloat162_rn(e.x, e.y);
        pk ^= *reinterpret_cast<unsigned*>(&b);
        v[i] = x.x; v[i + 1] = x.y;
      }
    }
  }
  long long t1 = clock64();
  float s = acc.x + acc.y + __uint_as_float(pk);
#pragma unroll
  for (int i = 0; i < 16; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
int main() {
  float* out; long long* cyc;
  cudaMalloc(&out, 132 * 1024 * 4); cudaMalloc(&cyc, 132 * 8);
  const int iters = 2000;
  for (int mode = 0; mode < 2; ++mode)
    for (int threads : {32, 128, 256, 512, 1024}) {
      for (int rep = 0; rep < 2; ++rep) {
        if (mode == 0) k<0><<<132, threads>>>(out, cyc, iters); else k<1><<<132, threads>>>(out, cyc, iters);
        cudaDeviceSynchronize();
      }
      long long h[132]; cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
      double c = (double)h[0];
      int warps_per_smsp = threads <= 128 ? 1 : threads / 128;
      printf("mode %d threads %4d: %.0f cycles, %.2f cycles per MUFU warp-instr per SMSP (%d warp(s)/SMSP)\n", mode, threads, c,
             c / (double(iters) * 16 * warps_per_smsp), warps_per_smsp);
    }
  return 0;
}
