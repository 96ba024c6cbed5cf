/* c_abi_linear.c — the drop-in boundary from plain C: no Python, no torch, only librf_b200.so and
 * the CUDA runtime.  One nn.Linear (+ GELU) through rf_op_linear on device buffers, checked against
 * a scalar host loop with the reference's rounding points (bf16 after the bias add, bf16 output).
 *
 *   gcc -std=c11 -O2 -Iinclude -I/usr/local/cuda/include examples/c_abi_linear.c \
 *       -Lreflectionflow_b200 -lrf_b200 -L/usr/local/cuda/lib64 -lcudart -lm \
 *       -Wl,-rpath,$PWD/reflectionflow_b200 -o examples/c_abi_linear
 *   ./examples/c_abi_linear            (needs an H100; exits 2 with the library's message otherwise)
 */
#include <cuda_runtime_api.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "rf_b200.h"

static uint16_t f2bf(float f) { /* round to nearest even */
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static float lcg(uint32_t* s) { /* uniform in [-1, 1) */
  *s = *s * 1664525u + 1013904223u;
  return (float)((*s >> 8) & 0xFFFF) / 32768.0f - 1.0f;
}
static float gelu_tanh(float x) {
  return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

int main(void) {
  enum { M = 384, N = 256, K = 192 };
  if (rf_abi_version() != RF_B200_ABI_VERSION) {
    fprintf(stderr, "ABI mismatch\n");
    return 1;
  }
  uint16_t *x = malloc(2 * M * K), *w = malloc(2 * N * K), *b = malloc(2 * N), *y = malloc(2 * M * N);
  uint32_t seed = 12345u;
  for (int i = 0; i < M * K; ++i) x[i] = f2bf(lcg(&seed));
  for (int i = 0; i < N * K; ++i) w[i] = f2bf(lcg(&seed) * 0.1f);
  for (int i = 0; i < N; ++i) b[i] = f2bf(lcg(&seed));
  void *dx, *dw, *db, *dy;
  if (cudaMalloc(&dx, 2 * M * K) != cudaSuccess || cudaMalloc(&dw, 2 * N * K) != cudaSuccess ||
      cudaMalloc(&db, 2 * N) != cudaSuccess || cudaMalloc(&dy, 2 * M * N) != cudaSuccess) {
    fprintf(stderr, "no CUDA device: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 2;
  }
  cudaMemcpy(dx, x, 2 * M * K, cudaMemcpyHostToDevice);
  cudaMemcpy(dw, w, 2 * N * K, cudaMemcpyHostToDevice);
  cudaMemcpy(db, b, 2 * N, cudaMemcpyHostToDevice);
  for (int epi = RF_EPI_BIAS; epi <= RF_EPI_GELU; ++epi) {
    int rc = rf_op_linear(epi, M, N, K, dx, K, dw, db, dy, N, NULL, 0, NULL, 0, NULL, NULL, NULL, NULL, NULL,
                          NULL);
    if (rc != 0) {
      fprintf(stderr, "rf_op_linear failed (%d): %s\n", rc, rf_last_error());
      return 2;
    }
    if (cudaDeviceSynchronize() != cudaSuccess) {
      fprintf(stderr, "kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
      return 2;
    }
    cudaMemcpy(y, dy, 2 * M * N, cudaMemcpyDeviceToHost);
    int bad = 0, off1 = 0;
    for (int i = 0; i < M; ++i)
      for (int j = 0; j < N; ++j) {
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc += bf2f(x[i * K + k]) * bf2f(w[j * K + k]);
        float v = bf2f(f2bf(acc + bf2f(b[j])));
        if (epi == RF_EPI_GELU) v = gelu_tanh(v);
        const uint16_t want = f2bf(v), got = y[i * N + j];
        if (want != got) { /* summation order differs from the tensor core's: allow one bf16 ulp
                              (plus an absolute 1e-3 where bias and product cancel) */
          const float fw = bf2f(want), fg = bf2f(got);
          const float tol = fmaxf(fabsf(fw), fabsf(fg)) * (1.0f / 128.0f) + 1e-3f;
          if (fabsf(fw - fg) <= tol) ++off1; else ++bad;
        }
      }
    printf("epilogue %d: %d x %d outputs, %d within one bf16 ulp, %d wrong\n", epi, M, N, off1, bad);
    if (bad != 0 || off1 > M * N / 50) return 3;
  }
  printf("c_abi_linear: OK\n");
  return 0;
}
