// crepe_tc.h -- 3xTF32 tensor-core convolution of the CREPE layers (crepe_tc.cu).
#pragma once
#include <stddef.h>

#include "common.cuh"

namespace ryk {

// y[m][n] = ReLU(bias[n] + sum_k A[m][k] * w[k][n]) with A[m][k] = x[(m / W) * fstride + (m % W) * wstep + k]; row-major y [M][N].
struct CrepeGemm {
  const float* x = nullptr; int M = 0, W = 1; long long fstride = 0; int wstep = 0;
  int K = 0, N = 0;
  const float* w = nullptr; const float* bias = nullptr; float* y = nullptr;
};

size_t crepe_tc_ws_floats(int M, int K, int N);                       // split-K workspace the layer needs (0: none)
int crepe_tc_run(const CrepeGemm& g, float* ws, cudaStream_t st);

}  // namespace ryk
