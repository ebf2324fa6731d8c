// tools/gemv_bench.cu -- m = 1 W4A16 GEMV through the C ABI (bb_matmul): full-output check against a double-precision CPU
// dequantise+dot, then back-to-back timing over rotating weight copies (cold L2), for a list of shapes.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/gemv_bench tools/gemv_bench.cu \
//        -Lbitblas_b200/lib -lbitblas_b200 -Xlinker -rpath -Xlinker '$ORIGIN/../bitblas_b200/lib'
//   tools/gemv_bench [--kernel ID] [--iters N] [--tile] [--nocheck] NxK [NxK ...]
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../include/bitblas_b200.h"

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
#define BB(x) do { int rc = (x); if (rc) { printf("bb error %d at line %d: %s\n", rc, __LINE__, bb_last_error()); exit(1);} } while (0)

int main(int argc, char** argv) {
  int kernel = BB_KERNEL_AUTO, iters = 200;
  bool check = true, tile = false;   // --tile: BB_TILE_SLAB weight storage (MatmulConfig.propagate_b)
  std::vector<std::pair<int, int>> shapes;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    if (a == "--kernel") kernel = atoi(argv[++i]);
    else if (a == "--iters") iters = atoi(argv[++i]);
    else if (a == "--nocheck") check = false;
    else if (a == "--tile") tile = true;
    else { int n, k; if (sscanf(a.c_str(), "%dx%d", &n, &k) == 2) shapes.push_back({n, k}); }
  }
  if (shapes.empty()) shapes.push_back({12288, 12288});
  BB(bb_init(0));
  bb_set_kernel_override(kernel);
  cudaStream_t st; CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int g = 128;
  for (auto [N, K] : shapes) {
    const int G = K / g;
    const size_t wbytes = size_t(N) * K / 2;
    const int copies = std::max(2, int((400ull << 20) / wbytes) + 1);   // > 50 MB of L2 between reuses
    bb_matmul_desc d; memset(&d, 0, sizeof(d));
    d.N = N; d.K = K; d.a_dtype = BB_F16; d.w_fmt = BB_W_UINT; d.w_bits = 4; d.accum_dtype = BB_F32; d.out_dtype = BB_F16;
    d.group_size = g; d.with_scaling = 1; d.with_zeros = 1; d.zeros_mode = BB_ZEROS_QUANTIZED; d.with_bias = 0;
    d.w_layout = BB_LAYOUT_INTERLEAVED_16;
    d.w_tile = tile ? BB_TILE_SLAB : BB_TILE_ROW_MAJOR;
    std::mt19937 rng(1234);
    std::vector<uint32_t> hW(wbytes / 4);
    for (auto& v : hW) v = rng();
    std::vector<__half> hS(size_t(N) * G), hA(K);
    std::vector<uint8_t> hZ(size_t(G) * N / 2);
    std::uniform_real_distribution<float> us(0.01f, 0.135f), ua(-0.5f, 0.5f);
    for (auto& v : hS) v = __float2half(us(rng));
    for (auto& v : hA) v = __float2half(ua(rng));
    for (auto& v : hZ) v = uint8_t(rng());
    std::vector<uint8_t*> dW(copies);
    for (int c = 0; c < copies; ++c) {
      CK(cudaMalloc(&dW[c], wbytes));
      if (tile) {   // upload row-major, re-tile on the device with the library's own kernel
        uint8_t* tmp; CK(cudaMalloc(&tmp, wbytes)); CK(cudaMemcpy(tmp, hW.data(), wbytes, cudaMemcpyHostToDevice));
        BB(bb_retile_weight_device(reinterpret_cast<const int8_t*>(tmp), reinterpret_cast<int8_t*>(dW[c]), N, K / 2, 0, nullptr));
        CK(cudaDeviceSynchronize()); CK(cudaFree(tmp));
      } else {
        CK(cudaMemcpy(dW[c], hW.data(), wbytes, cudaMemcpyHostToDevice));
      }
    }
    __half *dS, *dA, *dC; uint8_t* dZ; void* ws;
    CK(cudaMalloc(&dS, hS.size() * 2)); CK(cudaMemcpy(dS, hS.data(), hS.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&dA, K * 2)); CK(cudaMemcpy(dA, hA.data(), K * 2, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&dZ, hZ.size())); CK(cudaMemcpy(dZ, hZ.data(), hZ.size(), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&dC, N * 2));
    const size_t wsb = std::max<size_t>(bb_workspace_bytes(&d, 1), 256);
    CK(cudaMalloc(&ws, wsb)); CK(cudaMemset(ws, 0, wsb));
    const int kid = bb_select_kernel(&d, 1);
    const double alg = double(wbytes) + double(N) * G * 2 + double(G) * N / 2 + K * 2.0 + N * 2.0;
    // CPU reference (interleaved-16 layout: element o of a 32-bit word sits at bit (o%2)*16 + (o/2)*4)
    std::vector<double> ref;
    if (check) {
      ref.assign(N, 0.0);
      std::vector<float> fa(K);
      for (int k = 0; k < K; ++k) fa[k] = __half2float(hA[k]);
      for (int n = 0; n < N; ++n) {
        double acc = 0;
        const uint32_t* row = hW.data() + size_t(n) * (K / 8);
        for (int gi = 0; gi < G; ++gi) {
          const float s = __half2float(hS[size_t(n) * G + gi]);
          const int z = (hZ[size_t(gi) * (N / 2) + n / 2] >> (4 * (n & 1))) & 15;
          double gs = 0;
          for (int wi = gi * (g / 8); wi < (gi + 1) * (g / 8); ++wi) {
            const uint32_t w = row[wi];
            for (int o = 0; o < 8; ++o) {
              const int u = (w >> ((o % 2) * 16 + (o / 2) * 4)) & 15;
              gs += double(u - z) * fa[wi * 8 + o];
            }
          }
          acc += gs * s;
        }
        ref[n] = acc;
      }
    }
    double maxerr = -1, maxref = 0;
    if (check) {
      CK(cudaMemset(dC, 0xff, N * 2));
      BB(bb_matmul(&d, dA, dW[0], nullptr, dS, dZ, nullptr, dC, 1, ws, wsb, st));
      CK(cudaStreamSynchronize(st));
      std::vector<__half> hC(N);
      CK(cudaMemcpy(hC.data(), dC, N * 2, cudaMemcpyDeviceToHost));
      maxerr = 0;
      int bad = -1;
      for (int n = 0; n < N; ++n) {
        const double e = fabs(double(__half2float(hC[n])) - ref[n]);
        if (!(e <= maxerr)) { maxerr = e; bad = n; }
        maxref = std::max(maxref, fabs(ref[n]));
      }
      if (!(maxerr <= 0.02 * maxref)) printf("  MISMATCH at n=%d: got %f ref %f\n", bad, __half2float(hC[bad]), ref[bad]);
    }
    for (int i = 0; i < 10; ++i) BB(bb_matmul(&d, dA, dW[i % copies], nullptr, dS, dZ, nullptr, dC, 1, ws, wsb, st));
    CK(cudaStreamSynchronize(st));
    float best = 1e30f, sum = 0;
    const int reps = 3;
    for (int r = 0; r < reps; ++r) {
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < iters; ++i) BB(bb_matmul(&d, dA, dW[i % copies], nullptr, dS, dZ, nullptr, dC, 1, ws, wsb, st));
      CK(cudaEventRecord(e1, st));
      CK(cudaEventSynchronize(e1));
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      best = std::min(best, ms / iters); sum += ms / iters;
    }
    const double us_best = best * 1e3, us_mean = sum / reps * 1e3;
    printf("N=%d K=%d kernel=%s%s : %.2f us best %.2f us mean  %.0f GB/s  frac(6576)=%.3f  maxerr=%.3g (max|ref|=%.3g)\n",
           N, K, bb_kernel_name(kid), tile ? " (slab-tiled W)" : "", us_best, us_mean, alg / (us_mean * 1e-6) / 1e9,
           alg / (us_mean * 1e-6) / 1e9 / 6576.1, maxerr, maxref);
    fflush(stdout);
    for (auto p : dW) cudaFree(p);
    cudaFree(dS); cudaFree(dA); cudaFree(dZ); cudaFree(dC); cudaFree(ws);
  }
  return 0;
}
