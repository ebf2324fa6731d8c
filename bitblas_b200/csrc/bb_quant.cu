// bb_quant.cu -- quantization of 16-bit activations on the device.  bb_quantize_act_fp8 (below): e4m3 per (token, 128-column
// block).  bb_quantize_act_int8: per-token int8, BitNet b1.58's activation_quant:
//     amax = max_k |x[r, k]|,   s[r] = 127 * (1 / max(amax, 1e-5)),   q[r, k] = clamp(rint(x[r, k] * s[r]), -128, 127)
// in fp32, each operation correctly rounded (the int8 matmuls' bb_matmul_scaled then divides by s[r]).  The scale is a reciprocal
// and a product, not one division: that is what torch evaluates for BitNet's `127.0 / t` (Tensor.__rtruediv__ is
// reciprocal() * 127), and one correctly rounded division differs from it in the last bit for about a quarter of the rows.
//
// Schedule: one CTA per row.  Each thread takes 16-byte vectors of 8 values, strided by the block, twice: the first pass reduces
// |x| to the row maximum (warp shuffles, then one value per warp in shared memory), the second reads the same vectors again --
// from L1 / L2, the row was just read -- and stores 8 int8 values as one 8-byte vector.  HBM sees the row read once and q written
// once: rows * K * 3 + 4 * rows bytes.
// PDL: griddepcontrol.wait before the first read of x (the preceding kernel's output); launch_dependents after the last store, as
// bb_permute_cols does (an early trigger made the kernels after the column gather slower, DESIGN.md §3.2.2).
#include <algorithm>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int QUANT_MAX_THREADS = 256;

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = raw_to_float<T>(uint16_t(w[i] & 0xffffu));
    f[2 * i + 1] = raw_to_float<T>(uint16_t(w[i] >> 16));
  }
}

__device__ __forceinline__ uint32_t quant4(const float* f, float s) {
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int v = min(max(__float2int_rn(__fmul_rn(f[i], s)), -128), 127);   // round half to even; NaN converts to 0
    r |= uint32_t(v & 0xff) << (8 * i);
  }
  return r;
}

template <typename T>
__global__ void __launch_bounds__(QUANT_MAX_THREADS)
quantize_act_int8_kernel(const uint16_t* __restrict__ x, int K, int8_t* __restrict__ q, float* __restrict__ scale) {
  __shared__ float warp_max[QUANT_MAX_THREADS / 32];
  const int r = blockIdx.x, vecs = K / 8;
  const uint4* row = reinterpret_cast<const uint4*>(x + size_t(r) * K);
  pdl_wait();
  float amax = 0.f;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    float f[8];
    unpack8<T>(row[v], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) warp_max[warp] = amax;
  __syncthreads();
  amax = warp_max[0];
  for (int w = 1; w < nwarps; ++w) amax = fmaxf(amax, warp_max[w]);
  const float s = __fmul_rn(__frcp_rn(fmaxf(amax, 1e-5f)), 127.f);
  uint2* qrow = reinterpret_cast<uint2*>(q + size_t(r) * K);
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    float f[8];
    unpack8<T>(row[v], f);
    qrow[v] = make_uint2(quant4(f, s), quant4(f + 4, s));
  }
  if (threadIdx.x == 0) scale[r] = s;
  pdl_launch_dependents();
}

// ---- bb_quantize_act_fp8: per (row, 128-column block) e4m3 quantization, vLLM's per_token_group_quant_fp8 with IEEE division:
//     amax = max(max_{k in block} |x[r, k]|, 1e-10),   s[r, b] = amax / 448,   q[r, k] = e4m3_rn(clamp(x[r, k] / s[r, b], +-448))
// Schedule: one half-warp per block, 16 lanes x one 16-byte vector of 8 values; the amax is four shuffles inside the half-warp,
// and each lane stores its 8 e4m3 bytes as one 8-byte vector.  Consecutive half-warps take consecutive blocks of a row, so a
// warp reads 512 contiguous bytes.  The scale goes to scale[b * scale_ld + r] (k-block-major, the GEMM's layout).
constexpr int QUANT_FP8_THREADS = 256;
constexpr float E4M3_MAX = 448.f;

// two floats -> two e4m3 bytes (lo first), round to nearest even, saturating
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

template <typename T>
__global__ void __launch_bounds__(QUANT_FP8_THREADS)
quantize_act_fp8_kernel(const uint16_t* __restrict__ x, int rows, int K, uint8_t* __restrict__ q, float* __restrict__ scale,
                        int scale_ld) {
  const int nkb = K / 128;
  const long long blk = (long long)blockIdx.x * (QUANT_FP8_THREADS / 16) + (threadIdx.x >> 4);
  const int l = threadIdx.x & 15;
  pdl_wait();
  if (blk < (long long)rows * nkb) {   // (whole half-warps leave together: the shuffles below stay inside live ones)
    const int r = int(blk / nkb), b = int(blk - (long long)r * nkb);
    const size_t e0 = size_t(r) * K + size_t(b) * 128 + size_t(l) * 8;
    float f[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(x + e0), f);
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
    const unsigned hmask = 0xffffu << (threadIdx.x & 16);
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(hmask, amax, off));
    const float s = __fdiv_rn(fmaxf(amax, 1e-10f), E4M3_MAX);
    uint32_t w[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = fminf(fmaxf(__fdiv_rn(f[4 * h + i], s), -E4M3_MAX), E4M3_MAX);
      w[h] = e4m3x2(v[0], v[1]) | (e4m3x2(v[2], v[3]) << 16);
    }
    *reinterpret_cast<uint2*>(q + e0) = make_uint2(w[0], w[1]);
    if (l == 0) scale[size_t(b) * scale_ld + r] = s;
  }
  pdl_launch_dependents();
}

}  // namespace

int launch_quantize_act_fp8(const void* x, int a_dtype, int rows, int K, uint8_t* q, float* scale, int scale_ld, cudaStream_t stream) {
  const long long blocks = (long long)rows * (K / 128);
  const unsigned grid = unsigned((blocks + QUANT_FP8_THREADS / 16 - 1) / (QUANT_FP8_THREADS / 16));
  auto kernel = a_dtype == BB_F16 ? quantize_act_fp8_kernel<__half> : quantize_act_fp8_kernel<__nv_bfloat16>;
  return launch_pdl(kernel, grid, QUANT_FP8_THREADS, 0, stream, pdl_enabled(), reinterpret_cast<const uint16_t*>(x), rows, K, q,
                    scale, scale_ld);
}

int launch_quantize_act_int8(const void* x, int a_dtype, int rows, int K, int8_t* q, float* scale, cudaStream_t stream) {
  // one thread per 16-byte vector up to the block size, in whole warps
  const int threads = std::min(QUANT_MAX_THREADS, (K / 8 + 31) / 32 * 32);
  auto kernel = a_dtype == BB_F16 ? quantize_act_int8_kernel<__half> : quantize_act_int8_kernel<__nv_bfloat16>;
  return launch_pdl(kernel, unsigned(rows), threads, 0, stream, pdl_enabled(), reinterpret_cast<const uint16_t*>(x), K, q, scale);
}

}  // namespace bb
