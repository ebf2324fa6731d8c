// bb_quant.cu -- per-token int8 quantization of 16-bit activations (bb_quantize_act_int8), BitNet b1.58's activation_quant:
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

}  // namespace

int launch_quantize_act_int8(const void* x, int a_dtype, int rows, int K, int8_t* q, float* scale, cudaStream_t stream) {
  // one thread per 16-byte vector up to the block size, in whole warps
  const int threads = std::min(QUANT_MAX_THREADS, (K / 8 + 31) / 32 * 32);
  auto kernel = a_dtype == BB_F16 ? quantize_act_int8_kernel<__half> : quantize_act_int8_kernel<__nv_bfloat16>;
  return launch_pdl(kernel, unsigned(rows), threads, 0, stream, pdl_enabled(), reinterpret_cast<const uint16_t*>(x), K, q, scale);
}

}  // namespace bb
