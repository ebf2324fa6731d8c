// bb_generic.cu -- the "every config" SIMT kernel.
//
// Follows the operator semantics of the reference's TE definition literally
// (bitblas/ops/general_matmul/tirscript/matmul_dequantize_impl.py:391-478): decode one element, apply
// zeros/scale in A_dtype arithmetic, accumulate (fp32 stand-in for tensor-core accumulation, or exact
// int32), cast to out_dtype, add bias.  It is the fallback for shapes/formats the streaming and wgmma
// kernels do not cover (odd K, 1-bit, NF4/FP4/FP8 weights, group sizes < 128 ...) and the on-device
// cross-check for them.  One warp per output column n, up to MT rows of A per warp.
#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int MT = 4;          // rows of A per warp pass
constexpr int WARPS = 8;       // warps (= output columns) per block

// Wrow: row-major storage -> the row's first byte; BB_TILE_SLAB storage -> the first byte of the row's first 512-byte segment
// (segments of one row are then 32 x 512 bytes apart)
__device__ __forceinline__ uint32_t load_field(const uint8_t* __restrict__ Wrow, int k, int bits, int layout, int tiled) {
  auto at = [&](size_t b) -> size_t {
    return tiled ? (b / BB_TILE_ROW_BYTES) * (size_t(BB_TILE_ROWS) * BB_TILE_ROW_BYTES) + b % BB_TILE_ROW_BYTES : b;
  };
  if (bits == 8) return Wrow[at(size_t(k))];
  const int epw = 32 / bits;
  const uint32_t word = *reinterpret_cast<const uint32_t*>(Wrow + at(size_t(k / epw) * 4));
  const int pos = field_bitpos(k % epw, bits, layout);
  return (word >> pos) & ((1u << bits) - 1u);
}

template <typename T>
__device__ __forceinline__ T cvt_int(int v);
template <>
__device__ __forceinline__ __half cvt_int<__half>(int v) { return __int2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 cvt_int<__nv_bfloat16>(int v) { return __int2bfloat16_rn(v); }

template <typename T>
__device__ __forceinline__ T from_f16_bits(uint16_t b) {
  __half h = *reinterpret_cast<__half*>(&b);
  if constexpr (sizeof(T) == 2 && std::is_same<T, __half>::value) return h;
  else return TypeTraits<T>::from_float(__half2float(h));
}

// float-typed A (half / bf16)
template <typename T>
__device__ __forceinline__ T decode_value(uint32_t u, int fmt, int bits, const T* __restrict__ lut) {
  switch (fmt) {
    case BB_W_UINT: return cvt_int<T>(int(u));
    case BB_W_INT:
      if (bits == 1) return cvt_int<T>(2 * int(u) - 1);
      if (bits == 8) return cvt_int<T>(int(int8_t(u)));
      return cvt_int<T>(int(u) - (1 << (bits - 1)));
    case BB_W_NF: return lut[u];
    case BB_W_FP4: {
      uint32_t s = u >> 3, e = u & 7;
      uint16_t b = uint16_t(((e | 8) | (s << 5)) << 10);
      return e == 0 ? cvt_int<T>(0) : from_f16_bits<T>(b);
    }
    case BB_W_FP8_E4M3: {
      uint32_t v = u & 0xff;
      uint32_t s = (v >> 7) << 15, e4 = v & 0x40;
      uint32_t e16 = (((v & 63) << 7) | (e4 << 8) | (e4 << 7)) ^ 0x2000;
      return from_f16_bits<T>(uint16_t(s | e16));
    }
    case BB_W_FP8_E5M2: return from_f16_bits<T>(uint16_t((u & 0xff) << 8));
  }
  return cvt_int<T>(0);
}

template <typename T>
__device__ __forceinline__ T t_sub(T a, T b) { return __hsub(a, b); }
template <typename T>
__device__ __forceinline__ T t_mul(T a, T b) { return __hmul(a, b); }
template <typename T>
__device__ __forceinline__ T t_fma(T a, T b, T c) { return __hfma(a, b, c); }

template <typename TO>
__device__ __forceinline__ void store_out(void* C, size_t idx, float acc, const void* bias, int n, int a_dtype);

template <typename TA>
__device__ __forceinline__ float bias_as_float(const void* bias, int n) {
  return TypeTraits<TA>::to_float(reinterpret_cast<const TA*>(bias)[n]);
}

// out = cast(acc) (+ bias, added in out_dtype arithmetic)   -- impl.py:462-477
template <typename TA>
__device__ __forceinline__ void store_float_out(void* C, int out_dtype, size_t idx, float acc, const void* bias, int n) {
  switch (out_dtype) {
    case BB_F16: {
      __half v = __float2half_rn(acc);
      if (bias) v = __hadd(v, __float2half_rn(bias_as_float<TA>(bias, n)));
      reinterpret_cast<__half*>(C)[idx] = v;
      break;
    }
    case BB_BF16: {
      __nv_bfloat16 v = __float2bfloat16_rn(acc);
      if (bias) v = __hadd(v, __float2bfloat16_rn(bias_as_float<TA>(bias, n)));
      reinterpret_cast<__nv_bfloat16*>(C)[idx] = v;
      break;
    }
    default: {
      float v = acc;
      if (bias) v += bias_as_float<TA>(bias, n);
      reinterpret_cast<float*>(C)[idx] = v;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(WARPS * 32)
generic_float_kernel(const bb_matmul_desc d, const T* __restrict__ A, const uint8_t* __restrict__ W,
                     const T* __restrict__ lut, const T* __restrict__ scale, const void* __restrict__ zeros,
                     const void* __restrict__ bias, void* __restrict__ C, int M) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * WARPS + warp;
  const int m0 = blockIdx.y * MT;
  if (n >= d.N) return;
  const int K = d.K, bits = d.w_bits;
  const int g = d.group_size <= 0 ? K : d.group_size;
  const int G = K / g;
  const size_t row_bytes = size_t(K) * bits / 8;
  const int tiled = d.w_tile == BB_TILE_SLAB;
  const uint8_t* Wrow = W + (tiled ? tiled_byte_offset(n, 0, (long long)row_bytes) : size_t(n) * row_bytes);
  const bool use_fma = d.w_layout != BB_LAYOUT_COMPRESSED && (d.w_fmt == BB_W_UINT || d.w_fmt == BB_W_INT) &&
                       std::is_same<T, __half>::value;
  float acc[MT];
#pragma unroll
  for (int i = 0; i < MT; ++i) acc[i] = 0.f;

  for (int k = lane; k < K; k += 32) {
    const uint32_t u = load_field(Wrow, k, bits, d.w_layout, tiled);
    const int gi = k / g;
    T w;
    if (d.with_zeros && d.zeros_mode == BB_ZEROS_QUANTIZED) {
      const uint8_t* qz = reinterpret_cast<const uint8_t*>(zeros);
      const int epb = 8 / bits;
      const uint32_t z = (qz[size_t(gi) * (size_t(d.N) * bits / 8) + n / epb] >> (bits * (n % epb))) & ((1u << bits) - 1u);
      w = cvt_int<T>(int(u) - int(z));
    } else {
      w = decode_value<T>(u, d.w_fmt, bits, lut);
    }
    if (d.with_scaling) {
      const T s = scale[size_t(n) * G + gi];
      if (!d.with_zeros || d.zeros_mode == BB_ZEROS_QUANTIZED) {
        w = t_mul(w, s);
      } else {
        const T z = reinterpret_cast<const T*>(zeros)[size_t(n) * G + gi];
        if (d.zeros_mode == BB_ZEROS_ORIGINAL) w = t_mul(t_sub(w, z), s);
        else if (use_fma) w = t_fma(w, s, __hneg(z));
        else w = t_sub(t_mul(w, s), z);
      }
    }
    const float wf = TypeTraits<T>::to_float(w);
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      if (m0 + i < M) acc[i] = fmaf(TypeTraits<T>::to_float(A[size_t(m0 + i) * K + k]), wf, acc[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < MT; ++i) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < MT; ++i)
      if (m0 + i < M) store_float_out<T>(C, d.out_dtype, size_t(m0 + i) * d.N + n, acc[i], d.with_bias ? bias : nullptr, n);
  }
}

// int8 activations, exact int32 accumulate
__global__ void __launch_bounds__(WARPS * 32)
generic_int_kernel(const bb_matmul_desc d, const int8_t* __restrict__ A, const uint8_t* __restrict__ W,
                   const int8_t* __restrict__ scale, const void* __restrict__ zeros,
                   const int8_t* __restrict__ bias, void* __restrict__ C, int M) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * WARPS + warp;
  const int m0 = blockIdx.y * MT;
  if (n >= d.N) return;
  const int K = d.K, bits = d.w_bits;
  const int g = d.group_size <= 0 ? K : d.group_size;
  const int G = K / g;
  const int tiled = d.w_tile == BB_TILE_SLAB;
  const uint8_t* Wrow = W + (tiled ? tiled_byte_offset(n, 0, (long long)K * bits / 8) : size_t(n) * (size_t(K) * bits / 8));
  int acc[MT];
#pragma unroll
  for (int i = 0; i < MT; ++i) acc[i] = 0;
  for (int k = lane; k < K; k += 32) {
    const uint32_t u = load_field(Wrow, k, bits, d.w_layout, tiled);
    const int gi = k / g;
    int w;
    if (d.with_zeros && d.zeros_mode == BB_ZEROS_QUANTIZED) {
      const uint8_t* qz = reinterpret_cast<const uint8_t*>(zeros);
      const int epb = 8 / bits;
      const uint32_t z = (qz[size_t(gi) * (size_t(d.N) * bits / 8) + n / epb] >> (bits * (n % epb))) & ((1u << bits) - 1u);
      w = int(u) - int(z);
    } else if (d.w_fmt == BB_W_INT) {
      w = bits == 1 ? 2 * int(u) - 1 : (bits == 8 ? int(int8_t(u)) : int(u) - (1 << (bits - 1)));
    } else {
      w = int(u);
    }
    if (d.with_scaling) {  // int8 arithmetic per the TE definition (values wrap to int8)
      const int s = scale[size_t(n) * G + gi];
      if (!d.with_zeros || d.zeros_mode == BB_ZEROS_QUANTIZED) w = int(int8_t(w * s));
      else {
        const int z = reinterpret_cast<const int8_t*>(zeros)[size_t(n) * G + gi];
        w = d.zeros_mode == BB_ZEROS_ORIGINAL ? int(int8_t(int(int8_t(w - z)) * s)) : int(int8_t(int(int8_t(w * s)) - z));
      }
    }
#pragma unroll
    for (int i = 0; i < MT; ++i)
      if (m0 + i < M) acc[i] += int(A[size_t(m0 + i) * K + k]) * w;
  }
#pragma unroll
  for (int i = 0; i < MT; ++i) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      if (m0 + i >= M) continue;
      const size_t idx = size_t(m0 + i) * d.N + n;
      const int b = d.with_bias ? int(bias[n]) : 0;
      switch (d.out_dtype) {
        case BB_I32: reinterpret_cast<int*>(C)[idx] = acc[i] + b; break;
        case BB_I8: reinterpret_cast<int8_t*>(C)[idx] = int8_t(int8_t(acc[i]) + b); break;
        case BB_F32: reinterpret_cast<float*>(C)[idx] = float(acc[i]) + float(b); break;
        case BB_F16: reinterpret_cast<__half*>(C)[idx] = __hadd(__int2half_rn(acc[i]), __int2half_rn(b)); break;
        default: reinterpret_cast<__nv_bfloat16*>(C)[idx] = __hadd(__int2bfloat16_rn(acc[i]), __int2bfloat16_rn(b));
      }
    }
  }
}

}  // namespace

bool generic_supported(const bb_matmul_desc& d) {
  if (d.w_bits != 1 && d.w_bits != 2 && d.w_bits != 4 && d.w_bits != 8) return false;
  if (d.w_bits < 8 && (d.K * d.w_bits) % 32 != 0) return false;  // whole 32-bit words per row
  if (d.a_dtype == BB_I8) return d.w_fmt == BB_W_UINT || d.w_fmt == BB_W_INT;
  return d.a_dtype == BB_F16 || d.a_dtype == BB_BF16;
}

int launch_generic(const MatmulArgs& a) {
  const bb_matmul_desc& d = a.d;
  dim3 grid((d.N + WARPS - 1) / WARPS, (a.m + MT - 1) / MT);
  dim3 block(WARPS * 32);
  if (d.a_dtype == BB_F16) {
    generic_float_kernel<__half><<<grid, block, 0, a.stream>>>(
        d, (const __half*)a.A, (const uint8_t*)a.W, (const __half*)a.lut, (const __half*)a.scale, a.zeros, a.bias, a.C, a.m);
  } else if (d.a_dtype == BB_BF16) {
    generic_float_kernel<__nv_bfloat16><<<grid, block, 0, a.stream>>>(
        d, (const __nv_bfloat16*)a.A, (const uint8_t*)a.W, (const __nv_bfloat16*)a.lut, (const __nv_bfloat16*)a.scale,
        a.zeros, a.bias, a.C, a.m);
  } else {
    generic_int_kernel<<<grid, block, 0, a.stream>>>(d, (const int8_t*)a.A, (const uint8_t*)a.W, (const int8_t*)a.scale,
                                                      a.zeros, (const int8_t*)a.bias, a.C, a.m);
  }
  BB_LAUNCH_CHECK();
  return 0;
}

}  // namespace bb
