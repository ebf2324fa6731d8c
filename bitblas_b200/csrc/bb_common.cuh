// bb_common.cuh -- shared host/device helpers for the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/bitblas_b200.h"

namespace bb {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define BB_CHECK_CUDA(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      bb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 2;                                                                              \
    }                                                                                        \
  } while (0)

#define BB_LAUNCH_CHECK()                                                                    \
  do {                                                                                       \
    bb::g_launches.fetch_add(1, std::memory_order_relaxed);                                  \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) {                                                                 \
      bb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 3;                                                                              \
    }                                                                                        \
  } while (0)

struct MatmulArgs {
  bb_matmul_desc d;
  const void* A;
  const void* W;
  const void* lut;
  const void* scale;
  const void* zeros;
  const void* bias;
  void* C;
  int m;
  // column-parallel scatter epilogue (n_peers == 0: plain single output C with row stride N)
  void* peer_C[BB_MAX_PEERS];
  int n_peers;
  long long ldc;         // row stride of the output(s) in elements
  long long col_offset;  // first output column of this shard
  void* workspace;
  size_t workspace_bytes;
  cudaStream_t stream;
  int groups() const { return d.K / (d.group_size <= 0 ? d.K : d.group_size); }
  int gsize() const { return d.group_size <= 0 ? d.K : d.group_size; }
};

constexpr int BB_MAX_DEVICES = 64;
int current_device();     // ordinal of the calling thread's current CUDA device, clamped to [0, BB_MAX_DEVICES)
int device_sm_count();    // SM count of the current device (cached per device)

// kernel family entry points (each returns 0 / error code; *_supported says whether the family covers it)
bool generic_supported(const bb_matmul_desc& d);
int launch_generic(const MatmulArgs& a);
bool gemv_mma_supported(const bb_matmul_desc& d, int m);
int launch_gemv_mma(const MatmulArgs& a);
bool gemv_streamk_supported(const bb_matmul_desc& d, int m);
int launch_gemv_streamk(const MatmulArgs& a);
size_t gemv_streamk_workspace_bytes();  // partial slots + flags
bool gemv_slab_supported(const bb_matmul_desc& d, int m);
int launch_gemv_slab(const MatmulArgs& a);
size_t gemv_slab_workspace_bytes();     // tagged partial slots (must be zero-initialised once by the caller)
bool gemv_i8_supported(const bb_matmul_desc& d, int m);
int launch_gemv_i8(const MatmulArgs& a);
bool gemm_ts_supported(const bb_matmul_desc& d, int m);
int launch_gemm_ts(const MatmulArgs& a);
size_t gemm_ts_workspace_bytes(const bb_matmul_desc& d, int m);
int gemm_ts_init(int device);

// bit position of logical element `o` (0 .. 32/bits-1) inside its 32-bit storage word, for each weight
// layout (restates bitblas/quantization/utils.py:73-110 + testing/cpp/lop3_type_conversion/fast_decoding.hpp:30-95,607-668)
__host__ __device__ __forceinline__ int field_bitpos(int o, int bits, int layout) {
  if (layout == BB_LAYOUT_COMPRESSED) return o * bits;
  const int S = (layout == BB_LAYOUT_INTERLEAVED_8) ? 8 : 16;
  const int G = 32 / S;
  int pos = (o % G) * S + (o / G) * bits;
  if (bits == 2 && S == 16) {
    const int byte = pos >> 3;
    if (byte == 1) pos += 8; else if (byte == 2) pos -= 8;
  } else if (bits == 1 && S == 16) {
    const int map[8] = {0, 2, 4, 6, 1, 3, 5, 7};
    pos = map[pos >> 2] * 4 + (pos & 3);
  } else if (bits == 1 && S == 8) {
    const int map[8] = {0, 4, 2, 6, 1, 5, 3, 7};
    pos = map[pos >> 2] * 4 + (pos & 3);
  }
  return pos;
}

// BB_TILE_SLAB storage: byte `b` of packed row `n` (row_bytes per row) lives at this offset
__host__ __device__ __forceinline__ size_t tiled_byte_offset(long long n, long long b, long long row_bytes) {
  const long long upr = row_bytes / BB_TILE_ROW_BYTES;
  return size_t((((n / BB_TILE_ROWS) * upr + b / BB_TILE_ROW_BYTES) * BB_TILE_ROWS + n % BB_TILE_ROWS) * BB_TILE_ROW_BYTES +
                b % BB_TILE_ROW_BYTES);
}
inline bool tile_shape_ok(const bb_matmul_desc& d) {
  return d.N % BB_TILE_ROWS == 0 && ((long long)d.K * d.w_bits / 8) % BB_TILE_ROW_BYTES == 0 && ((long long)d.K * d.w_bits) % 8 == 0;
}

// where a kernel epilogue stores C[m, n]: one local buffer, or the same element in every peer's buffer
struct OutSpec {
  void* ptr[BB_MAX_PEERS];
  int n;                 // number of destination buffers (>= 1)
  long long ld;          // row stride in elements
  long long col0;        // column offset of this shard
};
inline OutSpec make_outspec(const MatmulArgs& a) {
  OutSpec o;
  if (a.n_peers > 0) {
    o.n = a.n_peers;
    for (int i = 0; i < BB_MAX_PEERS; ++i) o.ptr[i] = i < a.n_peers ? a.peer_C[i] : nullptr;
    o.ld = a.ldc; o.col0 = a.col_offset;
  } else {
    o.n = 1;
    for (int i = 0; i < BB_MAX_PEERS; ++i) o.ptr[i] = i == 0 ? a.C : nullptr;
    o.ld = a.d.N; o.col0 = 0;
  }
  return o;
}

// ---- small device utilities -----------------------------------------------------------------
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t x, uint32_t mask, uint32_t orv) {
  uint32_t r;
  // (x & mask) | orv   -- immLut = (0xf0 & 0xcc) | 0xaa = 0xea
  asm("lop3.b32 %0, %1, %2, %3, 0xea;" : "=r"(r) : "r"(x), "r"(mask), "r"(orv));
  return r;
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldg_nc_v2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

template <typename T>
struct TypeTraits;
template <>
struct TypeTraits<__half> {
  static constexpr uint32_t kMagic = 0x64006400u;   // 1024.0 : (1024 + u) exact for u < 1024
  static constexpr uint32_t kMagicHi = 0x64006400u; // for nibble at bit 4: 1024 + 16u
  static constexpr int kMagicVal = 1024;
  using T2 = __half2;
  static __device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
};
template <>
struct TypeTraits<__nv_bfloat16> {
  static constexpr uint32_t kMagic = 0x43004300u;  // 128.0 : (128 + u) exact for u < 128
  static constexpr int kMagicVal = 128;
  using T2 = __nv_bfloat162;
  static __device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
};

__device__ __forceinline__ uint32_t h2_as_u32(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __half2 u32_as_h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }
__device__ __forceinline__ uint32_t b2_as_u32(__nv_bfloat162 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __nv_bfloat162 u32_as_b2(uint32_t v) { return *reinterpret_cast<__nv_bfloat162*>(&v); }

// packed 16-bit x2 arithmetic on raw registers, dispatched on element type
template <typename T>
__device__ __forceinline__ uint32_t sub2(uint32_t a, uint32_t b);
template <>
__device__ __forceinline__ uint32_t sub2<__half>(uint32_t a, uint32_t b) {
  return h2_as_u32(__hsub2(u32_as_h2(a), u32_as_h2(b)));
}
template <>
__device__ __forceinline__ uint32_t sub2<__nv_bfloat16>(uint32_t a, uint32_t b) {
  return b2_as_u32(__hsub2(u32_as_b2(a), u32_as_b2(b)));
}
template <typename T>
__device__ __forceinline__ uint32_t mul2(uint32_t a, uint32_t b);
template <>
__device__ __forceinline__ uint32_t mul2<__half>(uint32_t a, uint32_t b) {
  return h2_as_u32(__hmul2(u32_as_h2(a), u32_as_h2(b)));
}
template <>
__device__ __forceinline__ uint32_t mul2<__nv_bfloat16>(uint32_t a, uint32_t b) {
  return b2_as_u32(__hmul2(u32_as_b2(a), u32_as_b2(b)));
}
// a * b - c with TWO roundings (the _rn intrinsics are never contracted into an fma by the compiler)
template <typename T>
__device__ __forceinline__ uint32_t mul_then_sub2(uint32_t a, uint32_t b, uint32_t c);
template <>
__device__ __forceinline__ uint32_t mul_then_sub2<__half>(uint32_t a, uint32_t b, uint32_t c) {
  return h2_as_u32(__hsub2_rn(__hmul2_rn(u32_as_h2(a), u32_as_h2(b)), u32_as_h2(c)));
}
template <>
__device__ __forceinline__ uint32_t mul_then_sub2<__nv_bfloat16>(uint32_t a, uint32_t b, uint32_t c) {
  return b2_as_u32(__hsub2_rn(__hmul2_rn(u32_as_b2(a), u32_as_b2(b)), u32_as_b2(c)));
}
template <typename T>
__device__ __forceinline__ uint32_t fma2(uint32_t a, uint32_t b, uint32_t c);
template <>
__device__ __forceinline__ uint32_t fma2<__half>(uint32_t a, uint32_t b, uint32_t c) {
  return h2_as_u32(__hfma2(u32_as_h2(a), u32_as_h2(b), u32_as_h2(c)));
}
template <>
__device__ __forceinline__ uint32_t fma2<__nv_bfloat16>(uint32_t a, uint32_t b, uint32_t c) {
  return b2_as_u32(__hfma2(u32_as_b2(a), u32_as_b2(b), u32_as_b2(c)));
}
template <typename T>
__device__ __forceinline__ uint32_t dup2(T v) {
  uint16_t b = *reinterpret_cast<uint16_t*>(&v);
  return (uint32_t(b) << 16) | b;
}

// Per-group dequant constants (one weight row) of the tensor-core GEMM path:  v = ((x - mz) [- z2]) * s2 [+ negz2]
struct DqConst {
  uint32_t mz_lo, mz_hi;  // decode magic + folded integer zero point, for even / odd nibble positions
  uint32_t z2, s2, negz2;
};
// raw "magic + u" pair -> dequantised A_dtype pair, in A_dtype arithmetic with the reference's rounding order
// (bitblas/gpu/intrin/lop3.py:172-175 sub then mul; rescale: ONE fma for 4-bit (:256,269) but mul THEN sub -- two roundings --
// for 2-bit (:633-635); both orders are kept).  MODE: 0 none, 1 scale, 2 "original" zeros, 3 "rescale" zeros, 4 quantized zeros
// (integer zero point folded into mz).
template <typename T, int MODE, int BITS = 4>
__device__ __forceinline__ uint32_t dq_finish(uint32_t x, uint32_t mz, const DqConst& c) {
  const uint32_t t = sub2<T>(x, mz);
  if constexpr (MODE == 1 || MODE == 4) return mul2<T>(t, c.s2);
  if constexpr (MODE == 2) return mul2<T>(sub2<T>(t, c.z2), c.s2);
  if constexpr (MODE == 3) {
    if constexpr (BITS == 2) return mul_then_sub2<T>(t, c.s2, c.z2);
    else return fma2<T>(t, c.s2, c.negz2);
  }
  return t;
}

// ---- 16-entry table formats (NF4: caller's LUT, matmul_dequantize_impl.py:424-430; "fp4": sign + 3-bit exponent,
// quantization.py:141-156) decoded in registers with byte permutes ------------------------------------------------------------
// The table of 16 x 16-bit A_dtype values is kept as two byte planes of 16 bytes (4 registers each).  One PRMT looks up four
// 3-bit indices in 8 bytes; index bit 3 picks between the lower / upper half of the table with a second PRMT whose selector
// is built from those bits: 21 ALU operations per packed word (8 weights), no shared-memory or constant-bank traffic.
struct Lut4 { uint32_t lo[4], hi[4]; };

__host__ __device__ constexpr uint16_t fp4_table_bits(int u, bool bf16) {
  const int s = u >> 3, e = u & 7;
  if (e == 0) return 0;                                                    // exponent field 0 decodes to 0 (quantization.py:150-156)
  return bf16 ? uint16_t((s << 15) | ((120 + e) << 7))                     // 2^(e-7) in bfloat16
              : uint16_t(((e | 8) | (s << 5)) << 10);                      // the reference's fp16 bit pattern
}
__device__ __forceinline__ void lut4_from_pairs(Lut4& t, const uint32_t (&r)[8]) {   // r[j] = (entry 2j, entry 2j+1)
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    t.lo[k] = __byte_perm(r[2 * k], r[2 * k + 1], 0x6420);
    t.hi[k] = __byte_perm(r[2 * k], r[2 * k + 1], 0x7531);
  }
}
// fmt: BB_W_NF -> 16 entries from `lut` (A_dtype, any 2-byte alignment); BB_W_FP4 -> the fixed table
__device__ __forceinline__ void lut4_init(Lut4& t, int fmt, bool bf16, const void* lut) {
  uint32_t r[8];
  if (fmt == BB_W_NF) {
    const uint16_t* l = reinterpret_cast<const uint16_t*>(lut);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = uint32_t(__ldg(l + 2 * j)) | (uint32_t(__ldg(l + 2 * j + 1)) << 16);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      r[j] = bf16 ? (uint32_t(fp4_table_bits(2 * j, true)) | (uint32_t(fp4_table_bits(2 * j + 1, true)) << 16))
                  : (uint32_t(fp4_table_bits(2 * j, false)) | (uint32_t(fp4_table_bits(2 * j + 1, false)) << 16));
  }
  lut4_from_pairs(t, r);
}
// compressed storage (element j in nibble j): out[i] = (T[e(2i)], T[e(2i+1)])  i = 0..3
__device__ __forceinline__ void lut4_decode8(uint32_t w, const Lut4& t, uint32_t (&out)[4]) {
  const uint32_t s7 = w & 0x77777777u;                              // 3-bit indices (a selector's bit 3 would sign-replicate)
  const uint32_t pk = ((w >> 1) & 0x44444444u) | 0x32103210u;       // byte k of (lower-half result | upper-half result)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t s = h ? (s7 >> 16) : s7, p = h ? (pk >> 16) : pk;
    const uint32_t l4 = __byte_perm(__byte_perm(t.lo[0], t.lo[1], s), __byte_perm(t.lo[2], t.lo[3], s), p);
    const uint32_t h4 = __byte_perm(__byte_perm(t.hi[0], t.hi[1], s), __byte_perm(t.hi[2], t.hi[3], s), p);
    out[2 * h] = __byte_perm(l4, h4, 0x5140);
    out[2 * h + 1] = __byte_perm(l4, h4, 0x7362);
  }
}

// ---- in-register decode of packed low-bit words -----------------------------------------------
// 4-bit, 16-bit target.  Returns raw "magic + u" pairs (bias removed by the caller with one sub/fma).
//   interleaved layout (quantization/utils.py:73-110): out[i] = (u[2i], u[2i+1])       i = 0..3
//   compressed  layout:                                 out[i] = (u[i],  u[i+4])         i = 0..3
template <typename T>
__device__ __forceinline__ void decode_u4x8_raw(uint32_t w, uint32_t (&out)[4]) {
  constexpr uint32_t M = TypeTraits<T>::kMagic;
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = lop3_and_or(w >> (4 * i), 0x000f000fu, M);
}
// 2-bit, 16-bit target, interleaved layout: one 32-bit word = 16 values; out[i] = (u[2i], u[2i+1]) i = 0..7
template <typename T>
__device__ __forceinline__ void decode_u2x16_raw_interleaved(uint32_t w, uint32_t (&out)[8]) {
  constexpr uint32_t M = TypeTraits<T>::kMagic;
  uint32_t lo = __byte_perm(w, 0, 0x4140);  // [b0, 0, b1, 0]
  uint32_t hi = __byte_perm(w, 0, 0x4342);  // [b2, 0, b3, 0]
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    out[i] = lop3_and_or(lo >> (2 * i), 0x00030003u, M);
    out[4 + i] = lop3_and_or(hi >> (2 * i), 0x00030003u, M);
  }
}
// 2-bit, 16-bit target, compressed layout: out[i] = (u[i], u[i+8]) i = 0..7
template <typename T>
__device__ __forceinline__ void decode_u2x16_raw_compressed(uint32_t w, uint32_t (&out)[8]) {
  constexpr uint32_t M = TypeTraits<T>::kMagic;
#pragma unroll
  for (int i = 0; i < 8; ++i) out[i] = lop3_and_or(w >> (2 * i), 0x00030003u, M);
}

// 8-bit target.  interleaved-8 layout: out[i] = (u[4i..4i+3]) as 4 bytes.
//   2-bit: 16 values / word, i = 0..3 ; 4-bit: 8 values / word, i = 0..1
// `orv` is OR-ed in the same LOP3 (0 or 0x80808080 for the borrow-free signed trick).
__device__ __forceinline__ void decode_u2x16_to_u8(uint32_t w, uint32_t orv, uint32_t (&out)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = lop3_and_or(w >> (2 * i), 0x03030303u, orv);
}
__device__ __forceinline__ void decode_u4x8_to_u8(uint32_t w, uint32_t orv, uint32_t (&out)[2]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) out[i] = lop3_and_or(w >> (4 * i), 0x0f0f0f0fu, orv);
}
// bytes (u | 0x80) -> signed (u - zp) without inter-byte borrows: ((u|0x80) - zp) ^ 0x80
__device__ __forceinline__ uint32_t bytes_sub_zp(uint32_t v_or80, uint32_t zp4) {
  return (v_or80 - zp4) ^ 0x80808080u;
}

}  // namespace bb
