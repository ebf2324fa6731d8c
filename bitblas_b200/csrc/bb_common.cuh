// bb_common.cuh -- shared host/device helpers for the sm_90a kernels.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <type_traits>
#include <utility>

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

// The output form of a single-matrix matmul: Plain (bb_matmul, bb_matmul_scatter), SwiGLU (bb_matmul_swiglu: W holds gate/up
// interleaved, d.N = 2I rows, and C is [m, d.N / 2] = silu(gate) * up), Scaled (bb_matmul_scaled: the dequantizing epilogue
// store_out_scaled) and W4A8 (bb_matmul_w4a8: per-group fp32 weight scales, store_out_dequant)
enum class MatmulForm : int { Plain, SwiGLU, Scaled, W4A8 };
// the fp32 scales the Scaled and W4A8 forms read (both null in the other forms): a_scale [m], one per row of A (the preceding
// kernel's output, read after the PDL wait); w_scale: Scaled's per-column weight scales [N], W4A8's group scales [N, K/g]
struct ScaledArgs {
  const float* a_scale = nullptr;
  const float* w_scale = nullptr;
};

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
  MatmulForm form;
  ScaledArgs scaled;
  int groups() const { return d.K / (d.group_size <= 0 ? d.K : d.group_size); }
  int gsize() const { return d.group_size <= 0 ? d.K : d.group_size; }
};

constexpr int BB_MAX_DEVICES = 64;
int current_device();     // ordinal of the calling thread's current CUDA device, clamped to [0, BB_MAX_DEVICES)
int device_sm_count();    // SM count of the current device (cached per device), at most the bb_set_sm_count_cap cap
int device_sm_count_uncapped();   // the same without the cap
// whether the streaming kernels launch with programmatic dependent launch (default on; BB_PDL=0 restores plain stream order)
bool pdl_enabled();

// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-stream-serialization attribute set to `overlap`
// (pdl_enabled() for the library's matmul kernels): the launch may then begin while its predecessor on the stream finishes.
// Counts the launch; returns 0, or 2 / 3 with the error set as BB_CHECK_CUDA / BB_LAUNCH_CHECK do.
template <typename... Params, typename... Args>
int launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool overlap, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = overlap ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) {
    set_error("cudaLaunchKernelEx failed: %s (%s:%d)", cudaGetErrorString(e), __FILE__, __LINE__);
    return 2;
  }
  BB_LAUNCH_CHECK();
  return 0;
}

// One-time set-up of a kernel instance, done once per device.  A launcher keeps one `static KernelCache` per kernel instance
// (several instances share one function-pointer type, so the storage cannot be keyed on the type), with SLOTS results per
// device: one per block size it launches the instance with.
template <int SLOTS = 1>
struct KernelCache {
  std::atomic<int> v[BB_MAX_DEVICES][SLOTS];   // 0: not set up on that device yet; -1: cannot be resident
};
constexpr size_t kSmemOptinMax = ~size_t(0);

// Sets `kernel` up on device `dev` (the current device), once per (device, slot) of `cache`: raises its dynamic shared-memory
// limit to smem_limit bytes (kSmemOptinMax: the device's opt-in maximum; 0: leaves it), then, with threads > 0, queries how many
// CTAs of `threads` threads and `smem` dynamic bytes are resident per SM.  Returns that count (1 when threads == 0), or 0 when
// the kernel cannot be resident or a runtime call failed; a failed call's error is cleared and nothing is cached.
template <int SLOTS, typename Kernel>
int kernel_setup(KernelCache<SLOTS>& cache, Kernel kernel, size_t smem_limit, int threads = 0, size_t smem = 0, int slot = 0,
                 int dev = current_device()) {
  std::atomic<int>& c = cache.v[dev][slot];
  const int cached = c.load(std::memory_order_relaxed);
  if (cached != 0) return cached > 0 ? cached : 0;
  int limit = int(smem_limit), occ = 1;
  bool ok = true;
  if (smem_limit == kSmemOptinMax) ok = cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess;
  if (ok && smem_limit != 0) ok = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, limit) == cudaSuccess;
  if (ok && threads > 0) ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    return 0;
  }
  c.store(occ > 0 ? occ : -1, std::memory_order_relaxed);
  return occ > 0 ? occ : 0;
}

// the driver's cuTensorMapEncodeTiled, looked up once through the runtime (no libcuda link); null when unavailable
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder();
// a 2-D TMA map: `outer` rows of `inner` elements, `row_stride_bytes` apart; box = box_inner x box_outer.  Returns 0, or 4 with the
// error set
int make_map_2d(CUtensorMap* map, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw);

// The instance ladder of the kernels built for 16-bit activations x 4- / 2-bit weights x interleaved / compressed storage:
// f(TypeTag<T>, BITS, IL) for d's a_dtype (float16, else bfloat16), w_bits (4, else 2) and w_layout, BITS and IL as
// std::integral_constant / std::bool_constant.
template <typename T>
struct TypeTag { using type = T; };
template <typename F>
int dispatch_t_bits_il(const bb_matmul_desc& d, F&& f) {
  const bool il = d.w_layout == BB_LAYOUT_INTERLEAVED_16;
  auto bits_il = [&](auto t) {
    using std::integral_constant;
    if (d.w_bits == 4) return il ? f(t, integral_constant<int, 4>{}, std::true_type{}) : f(t, integral_constant<int, 4>{}, std::false_type{});
    return il ? f(t, integral_constant<int, 2>{}, std::true_type{}) : f(t, integral_constant<int, 2>{}, std::false_type{});
  };
  return d.a_dtype == BB_F16 ? bits_il(TypeTag<__half>{}) : bits_il(TypeTag<__nv_bfloat16>{});
}

// kernel family entry points (each returns 0 / error code; *_supported says whether the family covers it)
bool generic_supported(const bb_matmul_desc& d);
int launch_generic(const MatmulArgs& a);
bool gemv_mma_supported(const bb_matmul_desc& d, int m);
int launch_gemv_mma(const MatmulArgs& a);
bool gemv_slab_supported(const bb_matmul_desc& d, int m);
int launch_gemv_slab(const MatmulArgs& a);
size_t gemv_slab_workspace_bytes();     // tagged partial slots (must be zero-initialised once by the caller)
size_t gemv_slab_slot_bytes(int sms);   // the slot region of a launch on `sms` SMs (gemv_slab_workspace_bytes at device_sm_count)
bool gemv_i8_supported(const bb_matmul_desc& d, int m);
int launch_gemv_i8(const MatmulArgs& a);
bool gemm_ts_supported(const bb_matmul_desc& d, int m);
int launch_gemm_ts(const MatmulArgs& a);
size_t gemm_ts_workspace_bytes(const bb_matmul_desc& d, int m);
int gemm_ts_splits(int tiles, int num_kb, int sms);   // the wgmma GEMM's split-K factor for a tile grid and k-block count
// one bb_matmul_fp8 call, validated by bb_api.cu (bb_gemm_fp8.cu)
struct Fp8Args {
  bb_matmul_desc d;
  const void* A;          // e4m3 [m, K]
  const float* a_scale;   // fp32, element (r, b) at a_scale[b * a_scale_ld + r]
  int a_scale_ld;
  const void* W;          // e4m3 [N, K]
  const float* w_scale;   // fp32 [ceil(N / 128), K / 128]
  const void* bias;       // [N] out_dtype, or null
  void* C;
  int m;
  void* workspace;
  size_t workspace_bytes;
  cudaStream_t stream;
};
int launch_gemm_fp8(const Fp8Args& a);
size_t gemm_fp8_workspace_bytes(const bb_matmul_desc& d, int m);
// one bb_matmul_grouped_fp8[_swiglu] call, validated by bb_api.cu (bb_grouped_fp8.cu)
struct GroupedFp8Args {
  bb_matmul_desc d;
  int num_groups;
  const int32_t* offsets;   // [num_groups + 1], device
  const void* A;            // e4m3 [total_rows, K]
  const float* a_scale;     // fp32, element (r, b) at a_scale[b * a_scale_ld + r]
  int a_scale_ld;
  const void* W;            // e4m3 [E, N, K]
  const float* w_scale;     // fp32 [E, N / 128, K / 128]; swiglu: [E, 2 ceil(N / 256), K / 128], gate and up blocks alternating
  void* C;                  // [total_rows, N] (swiglu: [total_rows, N / 2]) out_dtype
  int total_rows;
  cudaStream_t stream;
  bool swiglu;
};
int launch_grouped_fp8(const GroupedFp8Args& a);
// one grouped (mixture-of-experts) call, validated by bb_api.cu: num_groups problems of descriptor d, group e on rows
// [offsets[e], offsets[e + 1]) of A and C; W, scale, zeros and bias are stacked over the groups
struct GroupedArgs {
  bb_matmul_desc d;
  int num_groups;
  const int32_t* offsets;   // [num_groups + 1], device
  const void* A;
  const void* W;
  const void* scale;
  const void* zeros;
  const void* bias;
  void* C;
  int total_rows;
  cudaStream_t stream;
  bool swiglu;              // W holds gate/up interleaved (2I = d.N rows), C is [total_rows, d.N / 2] = silu(gate) * up
  const int32_t* row_index; // gathering GEMM (swiglu only), else null: sorted row r reads A[clamp(row_index[r], 0, a_rows - 1)]
  int a_rows;               //   of A [a_rows, K] instead of A[r]
  long long w_stride, s_stride, z_stride, b_stride;   // bytes per group of W, scale, zeros and bias
};
// grouped matmul, bb_grouped.cu (the decode GEMV's kernel), and grouped wgmma GEMM, bb_grouped_gemm.cu: *_supported set the
// error message when they return false (store_swiglu below is the SwiGLU epilogue of both)
bool grouped_supported(const bb_matmul_desc& d);
int launch_grouped(const GroupedArgs& g);
bool grouped_gemm_supported(const bb_matmul_desc& d);
int launch_grouped_gemm(const GroupedArgs& g);
// mixture-of-experts routing and top-k combine, bb_moe.cu (arguments validated by the callers in bb_api.cu).  Routing copies x
// into x_sorted, or, with x_sorted == nullptr, writes row_token instead (bb_moe_route_index)
int launch_moe_route(const int32_t* topk_ids, int n_slots, int top_k, int num_experts, const void* x, int K, int32_t* offsets,
                     int32_t* slot_rows, void* x_sorted, int32_t* row_token, cudaStream_t stream);
int launch_moe_combine(const int32_t* slot_rows, const float* topk_weights, const void* Y, int out_dtype, void* out,
                       int num_tokens, int top_k, int N, cudaStream_t stream);
// top-k gating from router logits, bb_moe.cu (validated by bb_moe_topk in bb_api.cu)
int launch_moe_topk(const void* logits, int logits_dtype, int num_tokens, int num_experts, int top_k, int scoring,
                    const float* correction_bias, int num_expert_group, int topk_group, int group_score, int renormalize,
                    float routed_scaling_factor, int32_t* topk_ids, float* topk_weights, cudaStream_t stream);
// act-order column gather, bb_permute.cu (validated by bb_api.cu): one row of A is staged in shared memory, so K <= PERMUTE_MAX_K
// (H100: 227 KB per block, less the 3 KB of the kernel's static arrays)
constexpr int PERMUTE_MAX_K = 112640;
int launch_permute_cols(const void* A, void* out, const int32_t* perm, int rows, int K, int num_groups, const int32_t* offsets,
                        cudaStream_t stream);
// per-token int8 quantization of the activations, bb_quant.cu (validated by bb_quantize_act_int8 in bb_api.cu)
int launch_quantize_act_int8(const void* x, int a_dtype, int rows, int K, int8_t* q, float* scale, cudaStream_t stream);
// per-(token, 128-column block) e4m3 quantization, bb_quant.cu (validated by bb_quantize_act_fp8)
int launch_quantize_act_fp8(const void* x, int a_dtype, int rows, int K, uint8_t* q, float* scale, int scale_ld, cudaStream_t stream);

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
inline OutSpec make_outspec(void* C, long long ld) {   // the single output C
  OutSpec o;
  o.n = 1;
  for (int i = 0; i < BB_MAX_PEERS; ++i) o.ptr[i] = i == 0 ? C : nullptr;
  o.ld = ld; o.col0 = 0;
  return o;
}
inline OutSpec make_outspec(const MatmulArgs& a) {
  if (a.n_peers == 0) return make_outspec(a.C, a.form == MatmulForm::SwiGLU ? a.d.N / 2 : a.d.N);
  OutSpec o;
  o.n = a.n_peers;
  for (int i = 0; i < BB_MAX_PEERS; ++i) o.ptr[i] = i < a.n_peers ? a.peer_C[i] : nullptr;
  o.ld = a.ldc; o.col0 = a.col_offset;
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

// shared memory, mbarriers and TMA: each wrapper takes 32-bit shared-memory addresses; the pointer forms convert through smem_u32
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { mbar_init(smem_u32(bar), count); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_arrive_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { mbar_arrive(smem_u32(bar)); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// (`map` is a const void* here: typed as const CUtensorMap*, the slab GEMV's coordinate registers are assigned differently)
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  tma_load_2d(smem_u32(dst), map, c0, c1, smem_u32(bar));
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// L2 eviction policies for the .L2::cache_hint copies below: evict_first for bytes read exactly once, evict_last for bytes that
// later requests read again
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const void* map, int c0, int c1, uint32_t bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
               : "memory");
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

// the 16-bit pattern b as a T, widened to float
template <typename T>
__device__ __forceinline__ float raw_to_float(uint16_t b) {
  return TypeTraits<T>::to_float(*reinterpret_cast<const T*>(&b));
}

// c += A (16 x 16, T) * B (16 x 8, T) with fp32 accumulators
template <typename T>
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

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

// Programmatic dependent launch (the design notes are in bb_gemv_mma.cuh)
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- work schedule of the grouped (mixture-of-experts) kernels over untrusted device offsets ---------------------------------
// Run by the 32 lanes of one warp (lane = threadIdx.x) on the kernel's parameters g (g.offsets [g.E + 1], g.T rows; read from the
// parameter space as the kernel would): clamps offsets[e], offsets[e + 1] to [0, T] (a group whose end is below its start is
// empty) into row0_s[e] / rows_s[e], and gives group e the work items [item0_s[e], item0_s[e + 1]): per_chunk * ceil(rows / R)
// of them, numbered by one warp prefix sum; item0_s[E] = all items.  The caller synchronises the CTA before it reads the arrays.
template <typename GP>
__device__ __forceinline__ void grouped_schedule(const GP& g, int R, int per_chunk, int* row0_s, int* rows_s, int* item0_s) {
  const int lane = threadIdx.x;
  const int per = (g.E + 31) / 32;   // consecutive groups per lane
  const int e0 = lane * per;
  int cnt = 0;
  for (int i = 0; i < per; ++i) {
    const int e = e0 + i;
    if (e < g.E) {
      const int b = min(max(g.offsets[e], 0), g.T);
      const int m = max(min(max(g.offsets[e + 1], 0), g.T) - b, 0);
      row0_s[e] = b;
      rows_s[e] = m;
      cnt += per_chunk * ((m + R - 1) / R);
    }
  }
  int incl = cnt;   // inclusive prefix sum over the lanes
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  int run = incl - cnt;
  for (int i = 0; i < per; ++i) {
    const int e = e0 + i;
    if (e < g.E) {
      item0_s[e] = run;
      run += per_chunk * ((rows_s[e] + R - 1) / R);
    }
  }
  if (lane == 31) item0_s[g.E] = incl;
}
// ---- output rounding: how every epilogue turns one accumulator into an output element -------------------------------------------
// Float accumulators: cast to out_dtype, then the bias (a float of A_dtype, 0 without one) added in out_dtype; an fp32 output is
// one sum.  This is bb_matmul's rounding; the grouped kernels are bit-identical to it because they round the same way.
template <typename O>
__device__ __forceinline__ O round_out(float v, bool has_bias, float bias) {
  if constexpr (std::is_same<O, float>::value) {
    return v + bias;
  } else {
    O r = TypeTraits<O>::from_float(v);
    if (has_bias) r = __hadd(r, TypeTraits<O>::from_float(bias));
    return r;
  }
}
// Int32 accumulators (int8 activations): the sum and the int8 bias b are each converted to out_dtype and added there
__device__ __forceinline__ void store_out_i32(void* C, size_t o, int v, int b, int out_dtype) {
  switch (out_dtype) {
    case BB_I32: reinterpret_cast<int*>(C)[o] = v + b; break;
    case BB_I8: reinterpret_cast<int8_t*>(C)[o] = int8_t(int8_t(v) + b); break;
    case BB_F32: reinterpret_cast<float*>(C)[o] = float(v) + float(b); break;
    case BB_F16: reinterpret_cast<__half*>(C)[o] = __hadd(__int2half_rn(v), __int2half_rn(b)); break;
    default: reinterpret_cast<__nv_bfloat16*>(C)[o] = __hadd(__int2bfloat16_rn(v), __int2bfloat16_rn(b));
  }
}
// The dequantizing epilogue of bb_matmul_scaled: C[o] = round_out((float(acc) / s_a) / s_w) with the bias element n (out_dtype, null:
// none) added in out_dtype after the rounding; an fp32 output is one sum.  The scales are quantization scales (value x scale = the
// integer grid), so both steps divide, in BitNet's order; __fdiv_rn keeps them correctly rounded whatever the compiler flags.
__device__ __forceinline__ void store_out_scaled(void* C, size_t o, int acc, float s_a, float s_w, const void* bias, int n,
                                                 int out_dtype) {
  const float y = __fdiv_rn(__fdiv_rn(__int2float_rn(acc), s_a), s_w);
  const bool hb = bias != nullptr;
  if (out_dtype == BB_F16) {
    reinterpret_cast<__half*>(C)[o] = round_out<__half>(y, hb, hb ? __half2float(reinterpret_cast<const __half*>(bias)[n]) : 0.f);
  } else if (out_dtype == BB_BF16) {
    reinterpret_cast<__nv_bfloat16*>(C)[o] =
        round_out<__nv_bfloat16>(y, hb, hb ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(bias)[n]) : 0.f);
  } else {
    reinterpret_cast<float*>(C)[o] = round_out<float>(y, hb, hb ? reinterpret_cast<const float*>(bias)[n] : 0.f);
  }
}

// The epilogue of bb_matmul_w4a8: C[o] = round_out(y) with y = S / a_scale[r] already divided (__fdiv_rn), the bias element n
// (out_dtype, null: none) added in out_dtype after the rounding; an fp32 output is one sum
__device__ __forceinline__ void store_out_dequant(void* C, size_t o, float y, const void* bias, int n, int out_dtype) {
  const bool hb = bias != nullptr;
  if (out_dtype == BB_F16) {
    reinterpret_cast<__half*>(C)[o] = round_out<__half>(y, hb, hb ? __half2float(reinterpret_cast<const __half*>(bias)[n]) : 0.f);
  } else if (out_dtype == BB_BF16) {
    reinterpret_cast<__nv_bfloat16*>(C)[o] =
        round_out<__nv_bfloat16>(y, hb, hb ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(bias)[n]) : 0.f);
  } else {
    reinterpret_cast<float*>(C)[o] = round_out<float>(y, hb, hb ? reinterpret_cast<const float*>(bias)[n] : 0.f);
  }
}
// one group's promotion in bb_matmul_w4a8: S + float(acc) * s, each step rounded to nearest (never contracted into an fma)
__device__ __forceinline__ float w4a8_promote(float S, int acc, float s) { return __fadd_rn(S, __fmul_rn(__int2float_rn(acc), s)); }
// the zero point of 4-bit weight row n in group gi: its nibble of the packed quantized zeros [G, N / 2], or z_const (8 for int
// weights, 0 for uint weights without zeros) when qz is null
__device__ __forceinline__ int w4a8_zero(const uint8_t* qz, int N, int gi, int n, int z_const) {
  return qz ? int((__ldg(qz + size_t(gi) * (size_t(N) / 2) + n / 2) >> (4 * (n & 1))) & 15u) : z_const;
}

// ---- SwiGLU epilogue of bb_matmul_swiglu and the grouped SwiGLU calls (gate/up interleave: weight row 16b + i is gate row 8b + i for
// i < 8, up row 8b + i - 8 for i >= 8) ----------------------------------------------------------------------------------------------
// one pre-activation as the plain epilogue stores it
__device__ __forceinline__ float swiglu_operand(float v, bool has_bias, float bias, int out_dtype) {
  if (out_dtype == BB_F16) return __half2float(round_out<__half>(v, has_bias, bias));
  if (out_dtype == BB_BF16) return __bfloat162float(round_out<__nv_bfloat16>(v, has_bias, bias));
  return round_out<float>(v, has_bias, bias);
}
// C[o] = silu(g) * u = g / (1 + exp(-g)) * u in fp32, rounded once to out_dtype
__device__ __forceinline__ void store_swiglu(void* C, size_t o, float g, float u, int out_dtype) {
  const float y = g / (1.f + expf(-g)) * u;
  if (out_dtype == BB_F16) reinterpret_cast<__half*>(C)[o] = __float2half_rn(y);
  else if (out_dtype == BB_BF16) reinterpret_cast<__nv_bfloat16*>(C)[o] = __float2bfloat16_rn(y);
  else reinterpret_cast<float*>(C)[o] = y;
}

// the group of work item `item`: the last e with item0_s[e] <= item (an empty group shares its start with the next one)
__device__ __forceinline__ int grouped_find(const int* item0_s, int E, int item) {
  int lo = 0, hi = E - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (item0_s[mid] <= item) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace bb
