// bb_api.cu -- the C ABI (include/bitblas_b200.h): validation, kernel dispatch, error reporting.
//
// Dispatch mirrors the reference's run-time choice (bitblas/ops/general_matmul/tilelang/dequantize/
// matmul_dequantize.py:93-111: M < 8 -> SIMT GEMV, else MMA GEMM; and the per-opt_M if-chain emitted into
// `call`, bitblas/builder/wrapper/tl.py:278-300) but is keyed on the H100 regimes instead:
//   m <= 8   : memory-bound streaming kernels (bb_gemv.cu)
//   m  > 8   : wgmma tensor-core kernel (bb_gemm_ts.cu), split-K when the tile grid is smaller than the chip
//   anything the fast kernels do not cover: the generic SIMT kernel (bb_generic.cu).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "bb_common.cuh"

namespace bb {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_override{BB_KERNEL_AUTO};
static std::atomic<int> g_sm_count[BB_MAX_DEVICES];   // 0 = not queried yet; per-device state is keyed on the ordinal
static std::atomic<int> g_sm_cap{0};                  // bb_set_sm_count_cap; 0 = no cap

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
  return (dev < 0 || dev >= BB_MAX_DEVICES) ? 0 : dev;
}

int device_sm_count_uncapped() {
  const int dev = current_device();
  int n = g_sm_count[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); n = 132; }
    g_sm_count[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

int device_sm_count() {
  const int n = device_sm_count_uncapped();
  const int cap = g_sm_cap.load(std::memory_order_relaxed);
  return cap > 0 && cap < n ? cap : n;
}

bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("BB_PDL"); return e ? atoi(e) != 0 : true; }();
  return on;
}

EncodeTiledFn tensor_map_encoder() {
  static const EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}

int make_map_2d(CUtensorMap* map, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 4; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", int(r)); return 4; }
  return 0;
}

static int validate(const bb_matmul_desc* d) {
  if (!d) { set_error("null descriptor"); return 1; }
  if (d->N <= 0 || d->K <= 0) { set_error("N and K must be positive (N=%d K=%d)", d->N, d->K); return 1; }
  if (d->a_dtype != BB_F16 && d->a_dtype != BB_BF16 && d->a_dtype != BB_I8) {
    set_error("unsupported A_dtype id %d (float16 | bfloat16 | int8)", d->a_dtype); return 1;
  }
  if (d->w_bits != 1 && d->w_bits != 2 && d->w_bits != 4 && d->w_bits != 8) {
    set_error("unsupported weight bit width %d", d->w_bits); return 1;
  }
  if (d->w_fmt < BB_W_UINT || d->w_fmt > BB_W_FP8_E5M2) { set_error("unsupported weight format id %d", d->w_fmt); return 1; }
  if ((d->w_fmt == BB_W_NF || d->w_fmt == BB_W_FP4) && d->w_bits != 4) { set_error("nf4/fp4 need 4-bit storage"); return 1; }
  if ((d->w_fmt == BB_W_FP8_E4M3 || d->w_fmt == BB_W_FP8_E5M2) && d->w_bits != 8) { set_error("fp8 needs 8-bit storage"); return 1; }
  const int g = d->group_size <= 0 ? d->K : d->group_size;
  if (d->K % g) { set_error("K=%d is not divisible by group_size=%d", d->K, g); return 1; }
  if (d->with_zeros && (d->zeros_mode < 0 || d->zeros_mode > 2)) { set_error("bad zeros_mode %d", d->zeros_mode); return 1; }
  if (d->w_layout < 0 || d->w_layout > 2) { set_error("bad w_layout %d", d->w_layout); return 1; }
  if (d->w_layout != BB_LAYOUT_COMPRESSED && d->w_bits == 8) { set_error("8-bit weights cannot be interleaved"); return 1; }
  if (d->a_dtype == BB_I8 && d->accum_dtype != BB_I32) { set_error("int8 activations need accum_dtype=int32"); return 1; }
  if (d->a_dtype != BB_I8 && d->accum_dtype == BB_I32) { set_error("int32 accumulation needs int8 activations"); return 1; }
  if (d->a_dtype != BB_I8 && d->out_dtype != BB_F16 && d->out_dtype != BB_BF16 && d->out_dtype != BB_F32) {
    set_error("float path supports out_dtype float16 | bfloat16 | float32"); return 1;
  }
  if (d->reserved[0] || d->reserved[1]) { set_error("reserved fields must be zero"); return 1; }
  if (d->w_tile != BB_TILE_ROW_MAJOR && d->w_tile != BB_TILE_SLAB) { set_error("bad w_tile %d", d->w_tile); return 1; }
  if (d->w_tile == BB_TILE_SLAB && !((d->w_fmt == BB_W_UINT || d->w_fmt == BB_W_INT) && (d->w_bits == 4 || d->w_bits == 2))) {
    set_error("BB_TILE_SLAB is defined for 4- and 2-bit integer weights (the combinations the parity suite covers)");
    return 1;
  }
  if (d->w_tile == BB_TILE_SLAB && !tile_shape_ok(*d)) {
    set_error("BB_TILE_SLAB needs N %% %d == 0 and K*bits/8 %% %d == 0 (N=%d K=%d bits=%d)", BB_TILE_ROWS, BB_TILE_ROW_BYTES, d->N, d->K, d->w_bits);
    return 1;
  }
  if (!generic_supported(*d)) { set_error("configuration not supported (K*bits must be a multiple of 32)"); return 1; }
  return 0;
}

static int select(const bb_matmul_desc& d, int m) {
  const int ov = g_override.load();
  if (ov != BB_KERNEL_AUTO) {
    switch (ov) {
      case BB_KERNEL_GENERIC: return BB_KERNEL_GENERIC;
      case BB_KERNEL_GEMV_MMA: if (gemv_mma_supported(d, m)) return ov; break;
      case BB_KERNEL_GEMV_I8: if (gemv_i8_supported(d, m)) return ov; break;
      case BB_KERNEL_GEMM_TS: if (d.a_dtype != BB_I8 && gemm_ts_supported(d, m)) return ov; break;
      case BB_KERNEL_GEMM_TS_I8: if (d.a_dtype == BB_I8 && gemm_ts_supported(d, m)) return ov; break;
      case BB_KERNEL_GEMV_SLAB: if (gemv_slab_supported(d, m)) return ov; break;
    }
    return -1;
  }
  if (d.w_tile == BB_TILE_SLAB) {
    // slab-tiled storage is consumed by the two TMA kernels (a different tensor map, nothing else) and by the generic kernel;
    // the register-streaming kernels address rows directly and are not offered this layout
    if (gemv_slab_supported(d, m)) return BB_KERNEL_GEMV_SLAB;
    if (gemm_ts_supported(d, m)) return d.a_dtype == BB_I8 ? BB_KERNEL_GEMM_TS_I8 : BB_KERNEL_GEMM_TS;
    return BB_KERNEL_GENERIC;
  }
  // m <= 8 (one n8 MMA tile): streaming kernels; above that the wgmma kernel (split-K keeps the SMs busy at small m)
  // is faster (12288^2 sweep, tools/smallm_sweep.py); the streaming kernels stay as the fallback up to m = 32.
  if (m <= 8) {
    if (gemv_slab_supported(d, m)) return BB_KERNEL_GEMV_SLAB;
    if (gemv_mma_supported(d, m)) return BB_KERNEL_GEMV_MMA;
    if (gemv_i8_supported(d, m)) return BB_KERNEL_GEMV_I8;
  }
  if (gemm_ts_supported(d, m)) return d.a_dtype == BB_I8 ? BB_KERNEL_GEMM_TS_I8 : BB_KERNEL_GEMM_TS;
  if (m <= 32) {
    if (gemv_mma_supported(d, m)) return BB_KERNEL_GEMV_MMA;
    if (gemv_i8_supported(d, m)) return BB_KERNEL_GEMV_I8;
  }
  return BB_KERNEL_GENERIC;
}

// ---- cross-rank barrier of the column-parallel path -------------------------------------------------------------------
// One tiny kernel instead of a library collective: every rank bumps its own sequence number, release-stores it into slot [rank] of
// every peer's flag block (peer-mapped symmetric memory, NVLink) and acquire-spins until all of its own slots reached it.  The kernel
// is launched with the programmatic-dependent-launch attribute and starts with griddepcontrol.wait: all memory operations of the
// preceding matmul kernel(s) -- the peer stores of bb_matmul_scatter -- are complete and visible before the flag goes out, and
// the next matmul kernel (a programmatic dependent of this one) fetches its first weights while this one spins.
// Flag block (per rank, symmetric, zero-initialised once): uint32 slot[BB_MAX_PEERS]; uint32 pad[8]; uint32 seq (index 16).
struct PeerBarrierArgs { uint32_t* flags[BB_MAX_PEERS]; int n, rank; };

__global__ void peer_barrier_kernel(const PeerBarrierArgs a) {
  __shared__ uint32_t seq_s;
  pdl_wait();
  pdl_launch_dependents();
  uint32_t* mine = a.flags[a.rank];
  if (threadIdx.x == 0) {
    const uint32_t seq = mine[16] + 1u;
    mine[16] = seq;
    seq_s = seq;
  }
  __syncthreads();
  const uint32_t seq = seq_s;
  const int p = threadIdx.x;
  if (p < a.n) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.flags[p] + a.rank), "r"(seq) : "memory");
    const long long t0 = clock64();
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + p) : "memory");
      if (clock64() - t0 > (20ll << 30)) __trap();   // ~10 s at 2 GHz: a peer died; fail the launch instead of hanging the GPU
    } while (int(v - seq) < 0);
  }
}

}  // namespace bb

using namespace bb;

extern "C" {

int bb_version(void) { return BB_VERSION; }
const char* bb_last_error(void) { return g_err; }
uint64_t bb_launch_count(void) { return g_launches.load(); }

int bb_init(int device) {
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("no CUDA device available: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return 2;
  }
  if (device < 0 || device >= ndev) { set_error("device %d out of range (%d devices)", device, ndev); return 1; }
  // queries only: the caller's current device is left untouched (torch owns it)
  int major = 0;
  BB_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  int minor = 0;
  BB_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  if (major != 9 || minor != 0) { set_error("bitblas_b200 is built for sm_90a (H100, compute capability 9.0), found %d.%d", major, minor); return 2; }
  int n = 0;
  BB_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device));
  if (device < BB_MAX_DEVICES && n > 0) g_sm_count[device].store(n);
  tensor_map_encoder();   // the TMA kernels report a missing entry point at launch
  return 0;
}

int bb_select_kernel(const bb_matmul_desc* desc, int m) {
  if (validate(desc)) return -1;
  return select(*desc, m);
}

const char* bb_kernel_name(int id) {
  switch (id) {
    case BB_KERNEL_AUTO: return "auto";
    case BB_KERNEL_GENERIC: return "generic_simt";
    case BB_KERNEL_GEMV_MMA: return "gemv_mma";
    case BB_KERNEL_GEMV_I8: return "gemv_i8";
    case BB_KERNEL_GEMM_TS: return "gemm_ts_wgmma";
    case BB_KERNEL_GEMM_TS_I8: return "gemm_ts_wgmma_i8";
    case BB_KERNEL_GEMV_SLAB: return "gemv_slab";
    case BB_KERNEL_GEMM_FP8: return "gemm_fp8_wgmma";
  }
  return "unknown";
}

int bb_set_kernel_override(int id) { return g_override.exchange(id); }

int bb_set_sm_count_cap(int cap) {
  // a cap above the real count would launch grids larger than what is resident at once, and the slab kernel's collectors spin on
  // slots written by other CTAs of their own grid
  const int n = device_sm_count_uncapped();
  if (cap < 0 || cap > n) {
    set_error("bb_set_sm_count_cap: cap must be in [0, %d] (0 removes the cap; %d is this device's SM count), got %d", n, n, cap);
    return -1;
  }
  return g_sm_cap.exchange(cap);
}

size_t bb_workspace_bytes(const bb_matmul_desc* desc, int m) {
  if (validate(desc)) return 0;
  const int k = select(*desc, m);
  if (k == BB_KERNEL_GEMM_TS || k == BB_KERNEL_GEMM_TS_I8) return gemm_ts_workspace_bytes(*desc, m);
  if (k == BB_KERNEL_GEMV_SLAB) return gemv_slab_workspace_bytes();
  return 0;
}

// the gate/up interleave pairs 8 gate rows with 8 up rows in every 16-row block of W: N = 2I with I % 8 == 0
static bool swiglu_shape_ok(const bb_matmul_desc* desc) {
  if (desc && desc->N % 16) {
    set_error("SwiGLU: desc->N = 2I needs I %% 8 == 0 (gate/up interleave in blocks of 8 rows; N=%d)", desc->N);
    return false;
  }
  return true;
}

// the descriptor checks of bb_matmul_scaled on top of validate(): int8 activations, a 16- or 32-bit float output, no group scales or
// zeros (the weight's scale is w_scale)
static bool scaled_desc_ok(const bb_matmul_desc* desc) {
  if (desc->a_dtype != BB_I8) {
    set_error("bb_matmul_scaled: needs int8 activations (a_dtype=%d; quantize 16-bit ones with bb_quantize_act_int8)", desc->a_dtype);
    return false;
  }
  if (desc->out_dtype != BB_F16 && desc->out_dtype != BB_BF16 && desc->out_dtype != BB_F32) {
    set_error("bb_matmul_scaled: out_dtype must be float16, bfloat16 or float32 (got %d)", desc->out_dtype);
    return false;
  }
  if (desc->with_scaling) { set_error("bb_matmul_scaled: group scales are not supported (with_scaling must be 0; pass w_scale)"); return false; }
  if (desc->with_zeros) { set_error("bb_matmul_scaled: zero points are not supported (with_zeros must be 0)"); return false; }
  return true;
}

// the descriptor checks of bb_matmul_w4a8 on top of validate(), in the order of scaled_desc_ok
static bool w4a8_desc_ok(const bb_matmul_desc* desc) {
  if (desc->a_dtype != BB_I8) {
    set_error("bb_matmul_w4a8: needs int8 activations (a_dtype=%d; quantize 16-bit ones with bb_quantize_act_int8)", desc->a_dtype);
    return false;
  }
  if (desc->out_dtype != BB_F16 && desc->out_dtype != BB_BF16 && desc->out_dtype != BB_F32) {
    set_error("bb_matmul_w4a8: out_dtype must be float16, bfloat16 or float32 (got %d)", desc->out_dtype);
    return false;
  }
  if (!desc->with_scaling) { set_error("bb_matmul_w4a8: needs with_scaling = 1 (fp32 group scales [N, K/g])"); return false; }
  if (desc->with_zeros && desc->zeros_mode != BB_ZEROS_QUANTIZED) {
    set_error("bb_matmul_w4a8: zero points must be BB_ZEROS_QUANTIZED (packed [K/g, N/2]; got zeros_mode=%d)", desc->zeros_mode);
    return false;
  }
  if (desc->w_bits != 4 || (desc->w_fmt != BB_W_UINT && desc->w_fmt != BB_W_INT)) {
    set_error("bb_matmul_w4a8: needs 4-bit uint or int weights (w_bits=%d, w_fmt=%d)", desc->w_bits, desc->w_fmt);
    return false;
  }
  if (desc->with_zeros && desc->w_fmt == BB_W_INT) { set_error("bb_matmul_w4a8: int weights take no zero points"); return false; }
  return true;
}

// bb_matmul_w4a8's kernel: the family select() picks for the descriptor without group scales and zeros (so its workspace is
// bb_workspace_bytes of that descriptor), with gemv_i8 and gemm_ts_i8 replaced by generic_simt when g is not a multiple of 128
// (their 128-k steps and k-blocks must not straddle a group); under a kernel override forcing one of the two, such a g is not
// supported (-1)
static int select_w4a8(const bb_matmul_desc& d, int m) {
  bb_matmul_desc c = d;
  c.with_scaling = c.with_zeros = 0;
  const int k = select(c, m);
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if ((k == BB_KERNEL_GEMV_I8 || k == BB_KERNEL_GEMM_TS_I8) && g % 128)
    return g_override.load() == BB_KERNEL_AUTO ? BB_KERNEL_GENERIC : -1;
  return k;
}

// scaled: the scales of the Scaled and W4A8 forms (null in the other two)
static int matmul_impl(MatmulForm form, const ScaledArgs& scaled, const bb_matmul_desc* desc, const void* A, const void* W,
                       const void* lut, const void* scale, const void* zeros, const void* bias, void* C, void* const* peer_C,
                       int n_peers, long long ldc, long long col_offset, int m, void* workspace, size_t workspace_bytes,
                       void* stream) {
  if (validate(desc)) return 1;
  if (form == MatmulForm::SwiGLU) {
    if (desc->a_dtype == BB_I8) { set_error("bb_matmul_swiglu: int8 activations are not supported (float16 | bfloat16)"); return 1; }
    if (!swiglu_shape_ok(desc)) return 1;
  }
  if (form == MatmulForm::Scaled && !scaled_desc_ok(desc)) return 1;
  if (form == MatmulForm::W4A8 && !w4a8_desc_ok(desc)) return 1;
  if (m == 0) return 0;  // wrapper/tl.py:156-157
  if (m < 0) { set_error("m must be >= 0 (got %d)", m); return 1; }
  if (!A || !W || (!C && n_peers == 0)) { set_error("A, W and C must be non-null"); return 1; }
  if (form == MatmulForm::W4A8) {
    if (!scaled.a_scale) { set_error("bb_matmul_w4a8: a_scale must be non-null (fp32 [m], one scale per row of A)"); return 1; }
    if (!scaled.w_scale) { set_error("bb_matmul_w4a8: scale must be non-null (fp32 [N, K/g] group scales)"); return 1; }
    if ((reinterpret_cast<uintptr_t>(scaled.a_scale) & 3) || (reinterpret_cast<uintptr_t>(scaled.w_scale) & 3)) {
      set_error("bb_matmul_w4a8: a_scale and scale must be 4-byte aligned");
      return 5;
    }
  } else if (form == MatmulForm::Scaled) {
    if (!scaled.a_scale) { set_error("bb_matmul_scaled: a_scale must be non-null (fp32 [m], one scale per row of A)"); return 1; }
    if (!scaled.w_scale) { set_error("bb_matmul_scaled: w_scale must be non-null (fp32 [N], one scale per output column)"); return 1; }
    if ((reinterpret_cast<uintptr_t>(scaled.a_scale) & 3) || (reinterpret_cast<uintptr_t>(scaled.w_scale) & 3)) {
      set_error("bb_matmul_scaled: a_scale and w_scale must be 4-byte aligned");
      return 5;
    }
  }
  if (n_peers < 0 || n_peers > BB_MAX_PEERS) { set_error("n_peers must be in [0, %d]", BB_MAX_PEERS); return 1; }
  if (n_peers > 0) {
    if (!peer_C) { set_error("peer_C is null"); return 1; }
    for (int i = 0; i < n_peers; ++i) if (!peer_C[i]) { set_error("peer_C[%d] is null", i); return 1; }
    if (col_offset < 0 || col_offset + desc->N > ldc) { set_error("column shard [%lld, %lld) exceeds ldc=%lld", col_offset, col_offset + desc->N, ldc); return 1; }
  }
  if (desc->with_scaling && !scale) { set_error("with_scaling is set but scale is null"); return 1; }
  if (desc->with_zeros && !zeros) { set_error("with_zeros is set but zeros is null"); return 1; }
  if (desc->with_bias && !bias) { set_error("with_bias is set but bias is null"); return 1; }
  if (desc->w_fmt == BB_W_NF && !lut) { set_error("nf4 weights need the 16-entry LUT"); return 1; }
  MatmulArgs a;
  a.d = *desc; a.A = A; a.W = W; a.lut = lut; a.scale = scale; a.zeros = zeros; a.bias = bias; a.C = C; a.m = m;
  a.n_peers = n_peers; a.ldc = n_peers ? ldc : desc->N; a.col_offset = n_peers ? col_offset : 0;
  for (int i = 0; i < BB_MAX_PEERS; ++i) a.peer_C[i] = (i < n_peers) ? peer_C[i] : nullptr;
  a.workspace = workspace; a.workspace_bytes = workspace_bytes; a.stream = (cudaStream_t)stream;
  a.form = form;
  a.scaled = scaled;
  const int k = form == MatmulForm::W4A8 ? select_w4a8(a.d, m) : select(a.d, m);
  if (n_peers > 0 && k == BB_KERNEL_GENERIC) {
    set_error("the column-parallel scatter epilogue needs a fast kernel (gemv_mma / gemv_i8 / gemm_ts); this configuration dispatches to generic_simt");
    return 1;
  }
  switch (k) {
    case BB_KERNEL_GENERIC: return launch_generic(a);
    case BB_KERNEL_GEMV_MMA: return launch_gemv_mma(a);
    case BB_KERNEL_GEMV_I8: return launch_gemv_i8(a);
    case BB_KERNEL_GEMV_SLAB: return launch_gemv_slab(a);
    case BB_KERNEL_GEMM_TS:
    case BB_KERNEL_GEMM_TS_I8: return launch_gemm_ts(a);
  }
  set_error("kernel override %d does not support this configuration", g_override.load());
  return 1;
}

int bb_matmul(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
              const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes,
              void* stream) {
  return matmul_impl(MatmulForm::Plain, {}, desc, A, W, lut, scale, zeros, bias, C, nullptr, 0, 0, 0, m, workspace, workspace_bytes,
                     stream);
}

int bb_matmul_swiglu(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                     const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes,
                     void* stream) {
  return matmul_impl(MatmulForm::SwiGLU, {}, desc, A, W, lut, scale, zeros, bias, C, nullptr, 0, 0, 0, m, workspace, workspace_bytes,
                     stream);
}

int bb_matmul_scaled(const bb_matmul_desc* desc, const void* A, const void* W, const float* a_scale, const float* w_scale,
                     const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream) {
  return matmul_impl(MatmulForm::Scaled, {a_scale, w_scale}, desc, A, W, nullptr, nullptr, nullptr, bias, C, nullptr, 0, 0, 0, m,
                     workspace, workspace_bytes, stream);
}

int bb_matmul_w4a8(const bb_matmul_desc* desc, const void* A, const void* W, const float* a_scale, const float* scale,
                   const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream) {
  return matmul_impl(MatmulForm::W4A8, {a_scale, scale}, desc, A, W, nullptr, scale, zeros, bias, C, nullptr, 0, 0, 0, m, workspace,
                     workspace_bytes, stream);
}

int bb_select_kernel_w4a8(const bb_matmul_desc* desc, int m) {
  if (validate(desc) || !w4a8_desc_ok(desc)) return -1;
  return select_w4a8(*desc, m);
}

// the descriptor of bb_matmul_fp8 (validate() is not run: it refuses a_dtype = BB_E4M3, as every other entry point does)
static bool fp8_desc_ok(const bb_matmul_desc* d) {
  if (!d) { set_error("null descriptor"); return false; }
  if (d->a_dtype != BB_E4M3) {
    set_error("bb_matmul_fp8: needs e4m3 activations (a_dtype=%d; quantize 16-bit ones with bb_quantize_act_fp8)", d->a_dtype);
    return false;
  }
  if (d->w_fmt != BB_W_FP8_E4M3 || d->w_bits != 8) {
    set_error("bb_matmul_fp8: needs e4m3 weights (w_fmt=%d, w_bits=%d; want BB_W_FP8_E4M3, 8)", d->w_fmt, d->w_bits);
    return false;
  }
  if (d->accum_dtype != BB_F32) { set_error("bb_matmul_fp8: accum_dtype must be float32 (got %d)", d->accum_dtype); return false; }
  if (d->out_dtype != BB_F16 && d->out_dtype != BB_BF16 && d->out_dtype != BB_F32) {
    set_error("bb_matmul_fp8: out_dtype must be float16, bfloat16 or float32 (got %d)", d->out_dtype);
    return false;
  }
  if (d->group_size != 128) { set_error("bb_matmul_fp8: group_size must be 128 (128 x 128 scale blocks; got %d)", d->group_size); return false; }
  if (d->with_scaling != 1) { set_error("bb_matmul_fp8: needs with_scaling = 1 (fp32 block scales)"); return false; }
  if (d->with_zeros) { set_error("bb_matmul_fp8: zero points are not supported (with_zeros must be 0)"); return false; }
  if (d->w_layout != BB_LAYOUT_COMPRESSED || d->w_tile != BB_TILE_ROW_MAJOR) {
    set_error("bb_matmul_fp8: W must be row-major compressed storage (w_layout=%d, w_tile=%d)", d->w_layout, d->w_tile);
    return false;
  }
  if (d->reserved[0] || d->reserved[1]) { set_error("reserved fields must be zero"); return false; }
  if (d->N <= 0 || d->N % 16) { set_error("bb_matmul_fp8: needs N > 0 and N %% 16 == 0 (N=%d)", d->N); return false; }
  if (d->K <= 0 || d->K % 128) { set_error("bb_matmul_fp8: needs K > 0 and K %% 128 == 0 (K=%d)", d->K); return false; }
  return true;
}

static int select_fp8(int m) {
  const int ov = g_override.load();
  return m >= 1 && (ov == BB_KERNEL_AUTO || ov == BB_KERNEL_GEMM_FP8) ? BB_KERNEL_GEMM_FP8 : -1;
}

int bb_matmul_fp8(const bb_matmul_desc* desc, const void* A, const float* a_scale, int a_scale_ld, const void* W,
                  const float* w_scale, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream) {
  if (!fp8_desc_ok(desc)) return 1;
  if (m == 0) return 0;
  if (m < 0) { set_error("m must be >= 0 (got %d)", m); return 1; }
  if (a_scale_ld < m || a_scale_ld % 4) {
    set_error("bb_matmul_fp8: a_scale_ld must be >= m and a multiple of 4 (a_scale_ld=%d, m=%d)", a_scale_ld, m);
    return 1;
  }
  if (!A || !W || !C) { set_error("A, W and C must be non-null"); return 1; }
  if (!a_scale) { set_error("bb_matmul_fp8: a_scale must be non-null (fp32 [K/128][a_scale_ld], k-block-major)"); return 1; }
  if (!w_scale) { set_error("bb_matmul_fp8: w_scale must be non-null (fp32 [ceil(N/128), K/128])"); return 1; }
  if (desc->with_bias && !bias) { set_error("with_bias is set but bias is null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15)) {
    set_error("bb_matmul_fp8: A and W must be 16-byte aligned");
    return 5;
  }
  if (reinterpret_cast<uintptr_t>(a_scale) & 15) { set_error("bb_matmul_fp8: a_scale must be 16-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(w_scale) & 3) { set_error("bb_matmul_fp8: w_scale must be 4-byte aligned"); return 5; }
  if (select_fp8(m) < 0) {
    set_error("bb_matmul_fp8: kernel override %d does not support this entry (AUTO or BB_KERNEL_GEMM_FP8)", g_override.load());
    return 1;
  }
  Fp8Args a;
  a.d = *desc; a.A = A; a.a_scale = a_scale; a.a_scale_ld = a_scale_ld; a.W = W; a.w_scale = w_scale;
  a.bias = desc->with_bias ? bias : nullptr; a.C = C; a.m = m;
  a.workspace = workspace; a.workspace_bytes = workspace ? workspace_bytes : 0; a.stream = (cudaStream_t)stream;
  return launch_gemm_fp8(a);
}

int bb_select_kernel_fp8(const bb_matmul_desc* desc, int m) {
  if (!fp8_desc_ok(desc)) return -1;
  return select_fp8(m);
}

size_t bb_workspace_bytes_fp8(const bb_matmul_desc* desc, int m) {
  if (!fp8_desc_ok(desc) || select_fp8(m) < 0) return 0;
  return gemm_fp8_workspace_bytes(*desc, m);
}

// bb_matmul_grouped_fp8[_swiglu]: every rejection has its own message and code, so the order of the checks is part of the interface
static int grouped_fp8_call(bool swiglu, const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A,
                            const float* a_scale, int a_scale_ld, const void* W, const float* w_scale, void* C, int total_rows,
                            void* stream) {
  if (!fp8_desc_ok(desc)) return 1;
  if (desc->N % 128) {
    if (swiglu) set_error("grouped FP8 SwiGLU: desc->N = 2I needs 2I %% 128 == 0 (N=%d)", desc->N);
    else set_error("grouped FP8: needs N %% 128 == 0 (an expert's 128-row tile must not read the next expert's rows; N=%d)", desc->N);
    return 1;
  }
  if (desc->with_bias) { set_error("grouped FP8: with_bias must be 0 (expert biases are not supported)"); return 1; }
  if (num_groups < 1 || num_groups > BB_GROUPED_MAX_GROUPS) {
    set_error("num_groups must be in [1, %d] (got %d)", BB_GROUPED_MAX_GROUPS, num_groups);
    return 1;
  }
  if (total_rows < 0) { set_error("total_rows must be >= 0 (got %d)", total_rows); return 1; }
  if (total_rows == 0) return 0;
  if (a_scale_ld < total_rows || a_scale_ld % 4) {
    set_error("grouped FP8: a_scale_ld must be >= total_rows and a multiple of 4 (a_scale_ld=%d, total_rows=%d)", a_scale_ld,
              total_rows);
    return 1;
  }
  if (!offsets) { set_error("offsets must be a device pointer to num_groups + 1 int32 values"); return 1; }
  if (!A || !W || !C) { set_error("A, W and C must be non-null"); return 1; }
  if (!a_scale) { set_error("grouped FP8: a_scale must be non-null (fp32 [K/128][a_scale_ld], k-block-major)"); return 1; }
  if (!w_scale) { set_error("grouped FP8: w_scale must be non-null (fp32 [E, N/128, K/128])"); return 1; }
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15)) {
    set_error("grouped FP8: A and W must be 16-byte aligned");
    return 5;
  }
  if (reinterpret_cast<uintptr_t>(a_scale) & 15) { set_error("grouped FP8: a_scale must be 16-byte aligned"); return 5; }
  if ((reinterpret_cast<uintptr_t>(w_scale) & 3) || (reinterpret_cast<uintptr_t>(offsets) & 3)) {
    set_error("grouped FP8: w_scale and offsets must be 4-byte aligned");
    return 5;
  }
  if (select_fp8(total_rows) < 0) {
    set_error("grouped FP8: kernel override %d does not support this entry (AUTO or BB_KERNEL_GEMM_FP8)", g_override.load());
    return 1;
  }
  GroupedFp8Args a;
  a.d = *desc; a.num_groups = num_groups; a.offsets = offsets; a.A = A; a.a_scale = a_scale; a.a_scale_ld = a_scale_ld;
  a.W = W; a.w_scale = w_scale; a.C = C; a.total_rows = total_rows; a.stream = (cudaStream_t)stream; a.swiglu = swiglu;
  return launch_grouped_fp8(a);
}

int bb_matmul_grouped_fp8(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const float* a_scale,
                          int a_scale_ld, const void* W, const float* w_scale, void* C, int total_rows, void* stream) {
  return grouped_fp8_call(false, desc, num_groups, offsets, A, a_scale, a_scale_ld, W, w_scale, C, total_rows, stream);
}

int bb_matmul_grouped_fp8_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A,
                                 const float* a_scale, int a_scale_ld, const void* W, const float* w_scale, void* C, int total_rows,
                                 void* stream) {
  return grouped_fp8_call(true, desc, num_groups, offsets, A, a_scale, a_scale_ld, W, w_scale, C, total_rows, stream);
}

int bb_matmul_scatter(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                      const void* zeros, const void* bias, void* const* peer_C, int n_peers, int64_t ldc,
                      int64_t col_offset, int m, void* workspace, size_t workspace_bytes, void* stream) {
  if (n_peers < 1) { set_error("bb_matmul_scatter needs n_peers >= 1"); return 1; }
  return matmul_impl(MatmulForm::Plain, {}, desc, A, W, lut, scale, zeros, bias, nullptr, peer_C, n_peers, ldc, col_offset, m, workspace,
                     workspace_bytes, stream);
}

// the grouped entry points: gemm picks the grouped wgmma GEMM instead of the grouped GEMV, swiglu the fused gate/up epilogue,
// gather (GEMM with swiglu) the A rows through row_index.  Every rejection has its own message and code, so the order of the
// checks is part of the interface.
static int grouped_call(bool gemm, bool swiglu, bool gather, const bb_matmul_desc* desc, int num_groups, const int32_t* offsets,
                        const int32_t* row_index, const void* A, int a_rows, const void* W, const void* scale, const void* zeros,
                        const void* bias, void* C, int total_rows, void* stream) {
  if (validate(desc)) return 1;
  if (swiglu && !swiglu_shape_ok(desc)) return 1;
  if (!(gemm ? grouped_gemm_supported(*desc) : grouped_supported(*desc))) return 1;
  if (num_groups < 1 || num_groups > BB_GROUPED_MAX_GROUPS) {
    set_error("num_groups must be in [1, %d] (got %d)", BB_GROUPED_MAX_GROUPS, num_groups);
    return 1;
  }
  if (total_rows < 0) { set_error("total_rows must be >= 0 (got %d)", total_rows); return 1; }
  if (total_rows == 0) return 0;
  if (!offsets) { set_error("offsets must be a device pointer to num_groups + 1 int32 values"); return 1; }
  if (!A || !W || !C) { set_error("A, W and C must be non-null"); return 1; }
  if (desc->with_scaling && !scale) { set_error("with_scaling is set but scale is null"); return 1; }
  if (desc->with_zeros && !zeros) { set_error("with_zeros is set but zeros is null"); return 1; }
  if (desc->with_bias && !bias) { set_error("with_bias is set but bias is null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15) || (reinterpret_cast<uintptr_t>(offsets) & 3)) {
    set_error("grouped matmul: A and W must be 16-byte aligned, offsets 4-byte aligned");
    return 5;
  }
  if (gather) {
    if (!row_index) { set_error("gather: row_index must be a device pointer to total_rows int32 values"); return 1; }
    if (a_rows < 1) { set_error("gather: a_rows must be >= 1 (got %d)", a_rows); return 1; }
    if (reinterpret_cast<uintptr_t>(row_index) & 3) { set_error("gather: row_index must be 4-byte aligned"); return 5; }
  }
  GroupedArgs g;
  g.d = *desc; g.num_groups = num_groups; g.offsets = offsets; g.A = A; g.W = W; g.scale = scale; g.zeros = zeros; g.bias = bias;
  g.C = C; g.total_rows = total_rows; g.stream = (cudaStream_t)stream;
  g.swiglu = swiglu; g.row_index = row_index; g.a_rows = a_rows;
  // the stacked parameters: W [E, N, K * bits / 8], scale [E, N, G], zeros [E, N, G] ([E, G, N * bits / 8] quantized), bias [E, N]
  const long long N = desc->N, G = desc->K / (desc->group_size <= 0 ? desc->K : desc->group_size);
  g.w_stride = N * desc->K * desc->w_bits / 8;
  g.s_stride = N * G * 2;
  g.z_stride = desc->zeros_mode == BB_ZEROS_QUANTIZED ? G * (N * desc->w_bits / 8) : N * G * 2;
  g.b_stride = N * 2;
  return gemm ? launch_grouped_gemm(g) : launch_grouped(g);
}

int bb_matmul_grouped(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                      const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream) {
  return grouped_call(false, false, false, desc, num_groups, offsets, nullptr, A, 0, W, scale, zeros, bias, C, total_rows, stream);
}

int bb_matmul_grouped_gemm(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                           const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream) {
  return grouped_call(true, false, false, desc, num_groups, offsets, nullptr, A, 0, W, scale, zeros, bias, C, total_rows, stream);
}

int bb_matmul_grouped_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                             const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream) {
  return grouped_call(false, true, false, desc, num_groups, offsets, nullptr, A, 0, W, scale, zeros, bias, C, total_rows, stream);
}

int bb_matmul_grouped_gemm_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                                  const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream) {
  return grouped_call(true, true, false, desc, num_groups, offsets, nullptr, A, 0, W, scale, zeros, bias, C, total_rows, stream);
}

int bb_matmul_grouped_gemm_swiglu_gather(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets,
                                         const int32_t* row_index, const void* A, int a_rows, const void* W, const void* scale,
                                         const void* zeros, const void* bias, void* C, int total_rows, void* stream) {
  return grouped_call(true, true, true, desc, num_groups, offsets, row_index, A, a_rows, W, scale, zeros, bias, C, total_rows,
                      stream);
}

// the checks bb_moe_route and bb_moe_route_index share: 0 = valid
static int check_route_args(int num_tokens, int top_k, int num_experts) {
  if (num_experts < 1 || num_experts > BB_GROUPED_MAX_GROUPS) {
    set_error("moe route: num_experts must be in [1, %d] (got %d)", BB_GROUPED_MAX_GROUPS, num_experts);
    return 1;
  }
  if (top_k < 1) { set_error("moe route: top_k must be >= 1 (got %d)", top_k); return 1; }
  if (num_tokens < 0) { set_error("moe route: num_tokens must be >= 0 (got %d)", num_tokens); return 1; }
  if ((long long)num_tokens * top_k > INT_MAX) {
    set_error("moe route: num_tokens * top_k must be below 2^31 (got %d x %d)", num_tokens, top_k);
    return 1;
  }
  return 0;
}

int bb_moe_route(const int32_t* topk_ids, int num_tokens, int top_k, int num_experts, const void* x, int a_dtype, int K,
                 int32_t* offsets, int32_t* slot_rows, void* x_sorted, void* stream) {
  if (check_route_args(num_tokens, top_k, num_experts)) return 1;
  if (a_dtype != BB_F16 && a_dtype != BB_BF16) { set_error("moe route: x must be float16 or bfloat16 (a_dtype=%d)", a_dtype); return 1; }
  if (K <= 0 || K % 8) { set_error("moe route: needs K > 0 and K %% 8 == 0 (K=%d)", K); return 1; }
  if (num_tokens == 0) return 0;
  if (!topk_ids || !x || !offsets || !slot_rows || !x_sorted) { set_error("moe route: every pointer must be non-null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(x_sorted) & 15) ||
      (reinterpret_cast<uintptr_t>(topk_ids) & 3) || (reinterpret_cast<uintptr_t>(offsets) & 3) ||
      (reinterpret_cast<uintptr_t>(slot_rows) & 3)) {
    set_error("moe route: x and x_sorted must be 16-byte aligned, the int32 arrays 4-byte aligned");
    return 5;
  }
  return launch_moe_route(topk_ids, num_tokens * top_k, top_k, num_experts, x, K, offsets, slot_rows, x_sorted, nullptr,
                          (cudaStream_t)stream);
}

int bb_moe_route_index(const int32_t* topk_ids, int num_tokens, int top_k, int num_experts, int32_t* offsets,
                       int32_t* slot_rows, int32_t* row_token, void* stream) {
  if (check_route_args(num_tokens, top_k, num_experts)) return 1;
  if (num_tokens == 0) return 0;
  if (!topk_ids || !offsets || !slot_rows || !row_token) { set_error("moe route: every pointer must be non-null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(topk_ids) & 3) || (reinterpret_cast<uintptr_t>(offsets) & 3) ||
      (reinterpret_cast<uintptr_t>(slot_rows) & 3) || (reinterpret_cast<uintptr_t>(row_token) & 3)) {
    set_error("moe route: the int32 arrays must be 4-byte aligned");
    return 5;
  }
  return launch_moe_route(topk_ids, num_tokens * top_k, top_k, num_experts, nullptr, 8, offsets, slot_rows, nullptr, row_token,
                          (cudaStream_t)stream);
}

int bb_moe_combine(const int32_t* slot_rows, const float* topk_weights, const void* Y, int out_dtype, void* out, int num_tokens,
                   int top_k, int N, void* stream) {
  if (top_k < 1) { set_error("moe combine: top_k must be >= 1 (got %d)", top_k); return 1; }
  if (num_tokens < 0) { set_error("moe combine: num_tokens must be >= 0 (got %d)", num_tokens); return 1; }
  if ((long long)num_tokens * top_k > INT_MAX) {
    set_error("moe combine: num_tokens * top_k must be below 2^31 (got %d x %d)", num_tokens, top_k);
    return 1;
  }
  if (out_dtype != BB_F16 && out_dtype != BB_BF16 && out_dtype != BB_F32) {
    set_error("moe combine: out_dtype must be float16, bfloat16 or float32 (got %d)", out_dtype);
    return 1;
  }
  if (N <= 0 || N % 8) { set_error("moe combine: needs N > 0 and N %% 8 == 0 (N=%d)", N); return 1; }
  if (num_tokens == 0) return 0;
  if (!slot_rows || !topk_weights || !Y || !out) { set_error("moe combine: every pointer must be non-null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(Y) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(slot_rows) & 3) || (reinterpret_cast<uintptr_t>(topk_weights) & 3)) {
    set_error("moe combine: Y and out must be 16-byte aligned, slot_rows and topk_weights 4-byte aligned");
    return 5;
  }
  return launch_moe_combine(slot_rows, topk_weights, Y, out_dtype, out, num_tokens, top_k, N, (cudaStream_t)stream);
}

int bb_moe_topk(const void* logits, int logits_dtype, int num_tokens, int num_experts, int top_k, int scoring,
                const float* correction_bias, int num_expert_group, int topk_group, int group_score, int renormalize,
                float routed_scaling_factor, int32_t* topk_ids, float* topk_weights, void* stream) {
  if (logits_dtype != BB_F16 && logits_dtype != BB_BF16 && logits_dtype != BB_F32) {
    set_error("moe topk: logits must be float16, bfloat16 or float32 (logits_dtype=%d)", logits_dtype);
    return 1;
  }
  if (num_experts < 1 || num_experts > BB_GROUPED_MAX_GROUPS) {
    set_error("moe topk: num_experts must be in [1, %d] (got %d)", BB_GROUPED_MAX_GROUPS, num_experts);
    return 1;
  }
  if (top_k < 1 || top_k > std::min(num_experts, 32)) {
    set_error("moe topk: top_k must be in [1, min(num_experts, 32) = %d] (got %d)", std::min(num_experts, 32), top_k);
    return 1;
  }
  if (num_tokens < 0) { set_error("moe topk: num_tokens must be >= 0 (got %d)", num_tokens); return 1; }
  if ((long long)num_tokens * top_k > INT_MAX) {
    set_error("moe topk: num_tokens * top_k must be below 2^31 (got %d x %d)", num_tokens, top_k);
    return 1;
  }
  if (scoring != 0 && scoring != 1) { set_error("moe topk: scoring must be 0 (softmax) or 1 (sigmoid) (got %d)", scoring); return 1; }
  if (num_expert_group > 1) {
    const int n = num_expert_group;
    if (n > 32) { set_error("moe topk: num_expert_group must be <= 32 (got %d)", n); return 1; }
    if (num_experts % n) {
      set_error("moe topk: num_expert_group (%d) must divide num_experts (%d)", n, num_experts);
      return 1;
    }
    if (topk_group < 1 || topk_group > n) {
      set_error("moe topk: topk_group must be in [1, num_expert_group = %d] (got %d)", n, topk_group);
      return 1;
    }
    if (group_score != 0 && group_score != 1) {
      set_error("moe topk: group_score must be 0 (max) or 1 (top2_sum) (got %d)", group_score);
      return 1;
    }
    if (group_score == 1 && num_experts / n < 2) {
      set_error("moe topk: top2_sum needs at least 2 experts per group (num_experts / num_expert_group = %d)", num_experts / n);
      return 1;
    }
    if (top_k > topk_group * (num_experts / n)) {
      set_error("moe topk: top_k (%d) exceeds the %d experts of the topk_group kept groups", top_k, topk_group * (num_experts / n));
      return 1;
    }
  }
  if (!std::isfinite(routed_scaling_factor)) {
    set_error("moe topk: routed_scaling_factor must be finite (got %g)", (double)routed_scaling_factor);
    return 1;
  }
  if (num_tokens == 0) {   // counted like a launching call: every accepted call is one step of bb_launch_count
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return 0;
  }
  if (!logits) { set_error("moe topk: logits must be non-null"); return 1; }
  if (!topk_ids) { set_error("moe topk: topk_ids must be non-null"); return 1; }
  if (!topk_weights) { set_error("moe topk: topk_weights must be non-null"); return 1; }
  const uintptr_t elem = logits_dtype == BB_F32 ? 4 : 2;
  if (reinterpret_cast<uintptr_t>(logits) & (elem - 1)) {
    set_error("moe topk: logits must be aligned to their element size (%d bytes)", int(elem));
    return 5;
  }
  if (reinterpret_cast<uintptr_t>(topk_ids) & 3) { set_error("moe topk: topk_ids must be 4-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(topk_weights) & 3) { set_error("moe topk: topk_weights must be 4-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(correction_bias) & 3) { set_error("moe topk: correction_bias must be 4-byte aligned"); return 5; }
  return launch_moe_topk(logits, logits_dtype, num_tokens, num_experts, top_k, scoring, correction_bias, num_expert_group,
                         topk_group, group_score, renormalize, routed_scaling_factor, topk_ids, topk_weights,
                         (cudaStream_t)stream);
}

int bb_permute_cols(const void* A, void* out, const int32_t* perm, int rows, int K, int a_dtype, int num_groups,
                    const int32_t* offsets, void* stream) {
  if (a_dtype != BB_F16 && a_dtype != BB_BF16) { set_error("permute cols: A must be float16 or bfloat16 (a_dtype=%d)", a_dtype); return 1; }
  if (K <= 0 || K % 8) { set_error("permute cols: needs K > 0 and K %% 8 == 0 (K=%d)", K); return 1; }
  if (K > PERMUTE_MAX_K) { set_error("permute cols: K=%d exceeds %d (one row is staged in shared memory)", K, PERMUTE_MAX_K); return 1; }
  if (num_groups < 1 || num_groups > BB_GROUPED_MAX_GROUPS) {
    set_error("permute cols: num_groups must be in [1, %d] (got %d)", BB_GROUPED_MAX_GROUPS, num_groups);
    return 1;
  }
  if (num_groups > 1 && !offsets) { set_error("permute cols: num_groups > 1 needs offsets (a device pointer to num_groups + 1 int32 values)"); return 1; }
  if (rows < 0) { set_error("permute cols: rows must be >= 0 (got %d)", rows); return 1; }
  if (rows == 0) return 0;
  if (!A || !out || !perm) { set_error("permute cols: A, out and perm must be non-null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) {
    set_error("permute cols: A and out must be 16-byte aligned");
    return 5;
  }
  if ((reinterpret_cast<uintptr_t>(perm) & 3) || (reinterpret_cast<uintptr_t>(offsets) & 3)) {
    set_error("permute cols: perm and offsets must be 4-byte aligned");
    return 5;
  }
  return launch_permute_cols(A, out, perm, rows, K, num_groups, offsets, (cudaStream_t)stream);
}

int bb_quantize_act_int8(const void* x, int a_dtype, int rows, int K, int8_t* q, float* scale, void* stream) {
  if (a_dtype != BB_F16 && a_dtype != BB_BF16) { set_error("quantize act int8: x must be float16 or bfloat16 (a_dtype=%d)", a_dtype); return 1; }
  if (K <= 0 || K % 8) { set_error("quantize act int8: needs K > 0 and K %% 8 == 0 (K=%d)", K); return 1; }
  if (rows < 0) { set_error("quantize act int8: rows must be >= 0 (got %d)", rows); return 1; }
  if (rows == 0) return 0;
  if (!x) { set_error("quantize act int8: x must be non-null"); return 1; }
  if (!q) { set_error("quantize act int8: q must be non-null"); return 1; }
  if (!scale) { set_error("quantize act int8: scale must be non-null"); return 1; }
  if (reinterpret_cast<uintptr_t>(x) & 15) { set_error("quantize act int8: x must be 16-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(q) & 15) { set_error("quantize act int8: q must be 16-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(scale) & 3) { set_error("quantize act int8: scale must be 4-byte aligned"); return 5; }
  return launch_quantize_act_int8(x, a_dtype, rows, K, q, scale, (cudaStream_t)stream);
}

int bb_quantize_act_fp8(const void* x, int a_dtype, int rows, int K, void* q, float* scale, int scale_ld, void* stream) {
  if (a_dtype != BB_F16 && a_dtype != BB_BF16) { set_error("quantize act fp8: x must be float16 or bfloat16 (a_dtype=%d)", a_dtype); return 1; }
  if (K <= 0 || K % 128) { set_error("quantize act fp8: needs K > 0 and K %% 128 == 0 (K=%d)", K); return 1; }
  if (rows < 0) { set_error("quantize act fp8: rows must be >= 0 (got %d)", rows); return 1; }
  if (scale_ld < rows || scale_ld % 4) {
    set_error("quantize act fp8: scale_ld must be >= rows and a multiple of 4 (scale_ld=%d, rows=%d)", scale_ld, rows);
    return 1;
  }
  if (rows == 0) return 0;
  if (!x) { set_error("quantize act fp8: x must be non-null"); return 1; }
  if (!q) { set_error("quantize act fp8: q must be non-null"); return 1; }
  if (!scale) { set_error("quantize act fp8: scale must be non-null"); return 1; }
  if (reinterpret_cast<uintptr_t>(x) & 15) { set_error("quantize act fp8: x must be 16-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(q) & 15) { set_error("quantize act fp8: q must be 16-byte aligned"); return 5; }
  if (reinterpret_cast<uintptr_t>(scale) & 15) { set_error("quantize act fp8: scale must be 16-byte aligned"); return 5; }
  return launch_quantize_act_fp8(x, a_dtype, rows, K, static_cast<uint8_t*>(q), scale, scale_ld, (cudaStream_t)stream);
}

int bb_peer_barrier(void* const* peer_flags, int n_peers, int rank, void* stream) {
  if (!peer_flags || n_peers < 1 || n_peers > BB_MAX_PEERS || rank < 0 || rank >= n_peers) {
    set_error("bb_peer_barrier: need 1 <= n_peers <= %d flag blocks and 0 <= rank < n_peers", BB_MAX_PEERS);
    return 1;
  }
  PeerBarrierArgs a;
  for (int i = 0; i < BB_MAX_PEERS; ++i) a.flags[i] = i < n_peers ? reinterpret_cast<uint32_t*>(peer_flags[i]) : nullptr;
  for (int i = 0; i < n_peers; ++i) if (!a.flags[i] || (reinterpret_cast<uintptr_t>(a.flags[i]) & 3)) { set_error("bb_peer_barrier: flag block %d is null or unaligned", i); return 1; }
  a.n = n_peers; a.rank = rank;
  return launch_pdl(peer_barrier_kernel, 1, 32, 0, (cudaStream_t)stream, true, a);
}

}  // extern "C"
