// bb_api.cu -- the C ABI (include/bitblas_b200.h): validation, kernel dispatch, error reporting.
//
// Dispatch mirrors the reference's run-time choice (bitblas/ops/general_matmul/tilelang/dequantize/
// matmul_dequantize.py:93-111: M < 8 -> SIMT GEMV, else MMA GEMM; and the per-opt_M if-chain emitted into
// `call`, bitblas/builder/wrapper/tl.py:278-300) but is keyed on the H100 regimes instead:
//   m <= 8   : memory-bound streaming kernels (bb_gemv.cu)
//   m  > 8   : wgmma tensor-core kernel (bb_gemm_ts.cu), split-K when the tile grid is smaller than the chip
//   anything the fast kernels do not cover: the generic SIMT kernel (bb_generic.cu).
#include <cstring>
#include <mutex>

#include "bb_common.cuh"

namespace bb {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_override{BB_KERNEL_AUTO};
static std::atomic<int> g_sm_count[BB_MAX_DEVICES];   // 0 = not queried yet; per-device state is keyed on the ordinal

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

int device_sm_count() {
  const int dev = current_device();
  int n = g_sm_count[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); n = 132; }
    g_sm_count[dev].store(n, std::memory_order_relaxed);
  }
  return n;
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
      case BB_KERNEL_GEMV_STREAMK: if (gemv_streamk_supported(d, m)) return ov; break;
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
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
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
  return gemm_ts_init(device);
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
    case BB_KERNEL_GEMV_STREAMK: return "gemv_streamk";
    case BB_KERNEL_GEMV_SLAB: return "gemv_slab";
  }
  return "unknown";
}

int bb_set_kernel_override(int id) { return g_override.exchange(id); }

size_t bb_workspace_bytes(const bb_matmul_desc* desc, int m) {
  if (validate(desc)) return 0;
  const int k = select(*desc, m);
  if (k == BB_KERNEL_GEMM_TS || k == BB_KERNEL_GEMM_TS_I8) return gemm_ts_workspace_bytes(*desc, m);
  if (k == BB_KERNEL_GEMV_STREAMK) return gemv_streamk_workspace_bytes();
  if (k == BB_KERNEL_GEMV_SLAB) return gemv_slab_workspace_bytes();
  return 0;
}

static int matmul_impl(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                       const void* zeros, const void* bias, void* C, void* const* peer_C, int n_peers, long long ldc,
                       long long col_offset, int m, void* workspace, size_t workspace_bytes, void* stream) {
  if (validate(desc)) return 1;
  if (m == 0) return 0;  // wrapper/tl.py:156-157
  if (m < 0) { set_error("m must be >= 0 (got %d)", m); return 1; }
  if (!A || !W || (!C && n_peers == 0)) { set_error("A, W and C must be non-null"); return 1; }
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
  const int k = select(a.d, m);
  if (n_peers > 0 && k == BB_KERNEL_GENERIC) {
    set_error("the column-parallel scatter epilogue needs a fast kernel (gemv_mma / gemv_i8 / gemm_ts); this configuration dispatches to generic_simt");
    return 1;
  }
  switch (k) {
    case BB_KERNEL_GENERIC: return launch_generic(a);
    case BB_KERNEL_GEMV_MMA: return launch_gemv_mma(a);
    case BB_KERNEL_GEMV_I8: return launch_gemv_i8(a);
    case BB_KERNEL_GEMV_STREAMK: return launch_gemv_streamk(a);
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
  return matmul_impl(desc, A, W, lut, scale, zeros, bias, C, nullptr, 0, 0, 0, m, workspace, workspace_bytes, stream);
}

int bb_matmul_scatter(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                      const void* zeros, const void* bias, void* const* peer_C, int n_peers, int64_t ldc,
                      int64_t col_offset, int m, void* workspace, size_t workspace_bytes, void* stream) {
  if (n_peers < 1) { set_error("bb_matmul_scatter needs n_peers >= 1"); return 1; }
  return matmul_impl(desc, A, W, lut, scale, zeros, bias, nullptr, peer_C, n_peers, ldc, col_offset, m, workspace,
                     workspace_bytes, stream);
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
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(1); cfg.blockDim = dim3(32); cfg.dynamicSmemBytes = 0; cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  BB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, peer_barrier_kernel, a));
  BB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
