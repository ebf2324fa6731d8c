// tools/slabbench.cu -- round-2 hypothesis test for the m = 1 weight stream (DESIGN.md 3.2): does the DRAM side care about the
// granularity / pacing of the per-row requests?  Pure TMA loads of the N x (K/2)-byte packed-weight matrix, no arithmetic, with an
// optional spin of `delay` cycles after every consumed tile to emulate compute pacing.
//   box   : every warp streams its own 16-row block with [16 rows x 128 B] boxes (2 KB), DEPTH boxes in flight   (= gemv_sk_kernel)
//   slab  : every CTA streams 16-row blocks with [16 rows x SLAB B] boxes (uint32 tensor map, SLAB = 512 / 1024), DEPTH slabs in
//           flight, the 8 warps of the CTA each "consume" a 128 B K-slice of the slab
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/slabbench tools/slabbench.cu -lcuda
// Run:   tools/slabbench [N] [K] [delay_cycles]
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const void* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void spin(int cycles) {
  if (cycles <= 0) return;
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}

// ---- per-warp 2 KB boxes (the stream-K kernel's pattern) ----
template <int DEPTH>
__global__ void __launch_bounds__(256, 2) k_box(const __grid_constant__ CUtensorMap tm, int row_blocks, int chunks_per_row, int delay, unsigned* out) {
  extern __shared__ uint8_t raw[];
  const uint32_t base = (smem_u32(raw) + 1023u) & ~1023u;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t ring = base + w * DEPTH * 2048, bars = base + 8 * DEPTH * 2048 + w * DEPTH * 8;
  if (lane == 0) { for (int s = 0; s < DEPTH; ++s) mbar_init(bars + s * 8, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncwarp();
  const long long T = (long long)row_blocks * chunks_per_row;
  const int Wtot = gridDim.x * 8, gw = blockIdx.x * 8 + w;
  long long t = gw * T / Wtot, ti = t;
  const long long t1 = (gw + 1) * T / Wtot;
  int islot = 0, cslot = 0; uint32_t par = 0; unsigned acc = 0;
  auto issue = [&]() {
    if (lane == 0) {
      const int rb = int(ti / chunks_per_row), kc = int(ti % chunks_per_row);
      mbar_expect_tx(bars + islot * 8, 2048);
      tma_2d(ring + islot * 2048, &tm, kc * 128, rb * 16, bars + islot * 8);
    }
    if (++islot == DEPTH) islot = 0;
    ++ti;
  };
  for (int i = 0; i < DEPTH && ti < t1; ++i) issue();
  for (; t < t1; ++t) {
    mbar_wait(bars + cslot * 8, par);
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(ring + cslot * 2048 + lane * 64));
    acc ^= v;
    if (++cslot == DEPTH) { cslot = 0; par ^= 1; }
    __syncwarp();
    if (ti < t1) issue();
    spin(delay);
  }
  if (acc == 0x12345678u) out[0] = acc;
}

// ---- per-CTA slabs: [16 rows x SLAB bytes] per request, 8 warps share it ----
template <int DEPTH, int SLAB>
__global__ void __launch_bounds__(288, 2) k_slab(const __grid_constant__ CUtensorMap tm, int row_blocks, int slabs_per_row, int delay, unsigned* out) {
  extern __shared__ uint8_t raw[];
  const uint32_t base = (smem_u32(raw) + 1023u) & ~1023u;
  constexpr int SB = 16 * SLAB;   // bytes per slab
  const uint32_t bars = base + DEPTH * SB;   // full[DEPTH], empty[DEPTH]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < DEPTH; ++s) { mbar_init(bars + s * 8, 1); mbar_init(bars + (DEPTH + s) * 8, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long T = (long long)row_blocks * slabs_per_row;
  long long t0 = blockIdx.x * T / gridDim.x;
  const long long t1 = (blockIdx.x + 1) * T / gridDim.x;
  if (w == 8) {   // producer
    if (lane == 0) {
      int slot = 0; uint32_t par = 1; long long n = 0;
      for (long long t = t0; t < t1; ++t, ++n) {
        if (n >= DEPTH) mbar_wait(bars + (DEPTH + slot) * 8, par);
        const int rb = int(t / slabs_per_row), ks = int(t % slabs_per_row);
        mbar_expect_tx(bars + slot * 8, SB);
        tma_2d(base + slot * SB, &tm, ks * (SLAB / 4), rb * 16, bars + slot * 8);   // uint32 elements
        if (++slot == DEPTH) { slot = 0; par ^= 1; }
      }
    }
    return;
  }
  int slot = 0; uint32_t par = 0; unsigned acc = 0;
  for (long long t = t0; t < t1; ++t) {
    mbar_wait(bars + slot * 8, par);
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(base + slot * SB + (lane & 15) * SLAB + w * (SLAB / 8) + (lane >> 4) * 4));
    acc ^= v;
    __syncwarp();
    if (lane == 0) mbar_arrive(bars + (DEPTH + slot) * 8);
    if (++slot == DEPTH) { slot = 0; par ^= 1; }
    spin(delay * (SLAB / 128) / 8);   // the slab's arithmetic is shared by 8 warps
  }
  if (acc == 0x12345678u) out[0] = acc;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main(int argc, char** argv) {
  const int N = argc > 1 ? atoi(argv[1]) : 12288, K = argc > 2 ? atoi(argv[2]) : 12288, delay = argc > 3 ? atoi(argv[3]) : 0;
  const size_t row_bytes = K / 2, bytes = (size_t)N * row_bytes;
  void* fn = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  EncodeFn enc = (EncodeFn)fn;
  std::vector<uint8_t*> bufs(5);
  for (auto& p : bufs) { CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 1, bytes)); }
  unsigned* out; CK(cudaMalloc(&out, 4));
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  auto time_it = [&](auto launch) {
    for (int i = 0; i < 3; ++i) launch(bufs[i % 5]);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(a);
    for (int i = 0; i < 20; ++i) launch(bufs[i % 5]);
    cudaEventRecord(b); CK(cudaEventSynchronize(b));
    float ms; cudaEventElapsedTime(&ms, a, b); return ms / 20;
  };
  auto rep = [&](const char* name, float ms) { printf("%-34s %8.2f us  %7.1f GB/s\n", name, ms * 1e3, bytes / (ms * 1e-3) / 1e9); };
  printf("N=%d K=%d bytes=%.1f MB delay=%d cycles per 2 KB\n", N, K, bytes / 1e6, delay);
  auto make_map = [&](uint8_t* w, CUtensorMapDataType dt, int esz, int box_inner_elems, CUtensorMapSwizzle sw) {
    CUtensorMap tm;
    cuuint64_t dims[2] = {row_bytes / esz, (cuuint64_t)N}; cuuint64_t strides[1] = {row_bytes};
    cuuint32_t box[2] = {(cuuint32_t)box_inner_elems, 16}; cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tm, dt, 2, w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode failed %d\n", (int)r); exit(1); }
    return tm;
  };
#define RUN_BOX(D) { const int smem = 1024 + 8 * D * 2048 + 8 * D * 8; CK(cudaFuncSetAttribute(k_box<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
    char nm[64]; snprintf(nm, 64, "box 16x128B per warp, depth %d", D); \
    rep(nm, time_it([&](uint8_t* w) { CUtensorMap tm = make_map(w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, 128, CU_TENSOR_MAP_SWIZZLE_128B); \
      k_box<D><<<2 * sms, 256, smem>>>(tm, N / 16, int(row_bytes / 128), delay, out); })); }
  RUN_BOX(1) RUN_BOX(2) RUN_BOX(4)
#define RUN_SLAB(D, S) if (row_bytes % S == 0) { const int smem = 1024 + D * 16 * S + 2 * D * 8; CK(cudaFuncSetAttribute(k_slab<D, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
    char nm[64]; snprintf(nm, 64, "slab 16x%dB per CTA, depth %d", S, D); \
    rep(nm, time_it([&](uint8_t* w) { CUtensorMap tm = make_map(w, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, S / 4, CU_TENSOR_MAP_SWIZZLE_NONE); \
      k_slab<D, S><<<2 * sms, 288, smem>>>(tm, N / 16, int(row_bytes / S), delay, out); })); }
  RUN_SLAB(2, 512) RUN_SLAB(4, 512) RUN_SLAB(2, 1024) RUN_SLAB(4, 1024)
  return 0;
}
