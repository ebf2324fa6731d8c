// tools/slab_stream.cu -- where the m = 1 decode GEMV's steady-state time goes (DESIGN.md 3.2): replays the exact request stream of
// gemv_slab_kernel (bitblas_b200/csrc/bb_gemv_slab.cu) with no arithmetic, for the bench workload's parameters (uint4, g = 128,
// fp16 scales [N, K/128], quantized zeros [K/128, N/2], fp16 activations):
//   the persistent grid of 2 CTAs per SM, the stream-K ranges ri*T/R in reverse CTA order, the unit order (row-block group, k, member),
//   the 4-stage ring per CTA, the TMA weight box {512 B, 32 rows}, the 2 KB activation bulk copy, the per-row 16-byte cp.async of
//   scales and packed zeros, programmatic dependent launch.  Each consumer warp only waits on its stage and arrives on `empty`.
// Request classes (bit mask): 1 weights, 2 activations, 4 group parameters; options: 8 one L2 prefetch of a row block's whole scale
// run at its first unit of the range, 16 evict_first on the weight box, 32 evict_last on the activation slab.
// Rows: (a) a linear ld.global.nc read of the same bytes (the ceiling), (b) weights, (c) + activations, (d) + parameters,
// (e1) (d) + the scale-run prefetch, (e2) (d) + both L2 policies, (e) (d) + all three options.
// Each row: one isolated launch (median of 20, each on a cold copy) and 40 back-to-back launches over rotated copies (>= 300 MB, as
// bench.py rotates; median of 5 passes); GB/s from bench.py's gemv_bytes (W + scales + zeros + A + C).
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/slab_stream tools/slab_stream.cu
// Run:   tools/slab_stream [--mask M ...] [NxK ...]     (default: the four bench shapes, rows a..e)
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

// the kernel's geometry (bb_gemv_slab.cu)
constexpr int ROWS = 32, ROW_BYTES = 512, KU = 1024, STEPS = 8, WBYTES = ROWS * ROW_BYTES, ABYTES = KU * 2, GW = 4, NG = 2, S = 4;
constexpr int THREADS = (GW * NG + 2) * 32;
constexpr int SMEM = 1024 + S * (WBYTES + ABYTES + 2048 + 1024 + 64) + NG * 2 * (2 * GW) * ROWS * 4 + 32 * S + 64;   // GS_SMEM_BYTES
constexpr int M_W = 1, M_A = 2, M_P = 4, M_PF = 8, M_POLW = 16, M_POLA = 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(n)); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_only(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n"
               ::"r"(bar), "r"(parity), "r"(20000u) : "memory");
}
__device__ __forceinline__ uint64_t policy_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t policy_last() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void tma_2d(uint32_t dst, const void* map, int c0, int c1, uint32_t bar, bool hint, uint64_t pol) {
  if (hint)
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
                 ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar), "l"(pol) : "memory");
  else
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, bool hint, uint64_t pol) {
  if (hint)
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
  else
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(bar) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* src, uint32_t bytes) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory"); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory"); }

struct P {
  const uint16_t* scale; const uint8_t* zeros; const uint8_t* A;
  int N, K, G, UPR, NRB, T, mask;
};

__global__ void __launch_bounds__(THREADS, 2) replay(const __grid_constant__ CUtensorMap tmW, const P p) {
  extern __shared__ uint8_t raw_smem[];
  const uint32_t base = (smem_u32(raw_smem) + 1023u) & ~1023u;
  const uint32_t Wb = base, Ab = Wb + S * WBYTES, RAWb = Ab + S * ABYTES + S * 2048, Bb = RAWb + S * 1024 + S * 64 + NG * 2 * (2 * GW) * ROWS * 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(Bb + 8u * s, 1); mbar_init(Bb + 8u * (2 * S + s), 32); mbar_init(Bb + 8u * (3 * S + s), GW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const bool mW = p.mask & M_W, mA = p.mask & M_A, mP = p.mask & M_P, mPF = p.mask & M_PF;
  const int R = gridDim.x, ri = R - 1 - int(blockIdx.x);
  const int t0 = int((long long)ri * p.T / R), t1 = int((long long)(ri + 1) * p.T / R), n_units = t1 - t0;
  const int UPR = p.UPR, npre = min(S, n_units);
  if (warp == NG * GW) {   // issuer
    const uint64_t pol_w = policy_first(), pol_a = policy_last();
    auto unit_w = [&](int rb, int ku, int slot) { tma_2d(Wb + slot * WBYTES, &tmW, ku * (ROW_BYTES / 4), rb * ROWS, Bb + 8u * slot, p.mask & M_POLW, pol_w); };
    auto unit_params = [&](int rb, int ku, int slot, bool first) {
      if (!mP) return;
      if (mPF && first && lane == 0) prefetch_l2(p.scale + size_t(rb) * ROWS * p.G, uint32_t(ROWS * p.G * 2));
      const uint32_t raw = RAWb + slot * 1024;
      cp_async16(raw + lane * 16u, p.scale + size_t(rb * ROWS + lane) * p.G + ku * STEPS);
      if (lane < STEPS) cp_async16(raw + 512u + lane * 16u, p.zeros + size_t(ku * STEPS + lane) * (p.N >> 1) + rb * (ROWS / 2));
      cp_async_arrive_noinc(Bb + 8u * (2 * S + slot));
    };
    const int rest = t0 / NG, g0 = t0 - rest * NG, q0 = rest / UPR, ku0 = rest - q0 * UPR;
    auto next_unit = [&](int& qq, int& kk, int& gg) { if (++gg == NG) { gg = 0; if (++kk == UPR) { kk = 0; ++qq; } } };
    {
      int qq = q0, kk = ku0, gg = g0;
      for (int u = 0; u < npre; ++u) {
        const int rb = qq * NG + gg;
        if (mW && lane == 0 && rb < p.NRB) { mbar_expect_tx_only(Bb + 8u * u, WBYTES); unit_w(rb, kk, u); }
        unit_params(rb, kk, u, u < NG || kk == 0);
        next_unit(qq, kk, gg);
      }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    int slot = 0, qq = q0, ku = ku0, gg = g0;
    uint32_t ephase = 1u;
    for (int i = 0; i < n_units; ++i) {
      const int rb = qq * NG + gg;
      mbar_wait(Bb + 8u * (3 * S + slot), ephase);
      const int k0 = ku * KU;
      const uint32_t abytes = mA ? uint32_t(min(KU, p.K - k0)) * 2u : 0u;
      if (lane == 0) {
        const bool w_now = mW && i >= npre && rb < p.NRB;
        mbar_arrive_expect_tx(Bb + 8u * slot, abytes + (w_now ? uint32_t(WBYTES) : 0u));
        if (w_now) unit_w(rb, ku, slot);
        if (mA) bulk_g2s(Ab + slot * ABYTES, p.A + size_t(k0) * 2, abytes, Bb + 8u * slot, p.mask & M_POLA, pol_a);
      }
      if (i >= npre) unit_params(rb, ku, slot, ku == 0);
      if (++slot == S) { slot = 0; ephase ^= 1u; }
      next_unit(qq, ku, gg);
    }
    return;
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (warp > NG * GW) return;   // (the finisher warp: its work is arithmetic)
  const int grp = warp / GW;
  int i = (grp - t0 % NG + NG) % NG, slot = i;
  uint32_t phase = 0u;
  for (; i < n_units; i += NG) {
    mbar_wait(Bb + 8u * slot, phase);
    if (mP) mbar_wait(Bb + 8u * (2 * S + slot), phase);
    __syncwarp();
    if (lane == 0) mbar_arrive(Bb + 8u * (3 * S + slot));
    slot += NG;
    if (slot >= S) { slot -= S; phase ^= 1u; }
  }
}

__global__ void __launch_bounds__(512) linear_read(const uint4* __restrict__ src, size_t n16, unsigned* out) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  uint32_t acc = 0;
  size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[j].x), "=r"(v[j].y), "=r"(v[j].z), "=r"(v[j].w) : "l"(src + i + j * stride));
#pragma unroll
    for (int j = 0; j < 4; ++j) acc ^= v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
  }
  for (; i < n16; i += stride) { const uint4 v = src[i]; acc ^= v.x ^ v.y ^ v.z ^ v.w; }
  if (acc == 0x9e3779b9u) out[0] = acc;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static double gemv_bytes(double N, double K) { return N * K / 2 + N * (K / 128) * 2 + (K / 128) * N / 2 + K * 2 + N * 2; }   // bench.py

int main(int argc, char** argv) {
  std::vector<std::pair<int, int>> shapes;
  std::vector<int> masks;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--mask" && i + 1 < argc) masks.push_back(int(strtol(argv[++i], nullptr, 0)));
    else { int n, k; if (sscanf(a.c_str(), "%dx%d", &n, &k) == 2) shapes.push_back({n, k}); }
  }
  if (shapes.empty()) shapes = {{8192, 8192}, {28672, 8192}, {8192, 28672}, {12288, 12288}};
  struct Row { const char* name; int mask; };
  std::vector<Row> rows = {{"(a) linear ld.global.nc", -1}, {"(b) weights", M_W}, {"(c) + activations", M_W | M_A},
                           {"(d) + parameters", M_W | M_A | M_P}, {"(e1) (d) + scale-run prefetch", M_W | M_A | M_P | M_PF},
                           {"(e2) (d) + L2 policies", M_W | M_A | M_P | M_POLW | M_POLA},
                           {"(e) (d) + prefetch + policies", M_W | M_A | M_P | M_PF | M_POLW | M_POLA}};
  if (!masks.empty()) {
    rows.clear();
    for (int m : masks) rows.push_back({"mask", m});
  }
  for (auto [N, K] : shapes)
    if (N % 64 || K % KU) { printf("%dx%d: N must be a multiple of 64 and K of 1024 (whole units, the fast parameter path)\n", N, K); return 1; }

  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  int sms = prop.multiProcessorCount, clk = 0;
  CK(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0));
  char smi[256] = "nvidia-smi unavailable";
  if (FILE* f = popen("nvidia-smi -i 0 --query-gpu=power.limit,clocks.max.sm --format=csv,noheader 2>/dev/null", "r")) {
    if (!fgets(smi, sizeof(smi), f)) snprintf(smi, sizeof(smi), "nvidia-smi gave no output");
    pclose(f);
    smi[strcspn(smi, "\n")] = 0;
  }
  printf("%s, %d SMs, max SM clock %d MHz; power limit, max SM clock (nvidia-smi): %s\n", prop.name, sms, clk / 1000, smi);

  void* fn = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  const EncodeFn enc = (EncodeFn)fn;
  CK(cudaFuncSetAttribute(replay, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  int occ = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, replay, THREADS, SMEM));
  if (occ < 2) { printf("replay kernel: %d CTAs per SM, expected 2\n", occ); return 1; }
  unsigned* out; CK(cudaMalloc(&out, 4));
  cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

  for (auto [N, K] : shapes) {
    const int G = K / 128;
    const size_t wb = size_t(N) * K / 2, sb = size_t(N) * G * 2, zb = size_t(G) * N / 2, ab = size_t(K) * 2;
    const size_t block = wb + sb + zb + ab + size_t(N) * 2 + 4096;   // + room for the linear read of gemv_bytes
    const double gb = gemv_bytes(N, K);
    const int copies = std::max(2, int(300e6 / double(wb + sb + zb + ab)) + 1);
    std::vector<uint8_t*> buf(copies);
    std::vector<CUtensorMap> maps(copies);
    std::vector<P> prm(copies);
    for (int c = 0; c < copies; ++c) {
      CK(cudaMalloc(&buf[c], block));
      CK(cudaMemset(buf[c], 0x11 * (c + 1), block));
      cuuint64_t dims[2] = {cuuint64_t(K / 8), cuuint64_t(N)}, strides[1] = {cuuint64_t(K / 2)};
      cuuint32_t box[2] = {ROW_BYTES / 4, ROWS}, es[2] = {1, 1};
      if (enc(&maps[c], CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, buf[c], dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) { printf("tensor map encode failed\n"); return 1; }
      P& p = prm[c];
      p.scale = reinterpret_cast<const uint16_t*>(buf[c] + wb); p.zeros = buf[c] + wb + sb; p.A = buf[c] + wb + sb + zb;
      p.N = N; p.K = K; p.G = G; p.UPR = K / KU; p.NRB = N / ROWS; p.T = ((p.NRB + NG - 1) / NG) * p.UPR * NG; p.mask = 0;
    }
    const int grid = std::min(prm[0].T, 2 * sms);
    auto launch = [&](int mask, int c) {
      if (mask < 0) { linear_read<<<4 * sms, 512, 0, st>>>(reinterpret_cast<const uint4*>(buf[c]), size_t(gb) / 16, out); return; }
      P p = prm[c]; p.mask = mask;
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = grid; cfg.blockDim = THREADS; cfg.dynamicSmemBytes = SMEM; cfg.stream = st;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      CK(cudaLaunchKernelEx(&cfg, replay, maps[c], p));
    };
    auto elapsed_us = [&]() { float ms; CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); return double(ms) * 1e3; };
    auto median = [](std::vector<double> v) { std::sort(v.begin(), v.end()); return v[v.size() / 2]; };
    printf("\nN=%d K=%d: %.2f MB per launch (gemv_bytes), %d copies (%.0f MB), grid %d x %d threads\n", N, K, gb / 1e6, copies,
           copies * (wb + sb + zb + ab) / 1e6, grid, THREADS);
    printf("  %-32s %11s %9s %11s %9s\n", "", "single us", "GB/s", "b2b x40 us", "GB/s");
    int rot = 0;
    for (const Row& r : rows) {
      for (int i = 0; i < 2 * copies; ++i) launch(r.mask, rot++ % copies);   // warm-up (module load, clocks)
      CK(cudaStreamSynchronize(st));
      std::vector<double> one, b2b;
      for (int rep = 0; rep < 20; ++rep) {
        CK(cudaEventRecord(e0, st)); launch(r.mask, rot++ % copies); CK(cudaEventRecord(e1, st));
        one.push_back(elapsed_us());
      }
      for (int rep = 0; rep < 5; ++rep) {
        CK(cudaEventRecord(e0, st));
        for (int i = 0; i < 40; ++i) launch(r.mask, rot++ % copies);
        CK(cudaEventRecord(e1, st));
        b2b.push_back(elapsed_us() / 40);
      }
      CK(cudaGetLastError());
      const double t1 = median(one), tb = median(b2b);
      char nm[48];
      if (r.mask >= 0 && !masks.empty()) snprintf(nm, sizeof(nm), "mask 0x%02x", r.mask); else snprintf(nm, sizeof(nm), "%s", r.name);
      printf("  %-32s %11.2f %9.0f %11.2f %9.0f\n", nm, t1, gb / (t1 * 1e3), tb, gb / (tb * 1e3));
      fflush(stdout);
    }
    for (auto b : buf) CK(cudaFree(b));
  }
  return 0;
}
