// bb_gemm_fp8.cu -- block-scaled FP8 GEMM on the FP8 tensor cores (bb_matmul_fp8): e4m3 activations x e4m3 weights, both
// wgmma operands read from shared memory ("SS"), one fp32 scale per (activation row, 128-k block) and one per (128 weight rows,
// 128-k block), as DeepSeek-V3 and the Qwen3 -FP8 checkpoints store them.
//
//     P[r, n, b] = sum_{k in block b} q_a[r, k] * q_w[n, k]              wgmma m64nBMk32 e4m3, fp32, per k-block
//     S[r, n]    = sum_b P[r, n, b] * (a_scale[r, b] * w_scale[n / 128, b])   fp32, each product and sum rounded, b ascending
//
// The geometry is gemm_ts's (bb_gemm_ts.cu): a CTA owns 128 weight rows -- the wgmma M side, two consumer warpgroups of 64 rows
// -- and BM activation rows (the wgmma N side); one producer warp streams each 128-k block through a ring of mbarrier stages:
//   W tile  [128 rows x 128 B]  e4m3, SW128 (a 2-D box on the checkpoint's [N, K] bytes; rows past N are zero-filled)
//   A tile  [BM rows  x 128 B]  e4m3, SW128 (the int8 path's descriptor, make_sw128_desc)
//   scales  [BM] fp32            that block's activation scales: one contiguous run of the k-block-major a_scale
// Per k-block a consumer warpgroup issues four wgmma k32 steps into a fresh accumulator P (the first with scale-d = 0), waits
// for them (wait<0>), releases the stage and promotes: acc = acc + P * (sa * sw).  The 128-row tile is the 128-row weight
// scale block, so the weight scale is one float per k-block, fetched one block ahead.  The loop body is the same for every
// k-block: a branch around the wgmmas or the wait makes ptxas serialize every wgmma (DESIGN.md §3.2.5).
//
// The k-loop is this file's own: sharing device functions with gemm_ts_kernel changes its register allocation (§3.2.1).
// Split-K (gemm_ts's rule, whole k-blocks): split j writes its fp32 S_j to [splits][m][N]; splitk_reduce_fp8_kernel adds the
// splits in order, rounds and adds the bias.
#include <algorithm>

#include "bb_gemm_ts.cuh"

namespace bb {

namespace {

struct Fp8Params {
  const float* w_scale;   // [ceil(N / 128), K / 128]
  const void* bias;       // [N] out_dtype, or null
  void* C;                // [M, N] out_dtype
  float* ws;              // [splits][M][N] fp32 partials (splits > 1)
  int M, N, KB;           // KB = K / 128
  int m_tiles, splits, kb_per_split;
  int out_dtype;
};

template <int BM>
struct Fp8Smem {
  static constexpr int kActBytes = BM * FP8_KB;
  static constexpr int kWBytes = TS_ROWS * FP8_KB;
  static constexpr int kScaleBytes = BM * 4;
  static constexpr int kStageBytes = kActBytes + kWBytes + kScaleBytes;
  static constexpr int kStagesRaw = (200 * 1024) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kBarBytes = 256;   // full[8] + empty[8]
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + 1024;   // + alignment slack
};

template <int BM>
__global__ void __launch_bounds__(TS_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                const __grid_constant__ CUtensorMap tmS, const Fp8Params p) {
  using SM = Fp8Smem<BM>;
  constexpr int S = SM::kStages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                                    // [S][BM][128 B], 1024-aligned
  uint8_t* sW = smem + S * SM::kActBytes;                                // [S][128][128 B], 1024-aligned
  float* sS = reinterpret_cast<float*>(sW + S * SM::kWBytes);            // [S][BM]
  uint64_t* full = reinterpret_cast<uint64_t*>(sS + S * BM);             // [S]   TMA -> consumers
  uint64_t* empty = full + S;                                            // [S]   consumer warps -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x % p.splits;
  const int tile = blockIdx.x / p.splits;
  const int m_tile = tile % p.m_tiles;
  const int n_tile = tile / p.m_tiles;
  const int kb0 = split * p.kb_per_split;
  const int m0 = m_tile * BM, n0 = n_tile * TS_ROWS;
  const int num_kb = p.kb_per_split;

  if (warp == TS_CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmS);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TS_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TS_CONSUMER_WARPS) {
    // ===== TMA producer =====
    if (lane == 0) {
      int s = 0;
      uint32_t par = 1;   // parity of the "previous use" of the stage: the first pass must not wait
      for (int kb = 0; kb < num_kb; ++kb) {
        if (kb >= S) mbar_wait(&empty[s], par);
        mbar_arrive_expect_tx(&full[s], SM::kStageBytes);
        tma_load_2d(sA + s * SM::kActBytes, &tmA, (kb0 + kb) * FP8_KB, m0, &full[s]);
        tma_load_2d(sW + s * SM::kWBytes, &tmW, (kb0 + kb) * FP8_KB, n0, &full[s]);
        tma_load_2d(sS + s * BM, &tmS, m0, kb0 + kb, &full[s]);
        if (++s == S) { s = 0; par ^= 1; }
      }
    }
    return;
  }

  // ===== consumer warpgroups =====
  const int g8 = lane >> 2, t = lane & 3;
  const int wg = warp >> 2;
  const int rA = wg * 64 + (warp & 3) * 16 + g8;   // accumulator rows rA and rA + 8 of this thread (tile-local)
  const int nA = n0 + rA, nB = nA + 8;
  float acc[BM / 2], P[BM / 2];
#pragma unroll
  for (int i = 0; i < BM / 2; ++i) acc[i] = 0.f;
  const float* wsc = p.w_scale + size_t(n_tile) * p.KB + kb0;
  float sw_next = __ldg(wsc);
  const uint32_t aW = smem_u32(sW) + uint32_t(wg * 64 * FP8_KB);   // this warpgroup's 64 weight rows

  int st = 0;
  uint32_t full_par = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const float sw = sw_next;
    sw_next = __ldg(wsc + min(kb + 1, num_kb - 1));
    mbar_wait(&full[st], full_par);
    const uint64_t adesc = make_sw128_desc(aW + uint32_t(st * SM::kWBytes));
    const uint64_t bdesc = make_sw128_desc(smem_u32(sA + st * SM::kActBytes));
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < 4; ++s) WgmmaFp8<BM>::mma(P, adesc + uint64_t(2 * s), bdesc + uint64_t(2 * s), s ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    // P[4i + 2h + j] = P^T[row rA + 8h][column 8i + 2t + j]; the column's activation scale is in the stage
    const float* ss = sS + st * BM + 2 * t;
#pragma unroll
    for (int i = 0; i < BM / 8; ++i) {
      const float2 sa = *reinterpret_cast<const float2*>(ss + 8 * i);
      const float c0 = __fmul_rn(sa.x, sw), c1 = __fmul_rn(sa.y, sw);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc[4 * i + 2 * h] = __fadd_rn(acc[4 * i + 2 * h], __fmul_rn(P[4 * i + 2 * h], c0));
        acc[4 * i + 2 * h + 1] = __fadd_rn(acc[4 * i + 2 * h + 1], __fmul_rn(P[4 * i + 2 * h + 1], c1));
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == S) { st = 0; full_par ^= 1; }
  }

  // ----- epilogue: acc[4i + 2h + j] = S^T[row rA + 8h][column 8i + 2t + j] -----
#pragma unroll
  for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + 8 * i + 2 * t + j;
      if (m >= p.M) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = h ? nB : nA;
        if (n >= p.N) continue;
        const float v = acc[4 * i + 2 * h + j];
        if (p.splits > 1) p.ws[(size_t(split) * p.M + m) * p.N + n] = v;   // the split's S_j; the reduce rounds
        else store_out_dequant(p.C, size_t(m) * p.N + n, v, p.bias, n, p.out_dtype);
      }
    }
  }
}

// S = ((0 + S_0) + S_1) + ... + S_{splits-1}, then round_out(S) with the bias in out_dtype.  One thread = 4 consecutive n
// (N % 16 == 0): one 128-bit load of each split's partials.
__global__ void splitk_reduce_fp8_kernel(const Fp8Params p) {
  const unsigned n4 = unsigned(p.N) >> 2;
  const unsigned total4 = unsigned(p.M) * n4;
  const size_t split_stride4 = size_t(p.M) * n4;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const unsigned m = i / n4, n = (i - m * n4) * 4u;
    float S[4] = {0.f, 0.f, 0.f, 0.f};
    for (int sp = 0; sp < p.splits; ++sp) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(p.ws) + size_t(sp) * split_stride4 + i);
      S[0] = __fadd_rn(S[0], v.x); S[1] = __fadd_rn(S[1], v.y); S[2] = __fadd_rn(S[2], v.z); S[3] = __fadd_rn(S[3], v.w);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) store_out_dequant(p.C, size_t(m) * p.N + n + j, S[j], p.bias, n + j, p.out_dtype);
  }
}

int bm_for(int m) { return m <= 32 ? 32 : (m <= 64 ? 64 : 128); }

// gemm_ts's split rule on this kernel's tile grid: only up to m = 128, only when the tiles leave SMs idle, whole k-blocks
int fp8_splits(const bb_matmul_desc& d, int m) {
  if (m > 128) return 1;
  const int bm = bm_for(m);
  const int tiles = ((m + bm - 1) / bm) * ((d.N + TS_ROWS - 1) / TS_ROWS);
  return gemm_ts_splits(tiles, d.K / FP8_KB, device_sm_count());
}

template <int BM>
int launch_fp8_inst(const Fp8Args& a) {
  using SM = Fp8Smem<BM>;
  auto kernel = gemm_fp8_kernel<BM>;
  static KernelCache<> cache;
  if (!kernel_setup(cache, kernel, SM::kTotal)) {
    set_error("gemm_fp8: cannot raise the kernel's dynamic shared memory to %d bytes on this device", SM::kTotal);
    return 2;
  }
  const bb_matmul_desc& d = a.d;
  Fp8Params p;
  p.w_scale = a.w_scale; p.bias = a.bias; p.C = a.C;
  p.M = a.m; p.N = d.N; p.KB = d.K / FP8_KB;
  p.m_tiles = (a.m + BM - 1) / BM;
  const int tiles = p.m_tiles * ((d.N + TS_ROWS - 1) / TS_ROWS);
  p.splits = fp8_splits(d, a.m);
  if (p.splits > 1 && a.workspace_bytes < size_t(p.splits) * a.m * d.N * 4) p.splits = 1;   // no scratch given
  p.kb_per_split = p.KB / p.splits;
  p.ws = static_cast<float*>(a.workspace);
  p.out_dtype = d.out_dtype;
  CUtensorMap tmA, tmW, tmS;
  int rc = make_map_2d(&tmA, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.A, uint64_t(d.K), uint64_t(a.m), uint64_t(d.K), FP8_KB, BM,
                       CU_TENSOR_MAP_SWIZZLE_128B);
  if (!rc) rc = make_map_2d(&tmW, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.W, uint64_t(d.K), uint64_t(d.N), uint64_t(d.K), FP8_KB, TS_ROWS,
                            CU_TENSOR_MAP_SWIZZLE_128B);
  // a_scale as [K / 128][m] fp32 rows a_scale_ld apart: one box = one k-block's BM scales (rows past m are zero-filled)
  if (!rc) rc = make_map_2d(&tmS, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a.a_scale, uint64_t(a.m), uint64_t(p.KB),
                            uint64_t(a.a_scale_ld) * 4, BM, 1, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  kernel<<<tiles * p.splits, TS_THREADS, SM::kTotal, a.stream>>>(tmA, tmW, tmS, p);
  BB_LAUNCH_CHECK();
  if (p.splits > 1) {
    const size_t total = size_t(a.m) * d.N / 4;   // one thread per 4 consecutive output columns
    const int rthreads = 256;
    const int rblocks = int(std::min<size_t>((total + rthreads - 1) / rthreads, size_t(device_sm_count()) * 8));
    splitk_reduce_fp8_kernel<<<rblocks, rthreads, 0, a.stream>>>(p);
    BB_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace

size_t gemm_fp8_workspace_bytes(const bb_matmul_desc& d, int m) {
  const int sp = fp8_splits(d, m);
  return sp > 1 ? size_t(sp) * m * d.N * 4 : 0;
}

int launch_gemm_fp8(const Fp8Args& a) {
  if (a.m <= 32) return launch_fp8_inst<32>(a);
  if (a.m <= 64) return launch_fp8_inst<64>(a);
  return launch_fp8_inst<128>(a);
}

}  // namespace bb
