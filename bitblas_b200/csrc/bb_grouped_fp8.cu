// bb_grouped_fp8.cu -- grouped block-scaled FP8 GEMM for mixture-of-experts layers (bb_matmul_grouped_fp8[_swiglu]): ONE launch
// over E experts of a 128 x 128 block-scaled e4m3 checkpoint (DeepSeek-V3 / R1, Qwen3 -FP8),
//     C[offsets[e] : offsets[e+1]] = A[offsets[e] : offsets[e+1]] x W[e]^T      block-scaled as bb_matmul_fp8, for every e,
// with the row offsets read on the device.
//
// Design:
//   * the per-tile arithmetic is gemm_fp8_kernel's (bb_gemm_fp8.cu): a TMA producer warp streams, per 128-k block, the e4m3
//     weight tile, the e4m3 activation tile and the block's BM activation scales into a ring of mbarrier stages; two consumer
//     warpgroups issue four wgmma k32 steps into a fresh accumulator P, wait for them and promote acc = acc + P * (sa * sw) with
//     every product and sum rounded, blocks ascending.  Then round_out.  There is no split-K and no workspace.  The k-loop is
//     written out here again: sharing device functions with gemm_fp8_kernel changes its register allocation (DESIGN.md §3.2.1).
//   * the schedule is gemm_ts_grouped_kernel's (bb_grouped_gemm.cu): A [T, K] is one 2-D tensor map over all T rows and a tile of
//     expert e starts at row offsets[e] + mt * BM (rows past the expert's end are loaded but never stored, rows past T are
//     zero-filled); W [E, N, K] is one map of E * N rows; the activation scales are one {BM + 4, 1} box of the k-block-major
//     [K/128][a_scale_ld] buffer that starts at the 16-byte boundary at or below the tile's first row.  None of the maps depends
//     on the offsets (graph-capturable).  The grid is persistent; every CTA clamps the offsets and numbers each expert's ceil(m_e / BM) * N / 128 tiles with
//     grouped_schedule and walks its share; the mbarrier ring runs on from one tile to the next.  BM is chosen on the host from
//     the mean rows per active expert.
//   * programmatic dependent launch: griddepcontrol.wait first (which weights to stream depends on the offsets), launch_dependents
//     after the CTA's last tile.  Offsets are untrusted: clamped to [0, T], a group ending before it starts is empty, rows no
//     group claims are not written.
//   * weight scales: [E, N/128, K/128] fp32, row e * N/128 + n_tile, one float per k-block fetched one block ahead.
//   * SWIGLU (the gate/up projection): N = 2I rows in the gate/up interleave, so stored tile t holds gate rows 64t .. 64t + 63 and
//     up rows 64t .. 64t + 63: thread row nA (tile-local row % 16 < 8) is a gate row and nA + 8 an up row.  The scales are
//     interleaved the same way, [E, 2 ceil(I/128), K/128] with row 2c gate block c and row 2c + 1 up block c, and tile t reads
//     rows 2(t >> 1) (for h = 0) and 2(t >> 1) + 1 (for h = 1).  C [T, I] = round_out(silu(g) * u), g and u as the plain form
//     stores them (store_swiglu's rule).
#include <algorithm>
#include <climits>

#include "bb_gemm_ts.cuh"

namespace bb {

namespace {

// gemm_fp8_kernel's stage (A tile, W tile, the block's activation scales), except that the scale box starts at the 16-byte
// boundary at or below the tile's first row (an expert's rows start anywhere) and so is BM + 4 floats wide; each stage's scale
// slot is padded to a multiple of 128 bytes
template <int BM>
struct GroupedFp8Smem {
  static constexpr int kActBytes = BM * FP8_KB;
  static constexpr int kWBytes = TS_ROWS * FP8_KB;
  static constexpr int kScaleBox = BM + 4;                  // floats per scale box
  static constexpr int kScaleSlot = BM + 32;                // floats per stage's scale slot
  static constexpr int kStageTx = kActBytes + kWBytes + kScaleBox * 4;   // bytes TMA delivers per stage
  static constexpr int kStageBytes = kActBytes + kWBytes + kScaleSlot * 4;
  static constexpr int kStagesRaw = (200 * 1024) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kBarBytes = 256;   // full[8] + empty[8]
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + 1024;   // + alignment slack
};

struct GroupedFp8Params {
  const int32_t* offsets;   // [E + 1], device
  int E;                    // groups
  int T;                    // rows of A and C
  const float* w_scale;     // [E][s_rows][KB]
  int s_rows;               // weight-scale rows per expert: N / 128, or (SWIGLU) 2 ceil(I / 128)
  void* C;                  // [T, N] (SWIGLU: [T, N / 2]) out_dtype
  int N, KB;                // N per expert, KB = K / 128
  int out_dtype;
};

template <int BM, bool SWIGLU>
__global__ void __launch_bounds__(TS_THREADS, 1)
gemm_fp8_grouped_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                        const __grid_constant__ CUtensorMap tmS, const GroupedFp8Params g) {
  using SM = GroupedFp8Smem<BM>;
  constexpr int S = SM::kStages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                                    // [S][BM][128 B], 1024-aligned
  uint8_t* sW = smem + S * SM::kActBytes;                                // [S][128][128 B], 1024-aligned
  float* sS = reinterpret_cast<float*>(sW + S * SM::kWBytes);            // [S][kScaleSlot]
  uint64_t* full = reinterpret_cast<uint64_t*>(sS + S * SM::kScaleSlot); // [S]   TMA -> consumers
  uint64_t* empty = full + S;                                            // [S]   consumer warps -> TMA
  __shared__ int row0_s[BB_GROUPED_MAX_GROUPS];       // clamped first row of each group
  __shared__ int rows_s[BB_GROUPED_MAX_GROUPS];       // rows of each group (0: empty)
  __shared__ int item0_s[BB_GROUPED_MAX_GROUPS + 1];  // first tile of each group; item0_s[E] = all tiles

  pdl_wait();   // offsets, A and a_scale are the preceding kernels' output; nothing is read before this
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = g.N / TS_ROWS;
  const int num_kb = g.KB;
  if (warp == TS_CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmS);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TS_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  if (threadIdx.x < 32) grouped_schedule(g, BM, n_tiles, row0_s, rows_s, item0_s);
  __syncthreads();
  const int total = item0_s[g.E];

  // tile `item`: expert e, activation rows [m0, m_end) of which the tile holds the first BM, expert-local n-tile nt
  auto tile_of = [&](int item, int& e, int& m0, int& m_end, int& nt) {
    e = grouped_find(item0_s, g.E, item);
    const int local = item - item0_s[e];
    const int m_tiles = (rows_s[e] + BM - 1) / BM;
    nt = local / m_tiles;
    m0 = row0_s[e] + (local - nt * m_tiles) * BM;
    m_end = row0_s[e] + rows_s[e];
  };

  if (warp == TS_CONSUMER_WARPS) {
    // ===== TMA producer: one continuous ring over all of this CTA's tiles =====
    if (lane == 0) {
      int s = 0, loads = 0;
      uint32_t par = 1;   // parity of the "previous use" of the stage: the first pass must not wait
      for (int item = blockIdx.x; item < total; item += gridDim.x) {
        int e, m0, m_end, nt;
        tile_of(item, e, m0, m_end, nt);
        const int wrow = e * g.N + nt * TS_ROWS;
        for (int kb = 0; kb < num_kb; ++kb, ++loads) {
          if (loads >= S) mbar_wait(&empty[s], par);
          mbar_arrive_expect_tx(&full[s], SM::kStageTx);
          tma_load_2d(sA + s * SM::kActBytes, &tmA, kb * FP8_KB, m0, &full[s]);
          tma_load_2d(sW + s * SM::kWBytes, &tmW, kb * FP8_KB, wrow, &full[s]);
          tma_load_2d(sS + s * SM::kScaleSlot, &tmS, m0 & ~3, kb, &full[s]);
          if (++s == S) { s = 0; par ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups, tile after tile =====
  const int g8 = lane >> 2, t = lane & 3;
  const int wg = warp >> 2;
  const int rA = wg * 64 + (warp & 3) * 16 + g8;   // accumulator rows rA and rA + 8 of this thread (tile-local)
  const uint32_t aW = smem_u32(sW) + uint32_t(wg * 64 * FP8_KB);   // this warpgroup's 64 weight rows
  int st = 0;
  uint32_t full_par = 0;
  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    int e, m0, m_end, nt;
    tile_of(item, e, m0, m_end, nt);
    const int nA = nt * TS_ROWS + rA, nB = nA + 8;   // expert-local weight rows (SWIGLU: gate and up)
    float acc[BM / 2], P[BM / 2];
#pragma unroll
    for (int i = 0; i < BM / 2; ++i) acc[i] = 0.f;
    // the weight-scale row of rows nA and nB (SWIGLU: the gate row for nA, the up row after it for nB)
    const float* wsc = g.w_scale + (size_t(e) * g.s_rows + (SWIGLU ? 2 * (nt >> 1) : nt)) * g.KB;
    float sw_next = __ldg(wsc), su_next = SWIGLU ? __ldg(wsc + g.KB) : 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      const float sw = sw_next, su = su_next;
      const int kn = min(kb + 1, num_kb - 1);
      sw_next = __ldg(wsc + kn);
      if constexpr (SWIGLU) su_next = __ldg(wsc + g.KB + kn);
      mbar_wait(&full[st], full_par);
      const uint64_t adesc = make_sw128_desc(aW + uint32_t(st * SM::kWBytes));
      const uint64_t bdesc = make_sw128_desc(smem_u32(sA + st * SM::kActBytes));
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 4; ++s) WgmmaFp8<BM>::mma(P, adesc + uint64_t(2 * s), bdesc + uint64_t(2 * s), s ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      // P[4i + 2h + j] = P^T[row rA + 8h][column 8i + 2t + j]; the column's activation scale is in the stage, m0 % 4 floats
      // into the box
      const float* ss = sS + st * SM::kScaleSlot + (m0 & 3) + 2 * t;
#pragma unroll
      for (int i = 0; i < BM / 8; ++i) {
        const float2 sa = make_float2(ss[8 * i], ss[8 * i + 1]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float swh = SWIGLU && h ? su : sw;
          const float c0 = __fmul_rn(sa.x, swh), c1 = __fmul_rn(sa.y, swh);
          acc[4 * i + 2 * h] = __fadd_rn(acc[4 * i + 2 * h], __fmul_rn(P[4 * i + 2 * h], c0));
          acc[4 * i + 2 * h + 1] = __fadd_rn(acc[4 * i + 2 * h + 1], __fmul_rn(P[4 * i + 2 * h + 1], c1));
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      if (++st == S) { st = 0; full_par ^= 1; }
    }

    // ----- epilogue: acc[4i + 2h + j] = S^T[row rA + 8h][column 8i + 2t + j], rows m < m_end of expert e -----
    if constexpr (SWIGLU) {
      const size_t col = size_t(nA >> 4) * 8 + size_t(nA & 7);
#pragma unroll
      for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int m = m0 + 8 * i + 2 * t + j;
          if (m >= m_end) continue;
          const float gv = swiglu_operand(acc[4 * i + j], false, 0.f, g.out_dtype);
          const float uv = swiglu_operand(acc[4 * i + 2 + j], false, 0.f, g.out_dtype);
          store_swiglu(g.C, size_t(m) * size_t(g.N / 2) + col, gv, uv, g.out_dtype);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int m = m0 + 8 * i + 2 * t + j;
          if (m >= m_end) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int n = h ? nB : nA;
            store_out_dequant(g.C, size_t(m) * size_t(g.N) + size_t(n), acc[4 * i + 2 * h + j], nullptr, n, g.out_dtype);
          }
        }
      }
    }
  }
  pdl_launch_dependents();
}

template <int BM, bool SWIGLU>
int launch_grouped_fp8_inst(const GroupedFp8Args& a, const GroupedFp8Params& g, long long max_tiles) {
  using SM = GroupedFp8Smem<BM>;
  auto kernel = gemm_fp8_grouped_kernel<BM, SWIGLU>;
  static KernelCache<> cache;
  const int resident_per_sm = kernel_setup(cache, kernel, SM::kTotal, TS_THREADS, SM::kTotal);
  if (resident_per_sm <= 0) { set_error("grouped FP8 GEMM: the kernel cannot be resident on this device"); return 2; }
  const bb_matmul_desc& d = a.d;
  CUtensorMap tmA, tmW, tmS;
  int rc = make_map_2d(&tmA, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.A, uint64_t(d.K), uint64_t(a.total_rows), uint64_t(d.K), FP8_KB,
                       BM, CU_TENSOR_MAP_SWIZZLE_128B);
  if (!rc) rc = make_map_2d(&tmW, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.W, uint64_t(d.K), uint64_t(a.num_groups) * uint64_t(d.N),
                            uint64_t(d.K), FP8_KB, TS_ROWS, CU_TENSOR_MAP_SWIZZLE_128B);
  // a_scale as [K / 128][T] fp32 rows a_scale_ld apart: one box = one k-block's scales of rows [m0 & ~3, (m0 & ~3) + BM + 4), a
  // 16-byte-aligned start (rows past T zero-filled)
  if (!rc) rc = make_map_2d(&tmS, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a.a_scale, uint64_t(a.total_rows), uint64_t(g.KB),
                            uint64_t(a.a_scale_ld) * 4, SM::kScaleBox, 1, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  const unsigned grid = unsigned(std::min<long long>(max_tiles, (long long)resident_per_sm * device_sm_count()));
  return launch_pdl(kernel, grid, TS_THREADS, SM::kTotal, a.stream, pdl_enabled(), tmA, tmW, tmS, g);
}

template <bool SWIGLU>
int launch_grouped_fp8_bm(const GroupedFp8Args& a, const GroupedFp8Params& g) {
  // rows of A per tile from the mean rows per active group (T rows over at most min(E, T) groups), as launch_grouped_gemm_bm
  // picks it; tiles: sum_e ceil(m_e / BM) per n-tile <= ceil(T / BM) + (groups with rows)
  const int active = std::min(a.num_groups, a.total_rows);
  const int mean_rows = (a.total_rows + active - 1) / active;
  const int bm = mean_rows <= 32 ? 32 : (mean_rows <= 64 ? 64 : 128);
  const long long max_tiles = (long long)(g.N / TS_ROWS) * ((a.total_rows + bm - 1) / bm + active);
  if (bm == 32) return launch_grouped_fp8_inst<32, SWIGLU>(a, g, max_tiles);
  if (bm == 64) return launch_grouped_fp8_inst<64, SWIGLU>(a, g, max_tiles);
  return launch_grouped_fp8_inst<128, SWIGLU>(a, g, max_tiles);
}

}  // namespace

int launch_grouped_fp8(const GroupedFp8Args& a) {
  const bb_matmul_desc& d = a.d;
  if ((long long)(d.N / TS_ROWS) * ((a.total_rows + 31) / 32 + std::min(a.num_groups, a.total_rows)) > INT_MAX) {
    set_error("grouped FP8 GEMM: N/128 x (T/32 + groups) exceeds 2^31 tiles");
    return 1;
  }
  if ((long long)a.num_groups * d.N > INT_MAX) {   // the kernel's weight row e * N + n0 is an int
    set_error("grouped FP8 GEMM: num_groups x N exceeds 2^31 weight rows");
    return 1;
  }
  GroupedFp8Params g;
  g.offsets = a.offsets; g.E = a.num_groups; g.T = a.total_rows;
  g.w_scale = a.w_scale;
  g.s_rows = a.swiglu ? 2 * ((d.N / 2 + FP8_KB - 1) / FP8_KB) : d.N / TS_ROWS;
  g.C = a.C; g.N = d.N; g.KB = d.K / FP8_KB; g.out_dtype = d.out_dtype;
  return a.swiglu ? launch_grouped_fp8_bm<true>(a, g) : launch_grouped_fp8_bm<false>(a, g);
}

}  // namespace bb
