// bb_grouped_gemm.cu -- grouped wgmma GEMM for mixture-of-experts prefill (bb_matmul_grouped_gemm): ONE launch over E experts,
//   C[offsets[e] : offsets[e+1]] = A[offsets[e] : offsets[e+1]] x dequant(W[e])^T (+ bias[e])     for every e,
// with the row offsets read on the device, at any number of rows per expert.
//
// Design:
//   * the per-tile arithmetic is gemm_ts_kernel's (bb_gemm_ts.cuh, DESIGN.md §3.1): a TMA producer warp, two consumer warpgroups
//     that decode the packed weights with LOP3 straight into wgmma A fragments, per-row group parameters fetched one group ahead,
//     and the same epilogue.  Numerics are those of bb_matmul on the wgmma GEMM; there is no split-K.
//   * operands: A [T, K] is one 2-D tensor map over all T rows; a tile of expert e starts at row offsets[e] + mt * BM.  Rows
//     past the expert's end belong to the next expert and are loaded but never stored; rows past T are zero-filled by TMA.  The
//     stacked W [E, N, K * bits / 8] is one 2-D map of E * N rows, and expert e's n-tile starts at row e * N + n0.  Neither map
//     depends on the offsets, so the launch is graph-capturable.
//   * the grid is persistent (an upper bound of the tiles, capped at the resident CTAs).  Every CTA clamps the offsets and counts
//     each expert's tiles, ceil(m_e / BM) * N / 128, with the grouped GEMV's warp prefix sum (grouped_schedule), then walks the
//     tiles blockIdx.x, blockIdx.x + gridDim.x, ...; an empty expert costs nothing.  Within an expert the m-tiles of one n-tile
//     are consecutive, so CTAs running at the same time share the weight tile in L2.
//   * the mbarrier ring (stage index and parity) runs on from one tile to the next: the producer loads the next tile's first
//     k-blocks while the consumers finish the MMAs and the epilogue of the current one.
//   * BM (32, 64 or 128 rows of A per tile) is chosen on the host from the mean rows per active expert.
//   * programmatic dependent launch as in bb_grouped.cu: griddepcontrol.wait comes first (which experts to stream is unknown until
//     the offsets are read); launch_dependents follows the CTA's last tile.
//   * the offsets are untrusted, with bb_matmul_grouped's contract: clamped to [0, T], a group whose end is below its start is
//     empty, and rows no group claims are not written.
//   * SWIGLU instances (bb_matmul_grouped_gemm_swiglu): gate/up interleaved W, C [T, N / 2] = silu(gate) * up (store_tile).
//   * GATHER instances (bb_matmul_grouped_gemm_swiglu_gather, SWIGLU only): sorted row r reads A[clamp(row_index[r], 0, a_rows - 1)]
//     of A [a_rows, K], so a mixture-of-experts block reads its token rows in place instead of a routed copy.  Only the producer
//     differs: TS_GATHER_WARPS producer warps (the launch has 3 more warps) copy the tile's rows with 16-byte cp.async, 8 lanes
//     per 128-byte row, straight into the SW128 layout the consumers' descriptor reads (chunk c of row i at byte
//     i * 128 + (c ^ (i & 7)) * 16 of the 1024-byte-aligned stage); each lane's cp.async.mbarrier.arrive and one arrival per
//     producer warp join the stage's `full` barrier next to the weight TMA.  One TMA box {KB, 1} per row gives the same bits
//     (TMA swizzles by the shared-memory address) but issues BM TMA operations per k-block and was slower still.  Rows past the
//     expert's end are not copied (they are never stored, and a wgmma output column depends on its own activation row only).
//     The consumers add one fence.proxy.async per stage: the cp.async writes are generic-proxy writes that wgmma reads through
//     the async proxy.  tmA is not used (the launch passes tmW in its place).
#include <algorithm>
#include <climits>

#include "bb_gemm_ts.cuh"

namespace bb {

namespace {

struct GroupedTsParams {
  TsParams p;                 // the problem of group 0 (p.M = T; p.out: C with row stride N; p.splits = 1)
  const int32_t* offsets;     // [E + 1], device
  int E;                      // groups
  int T;                      // rows of A and C
  long long s_stride, z_stride, b_stride;   // bytes per group: scale, zeros, bias
  const int32_t* row_index;   // [T], device (GATHER)
  const void* a;              // A [a_rows, K] (GATHER)
  int a_rows;
};

// the mbarrier's phase also waits for this thread's earlier cp.async copies (net-zero on its pending count)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// gemm_ts_kernel's epilogue for one destination and no split-K: acc[4i + 2h + j] = C^T[row rA + 8h][column 8i + 2t + j] ->
// C[m, n] for the rows m < m_end, cast to out_dtype, then bias[e][n] added in out_dtype (fp32: in one sum), as bb_matmul rounds.
// SWIGLU: store_tile_swiglu (bb_gemm_ts.cuh)
template <typename T, int BM, bool SWIGLU>
__device__ __forceinline__ void store_tile(const float (&acc)[BM / 2], const TsParams& p, const T* bias, int m0, int m_end,
                                           int nA, int nB, int t) {
  if constexpr (SWIGLU) {
    store_tile_swiglu<T, BM>(acc, p, bias, m0, m_end, nA, nB, t);
  } else {
    float bias_f[2] = {0.f, 0.f};
    if (bias) {
      bias_f[0] = TypeTraits<T>::to_float(bias[nA]);
      bias_f[1] = TypeTraits<T>::to_float(bias[nB]);
    }
    void* const C = p.out.ptr[0];
#pragma unroll
    for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int m = m0 + 8 * i + 2 * t + j;
        if (m >= m_end) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v = acc[4 * i + 2 * h + j];
          const size_t o = size_t(m) * size_t(p.N) + size_t(h ? nB : nA);
          if (p.out_dtype == BB_F16) {
            __half r = __float2half_rn(v);
            if (bias) r = __hadd(r, __float2half_rn(bias_f[h]));
            reinterpret_cast<__half*>(C)[o] = r;
          } else if (p.out_dtype == BB_BF16) {
            __nv_bfloat16 r = __float2bfloat16_rn(v);
            if (bias) r = __hadd(r, __float2bfloat16_rn(bias_f[h]));
            reinterpret_cast<__nv_bfloat16*>(C)[o] = r;
          } else {
            reinterpret_cast<float*>(C)[o] = v + (bias ? bias_f[h] : 0.f);
          }
        }
      }
    }
  }
}

// producer warps of the GATHER instances: one warp issuing the 16-byte copies left the gathering GEMM 1.8-3.8x slower than the
// plain one, four bring it to 1.06-1.55x (H100 80GB HBM3, 700 W, tools/moe_bench.py shapes)
constexpr int TS_GATHER_WARPS = 4;

template <bool GATHER>
constexpr int grouped_threads() { return TS_THREADS + (GATHER ? 32 * (TS_GATHER_WARPS - 1) : 0); }

template <typename T, int BITS, int BM, bool IL, bool SWIGLU = false, bool GATHER = false>
__global__ void __launch_bounds__(grouped_threads<GATHER>(), 1)
gemm_ts_grouped_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                       const GroupedTsParams g) {
  using SM = TsSmem<T, BITS, BM>;
  constexpr int S = SM::kStages;
  constexpr int KB = ElemInfo<T>::kKB;
  constexpr int PRB = SM::kPRB;
  const TsParams& p = g.p;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sW = smem + S * SM::kActBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * SM::kStageBytes);
  uint64_t* full = bars;                 // [S]   TMA -> consumers
  uint64_t* empty = bars + S;            // [S]   consumer warps -> TMA
  __shared__ int row0_s[BB_GROUPED_MAX_GROUPS];       // clamped first row of each group
  __shared__ int rows_s[BB_GROUPED_MAX_GROUPS];       // rows of each group (0: empty)
  __shared__ int item0_s[BB_GROUPED_MAX_GROUPS + 1];  // first tile of each group; item0_s[E] = all tiles

  pdl_wait();   // offsets and A are the preceding kernels' output; nothing is read before this (see the header)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = p.N / TS_ROWS;
  const int num_kb = p.K / KB;
  if (warp == TS_CONSUMER_WARPS && lane == 0) {
    if constexpr (!GATHER) tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    // GATHER: `full` completes on one arrival per producer warp (plus the weight bytes and every lane's cp.async copies)
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], GATHER ? TS_GATHER_WARPS : 1); mbar_init(&empty[i], TS_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  if (threadIdx.x < 32) grouped_schedule(g, BM, n_tiles, row0_s, rows_s, item0_s);
  __syncthreads();
  const int total = item0_s[g.E];

  // tile `item`: expert e, activation rows [m0, m_end) of which the tile holds the first BM, expert-local weight rows n0 + 128
  auto tile_of = [&](int item, int& e, int& m0, int& m_end, int& n0) {
    e = grouped_find(item0_s, g.E, item);
    const int local = item - item0_s[e];
    const int m_tiles = (rows_s[e] + BM - 1) / BM;
    const int nt = local / m_tiles;
    m0 = row0_s[e] + (local - nt * m_tiles) * BM;
    m_end = row0_s[e] + rows_s[e];
    n0 = nt * TS_ROWS;
  };

  if (GATHER ? warp >= TS_CONSUMER_WARPS : warp == TS_CONSUMER_WARPS) {
    // ===== TMA producer: one continuous ring over all of this CTA's tiles =====
    if constexpr (GATHER) {
      // producer warp pw owns tile rows [pw * RW, (pw + 1) * RW): it reads their indices once per tile (only it uses them, so
      // __syncwarp orders the reuse) and copies them every k-block, 8 lanes per 128-byte row
      constexpr int RW = BM / TS_GATHER_WARPS;
      __shared__ int src_s[BM];   // clamped source row of each tile row; -1 past the expert's end
      const int pw = warp - TS_CONSUMER_WARPS;
      int* const src_w = src_s + pw * RW;
      const int c = lane & 7;     // the 16-byte chunk of a 128-byte row this lane copies
      const T* a = reinterpret_cast<const T*>(g.a) + c * 8;
      int s = 0, loads = 0;
      uint32_t par = 1;
      for (int item = blockIdx.x; item < total; item += gridDim.x) {
        int e, m0, m_end, n0;
        tile_of(item, e, m0, m_end, n0);
        const int wrow = e * p.N + n0;
        const int r0 = m0 + pw * RW;
        __syncwarp();   // the previous tile's src_w reads are done
        for (int i = lane; i < RW; i += 32) src_w[i] = r0 + i < m_end ? min(max(g.row_index[r0 + i], 0), g.a_rows - 1) : -1;
        __syncwarp();
        for (int kb = 0; kb < num_kb; ++kb, ++loads) {
          if (loads >= S) mbar_wait(&empty[s], par);
          const uint32_t dst = smem_u32(sA + s * SM::kActBytes) + uint32_t(c << 4);
#pragma unroll
          for (int i = lane >> 3; i < RW; i += 4) {
            const int r = src_w[i], row = pw * RW + i;
            if (r >= 0) cp_async16((dst + uint32_t(row * 128)) ^ uint32_t((row & 7) << 4), a + size_t(r) * p.K + kb * KB);
          }
          cp_async_mbar_arrive(&full[s]);
          __syncwarp();   // every lane's tracking is registered before the warp's arrival can complete the phase
          if (lane == 0) {
            if (pw == 0) {
              mbar_arrive_expect_tx(&full[s], SM::kWBytes);
              tma_load_2d(sW + s * SM::kWBytes, &tmW, kb * PRB, wrow, &full[s]);
            } else {
              mbar_arrive(&full[s]);
            }
          }
          if (++s == S) { s = 0; par ^= 1; }
        }
      }
    } else if (lane == 0) {
      int s = 0, loads = 0;
      uint32_t par = 1;  // parity of the "previous use" of the stage: the first pass must not wait
      for (int item = blockIdx.x; item < total; item += gridDim.x) {
        int e, m0, m_end, n0;
        tile_of(item, e, m0, m_end, n0);
        const int wrow = e * p.N + n0;
        for (int kb = 0; kb < num_kb; ++kb, ++loads) {
          if (loads >= S) mbar_wait(&empty[s], par);
          mbar_arrive_expect_tx(&full[s], SM::kStageBytes);
          tma_load_2d(sA + s * SM::kActBytes, &tmA, kb * KB, m0, &full[s]);
          tma_load_2d(sW + s * SM::kWBytes, &tmW, kb * PRB, wrow, &full[s]);
          if (++s == S) { s = 0; par ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups: decode + wgmma, then the epilogue, tile after tile =====
  const int g8 = lane >> 2, t = lane & 3;
  const int rA = (warp >> 2) * 64 + (warp & 3) * 16 + g8;   // fragment rows rA and rA + 8 of this thread (tile-local)
  constexpr uint32_t MAGIC = TypeTraits<T>::kMagic;
  const uint32_t srcA = smem_u32(sW) + uint32_t(rA * PRB), srcB = srcA + 8u * PRB;
  Lut4 lut4;   // unused by the integer formats

  auto tiles = [&](auto mode_tag) {
    constexpr int MODE = decltype(mode_tag)::value;
    constexpr int EPB = 8 / BITS;
    const int kb_per_g = p.g / KB;
    int st = 0;
    uint32_t full_par = 0;
    for (int item = blockIdx.x; item < total; item += gridDim.x) {
      int e, m0, m_end, n0;
      tile_of(item, e, m0, m_end, n0);
      const int nA = n0 + rA, nB = nA + 8;   // expert-local weight rows
      float acc[BM / 2];
#pragma unroll
      for (int i = 0; i < BM / 2; ++i) acc[i] = 0.f;
      DqConst cA, cB;
      cA.mz_lo = cA.mz_hi = MAGIC + uint32_t(p.zp_const) * 0x00010001u;
      cA.z2 = cA.s2 = cA.negz2 = 0;
      cB = cA;
      RowGroup<MODE, BITS> gA, gB;
      const uint16_t* sc = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(p.scale) + size_t(e) * size_t(g.s_stride));
      const uint8_t* zb = reinterpret_cast<const uint8_t*>(p.zeros) + size_t(e) * size_t(g.z_stride);
      gA.sc = sc + size_t(nA) * p.G;
      gB.sc = sc + size_t(nB) * p.G;
      gA.z = reinterpret_cast<const uint16_t*>(zb) + size_t(nA) * p.G;
      gB.z = reinterpret_cast<const uint16_t*>(zb) + size_t(nB) * p.G;
      gA.qz = zb + nA / EPB;
      gB.qz = zb + nB / EPB;
      gA.qz_stride = gB.qz_stride = size_t(p.N) * BITS / 8;
      gA.qz_shift = BITS * (nA % EPB);
      gB.qz_shift = BITS * (nB % EPB);
      int gi = 0;       // group of the next k-block
      int g_end = 0;    // k-block at which group gi starts
      if constexpr (MODE != 0) { gA.fetch(gi); gB.fetch(gi); }

      int prev_st = -1;
      auto step = [&](int kb, uint32_t (&fa)[8], uint32_t (&fb)[8]) {
        if constexpr (MODE != 0) {
          if (kb >= g_end) {   // entering group gi: its parameters were fetched one group ago; fetch the next one now
            gA.apply(cA, MAGIC);
            gB.apply(cB, MAGIC);
            g_end += kb_per_g;
            ++gi;
            if (gi < p.G && g_end < num_kb) { gA.fetch(gi); gB.fetch(gi); }
          }
        }
        mbar_wait(&full[st], full_par);
        if constexpr (GATHER) fence_proxy_async_shared();
        const uint32_t wofs = uint32_t(st * SM::kWBytes);
        dequant_row<T, BITS, MODE, IL, 0>(srcA + wofs, t, fa, cA, lut4, false);
        dequant_row<T, BITS, MODE, IL, 0>(srcB + wofs, t, fb, cB, lut4, false);
        const uint64_t bdesc = make_sw128_desc(smem_u32(sA + st * SM::kActBytes));
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const uint32_t a[4] = {fa[2 * s], fb[2 * s], fa[2 * s + 1], fb[2 * s + 1]};
          Wgmma<BM>::template f16<T>(acc, a, bdesc + uint64_t(2 * s), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the MMAs of the previous k-block are done: its fragments and smem stage are free
        if (prev_st >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev_st]);
        }
        prev_st = st;
        if (++st == S) { st = 0; full_par ^= 1; }
      };
      uint32_t fa0[8], fb0[8], fa1[8], fb1[8];
      int kb = 0;
      for (; kb + 1 < num_kb; kb += 2) {
        step(kb, fa0, fb0);
        step(kb + 1, fa1, fb1);
      }
      if (kb < num_kb) step(kb, fa0, fb0);
      wgmma_wait<0>();
      __syncwarp();   // the tile's last stage is free too: the producer is already filling the others with the next tile
      if (lane == 0) mbar_arrive(&empty[prev_st]);
      const T* bias = p.bias ? reinterpret_cast<const T*>(reinterpret_cast<const uint8_t*>(p.bias) + size_t(e) * size_t(g.b_stride))
                             : nullptr;
      store_tile<T, BM, SWIGLU>(acc, p, bias, m0, m_end, nA, nB, t);
    }
  };
  switch (p.mode) {
    case 0: tiles(std::integral_constant<int, 0>{}); break;
    case 1: tiles(std::integral_constant<int, 1>{}); break;
    case 2: tiles(std::integral_constant<int, 2>{}); break;
    case 3: tiles(std::integral_constant<int, 3>{}); break;
    default: tiles(std::integral_constant<int, 4>{}); break;
  }
  pdl_launch_dependents();
}

template <typename T, int BITS, int BM, bool IL, bool SWIGLU, bool GATHER>
int launch_grouped_gemm_inst(const GroupedTsParams& g, const void* A, const void* W, long long max_tiles, cudaStream_t stream) {
  using SM = TsSmem<T, BITS, BM>;
  auto kernel = gemm_ts_grouped_kernel<T, BITS, BM, IL, SWIGLU, GATHER>;
  constexpr int threads = grouped_threads<GATHER>();
  static KernelCache<> cache;
  const int resident_per_sm = kernel_setup(cache, kernel, SM::kTotal, threads, SM::kTotal);
  if (resident_per_sm <= 0) { set_error("grouped GEMM: the kernel cannot be resident on this device"); return 2; }
  CUtensorMap tmA, tmW;
  const CUtensorMapDataType adt = std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const TsParams& p = g.p;
  const uint64_t wrow = uint64_t(p.K) * BITS / 8;
  int rc = make_map_2d(&tmW, CU_TENSOR_MAP_DATA_TYPE_UINT8, W, wrow, uint64_t(g.E) * uint64_t(p.N), wrow, SM::kPRB, TS_ROWS,
                       CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  if constexpr (GATHER) {
    tmA = tmW;   // the producer copies A with cp.async; the kernel never touches tmA
  } else {
    rc = make_map_2d(&tmA, adt, A, uint64_t(p.K), uint64_t(g.T), uint64_t(p.K) * sizeof(T), ElemInfo<T>::kKB, BM,
                     CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const unsigned grid = unsigned(std::min<long long>(max_tiles, (long long)resident_per_sm * device_sm_count()));
  return launch_pdl(kernel, grid, threads, SM::kTotal, stream, pdl_enabled(), tmA, tmW, g);
}

template <typename T, int BITS, bool IL, bool SWIGLU, bool GATHER>
int launch_grouped_gemm_bm(const GroupedTsParams& g, const void* A, const void* W, cudaStream_t stream) {
  // rows of A per tile from the mean rows per active group (T rows over at most min(E, T) groups), as launch_ts_bm picks BM
  // from m; tiles: sum_e ceil(m_e / BM) per n-tile <= ceil(T / BM) + (groups with rows)
  const int active = std::min(g.E, g.T);
  const int mean_rows = (g.T + active - 1) / active;
  const int bm = mean_rows <= 32 ? 32 : (mean_rows <= 64 ? 64 : 128);
  const long long max_tiles = (long long)(g.p.N / TS_ROWS) * ((g.T + bm - 1) / bm + active);
  if (bm == 32) return launch_grouped_gemm_inst<T, BITS, 32, IL, SWIGLU, GATHER>(g, A, W, max_tiles, stream);
  if (bm == 64) return launch_grouped_gemm_inst<T, BITS, 64, IL, SWIGLU, GATHER>(g, A, W, max_tiles, stream);
  return launch_grouped_gemm_inst<T, BITS, 128, IL, SWIGLU, GATHER>(g, A, W, max_tiles, stream);
}

template <bool SWIGLU, bool GATHER = false>
int launch_grouped_gemm_typed(const bb_matmul_desc& d, const GroupedTsParams& g, const void* A, const void* W, cudaStream_t s) {
  return dispatch_t_bits_il(d, [&](auto t, auto bits, auto il) {
    return launch_grouped_gemm_bm<typename decltype(t)::type, decltype(bits)::value, decltype(il)::value, SWIGLU, GATHER>(g, A, W, s);
  });
}

}  // namespace

// grouped_supported (bb_grouped.cu) plus the CTA tile of 128 weight rows; sets the error message otherwise
bool grouped_gemm_supported(const bb_matmul_desc& d) {
  if (!grouped_supported(d)) return false;
  if (d.N % TS_ROWS) {
    set_error("grouped GEMM: needs N %% 128 == 0 (N=%d); bb_matmul_grouped covers N %% 16 == 0", d.N);
    return false;
  }
  return true;
}

int launch_grouped_gemm(const GroupedArgs& a) {
  const bb_matmul_desc& d = a.d;
  GroupedTsParams g;
  g.p = make_ts_params(d, a.scale, a.zeros, a.bias, nullptr, make_outspec(a.C, d.N), a.total_rows);
  g.p.splits = 1; g.p.kb_per_split = d.K / 64; g.p.ws = nullptr; g.p.w_tiled = 0;
  g.offsets = a.offsets; g.E = a.num_groups; g.T = a.total_rows;
  g.s_stride = a.s_stride; g.z_stride = a.z_stride; g.b_stride = a.b_stride;
  g.row_index = a.row_index; g.a = a.A; g.a_rows = a.a_rows;
  if ((long long)(d.N / TS_ROWS) * ((a.total_rows + 31) / 32 + std::min(a.num_groups, a.total_rows)) > INT_MAX) {
    set_error("grouped GEMM: N/128 x (T/32 + groups) exceeds 2^31 tiles");
    return 1;
  }
  if (a.row_index) return launch_grouped_gemm_typed<true, true>(d, g, a.A, a.W, a.stream);
  return a.swiglu ? launch_grouped_gemm_typed<true>(d, g, a.A, a.W, a.stream)
                  : launch_grouped_gemm_typed<false>(d, g, a.A, a.W, a.stream);
}

}  // namespace bb
