// bb_gemm_ts.cu -- the tensor-core path: Hopper wgmma with the dequantised weights as the register ("RS") operand.
//
// Replaces the reference's generated mma.sync GEMM (bitblas/ops/general_matmul/tilelang/dequantize/
// matmul_dequantize_mma.py:333-506: cp.async -> smem(int8) -> regs -> LOP3 decode -> smem(fp16) -> ldmatrix
// -> mma.sync m16n8k16).  On H100 the decoded weights never touch shared memory:
//
//     C^T[n, m] = sum_k  Wdeq[n, k] * A[m, k]            (the operands are swapped: W is the MMA "A"/M side)
//
//   TMA warp      : per k-block, one 2-D tile of activations A[BM x 64] (fp16/bf16; 128 int8) into 128B-swizzled
//                   shared memory (the wgmma "B"/N operand, K-major) and one tile of PACKED weights
//                   W[128 rows x 32 B] (4-bit) -- 8x fewer bytes than a dequantised tile;
//   2 warpgroups  : each owns 64 weight rows.  A thread reads the packed bytes of its two fragment rows (g, g + 8) from
//                   shared memory, decodes them with LOP3 / PRMT + (w-z)*s straight into the register layout of the wgmma
//                   A fragment, and issues wgmma.mma_async m64nBMk16 (k32 for int8) with the activation tile as the smem
//                   descriptor operand; fp32 (s32) accumulators stay in registers.  Fragments are double-buffered: the
//                   decode of k-block kb + 1 overlaps the MMAs of kb, and wgmma.wait_group 1 releases the smem stage of kb - 1;
//   epilogue      : the accumulators are cast, biased and stored as C[m, n].
//
// Shared-memory traffic per k-block is therefore A-tile (TMA write + MMA read) + 4 KB packed W, instead of also writing and
// re-reading a 16-32 KB dequantised W tile (DESIGN.md §3.1).
#include <algorithm>

#include "bb_gemm_ts.cuh"

namespace bb {

namespace {

// FMT: 0 = integer formats (LOP3 magic-number decode), 1 = 16-entry table formats (NF4 / fp4; BITS = 4, compressed storage),
//      2 = 8-bit float weights (e4m3 / e5m2; BITS = 8).  F = SwiGLU (16-bit activations only): bb_matmul_swiglu -- without split-K
//      the epilogue is store_tile_swiglu; with it the raw partials are written as in the plain instance and splitk_reduce_kernel
//      forms silu(gate) * up.  F = Scaled (int8 activations only): bb_matmul_scaled -- without split-K the tile is stored through
//      store_out_scaled; with it the raw int32 partials are written as in the plain instance and splitk_reduce_kernel scales them.
//      The scales are a parameter of their own (null in every other instance): TsParams is also the grouped GEMM's.
//      F = W4A8 (int8 activations, 4-bit weights): bb_matmul_w4a8 -- per-group fp32 scales (sc.w_scale [N, G]) and zero points,
//      promoted from exact int32 group sums into fp32 (main loop below); the tile, or the split's fp32 partial, ends in
//      store_out_dequant / splitk_reduce_w4a8.
template <typename T, int BITS, int BM, bool IL, int FMT, MatmulForm F>
__global__ void __launch_bounds__(TS_THREADS, 1)
gemm_ts_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const TsParams p,
               const ScaledArgs sc) {
  using SM = TsSmem<T, BITS, BM>;
  using EI = ElemInfo<T>;
  constexpr int S = SM::kStages;
  constexpr int KB = EI::kKB;
  constexpr int PRB = SM::kPRB;
  constexpr bool INT8 = EI::kInt8;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sW = smem + S * SM::kActBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * SM::kStageBytes);
  uint64_t* full = bars;                 // [S]   TMA -> consumers
  uint64_t* empty = bars + S;            // [S]   consumer warps -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x % p.splits;
  const int tile = blockIdx.x / p.splits;
  const int m_tile = tile % p.m_tiles;
  const int n_tile = tile / p.m_tiles;
  const int kb0 = split * p.kb_per_split;  // first k-block of this CTA
  const int m0 = m_tile * BM, n0 = n_tile * TS_ROWS;
  const int num_kb = p.kb_per_split;

  if (warp == TS_CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TS_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TS_CONSUMER_WARPS) {
    // ===== TMA producer =====
    if (lane == 0) {
      int s = 0;
      uint32_t par = 1;  // parity of the "previous use" of the stage: first pass must not wait
      for (int kb = 0; kb < num_kb; ++kb) {
        if (kb >= S) mbar_wait(&empty[s], par);
        mbar_arrive_expect_tx(&full[s], SM::kStageBytes);
        tma_load_2d(sA + s * SM::kActBytes, &tmA, (kb0 + kb) * KB, m0, &full[s]);
        if (p.w_tiled) {   // the same 128 x PRB bytes, gathered from four 32-row blocks of the slab-tiled storage
          const int byte = (kb0 + kb) * PRB;
          tma_load_4d(sW + s * SM::kWBytes, &tmW, byte % BB_TILE_ROW_BYTES, 0, byte / BB_TILE_ROW_BYTES, n0 / BB_TILE_ROWS, &full[s]);
        } else {
          tma_load_2d(sW + s * SM::kWBytes, &tmW, (kb0 + kb) * PRB, n0, &full[s]);
        }
        if (++s == S) { s = 0; par ^= 1; }
      }
    }
    return;
  }

  // ===== consumer warpgroups: decode + wgmma, then the epilogue =====
  const int g8 = lane >> 2, t = lane & 3;
  const int rA = (warp >> 2) * 64 + (warp & 3) * 16 + g8;   // fragment rows rA and rA + 8 of this thread (tile-local)
  const int nA = n0 + rA, nB = nA + 8;
  using TF = typename std::conditional<INT8, __half, T>::type;  // 16-bit element type of the float path
  constexpr uint32_t MAGIC = INT8 ? 0u : TypeTraits<TF>::kMagic;
  using Acc = typename std::conditional<INT8, uint32_t, float>::type;
  Acc acc[BM / 2];
#pragma unroll
  for (int i = 0; i < BM / 2; ++i) acc[i] = Acc(0);

  Lut4 lut4;
  if constexpr (FMT == 1) lut4_init(lut4, p.w_fmt, std::is_same<TF, __nv_bfloat16>::value, p.lut);
  const bool e5m2 = p.w_fmt == BB_W_FP8_E5M2;
  const uint32_t zp4 = uint32_t(p.zp_const) * 0x01010101u;
  const uint32_t srcA = smem_u32(sW) + uint32_t(rA * PRB), srcB = srcA + 8u * PRB;

  if constexpr (F == MatmulForm::W4A8) {
    // Each group's k-blocks accumulate, exactly, into acc; the first wgmma of a group overwrites it (scale-d = 0).  Every k-block
    // decodes its fragments while the previous k-block's MMAs run, then wait<0> retires those MMAs; at a group's first k-block
    // the finished group is promoted into facc with its scale, and the new MMAs are issued.  So one k-block's MMAs are in flight
    // during each decode, and the tensor pipe drains once per k-block (at g = 128 every k-block closes a group anyway).  The
    // loop body is the same for every k-block: whether it opens a group only selects values (the promotion, scale-d).  A branch
    // on it, or on the group size, around the wait or the wgmmas makes ptxas serialize every wgmma (C7515 / C7520).  A split
    // starts on a group boundary (launch_ts_inst).
    float facc[BM / 2];
#pragma unroll
    for (int i = 0; i < BM / 2; ++i) facc[i] = 0.f;
    const float* scA = sc.w_scale + size_t(nA) * p.G;
    const float* scB = sc.w_scale + size_t(nB) * p.G;
    const uint8_t* qz = reinterpret_cast<const uint8_t*>(p.zeros);
    const int kpg = p.g / KB;                      // k-blocks per group
    // zero bytes and scales of the next k-block's group (fetched one k-block ahead), of this k-block's, and the previous
    // k-block's scale (0 before the first: promoting the zeroed acc then adds 0)
    uint32_t nzA, nzB;
    float nscA, nscB, pscA = 0.f, pscB = 0.f;
    auto fetch = [&](int kb) {
      const int g = min((kb0 + kb) / kpg, p.G - 1);
      nzA = uint32_t(w4a8_zero(qz, p.N, g, nA, p.zp_const)) * 0x01010101u;
      nzB = uint32_t(w4a8_zero(qz, p.N, g, nB, p.zp_const)) * 0x01010101u;
      nscA = __ldg(scA + g);
      nscB = __ldg(scB + g);
    };
    fetch(0);
    int st = 0;
    uint32_t full_par = 0;
    int prev_st = -1;
    auto step = [&](int kb, uint32_t (&fa)[8], uint32_t (&fb)[8]) {
      const uint32_t zA = nzA, zB = nzB;
      const float scaleA = nscA, scaleB = nscB;
      const bool start = kb % kpg == 0;
      fetch(kb + 1);
      mbar_wait(&full[st], full_par);
      const uint32_t wofs = uint32_t(st * SM::kWBytes);
      dequant_row_i8<BITS, IL>(srcA + wofs, t, fa, zA);   // bytes u - z, signed
      dequant_row_i8<BITS, IL>(srcB + wofs, t, fb, zB);
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BM / 2; ++i) {
        const float f = w4a8_promote(facc[i], int(acc[i]), ((i >> 1) & 1) ? pscB : pscA);
        facc[i] = start ? f : facc[i];
      }
      const uint64_t bdesc = make_sw128_desc(smem_u32(sA + st * SM::kActBytes));
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const uint32_t a[4] = {fa[2 * s], fb[2 * s], fa[2 * s + 1], fb[2 * s + 1]};
        Wgmma<BM>::template i8<true>(acc, a, bdesc + uint64_t(2 * s), (s == 0 && start) ? 0u : 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the MMAs of the previous k-block are done: its fragments and smem stage are free
      if (prev_st >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev_st]);
      }
      prev_st = st;
      if (++st == S) { st = 0; full_par ^= 1; }
      pscA = scaleA; pscB = scaleB;
    };
    uint32_t fa0[8], fb0[8], fa1[8], fb1[8];
    int kb = 0;
    for (; kb + 1 < num_kb; kb += 2) {
      step(kb, fa0, fb0);
      step(kb + 1, fa1, fb1);
    }
    if (kb < num_kb) step(kb, fa0, fb0);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BM / 2; ++i) facc[i] = w4a8_promote(facc[i], int(acc[i]), ((i >> 1) & 1) ? pscB : pscA);

    // ----- epilogue: facc[4i + 2h + j] = S^T[row rA + 8h][column 8i + 2t + j] -----
#pragma unroll
    for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int m = m0 + 8 * i + 2 * t + j;
        if (m >= p.M) continue;
        if (p.splits > 1) {   // the split's fp32 partial; splitk_reduce_w4a8 sums the splits in order
          float* ws = reinterpret_cast<float*>(p.ws) + (size_t(split) * p.M + m) * p.N;
          ws[nA] = facc[4 * i + j];
          ws[nB] = facc[4 * i + 2 + j];
          continue;
        }
        const float sa = sc.a_scale[m];
        store_out_dequant(p.out.ptr[0], size_t(m) * p.N + nA, __fdiv_rn(facc[4 * i + j], sa), p.bias, nA, p.out_dtype);
        store_out_dequant(p.out.ptr[0], size_t(m) * p.N + nB, __fdiv_rn(facc[4 * i + 2 + j], sa), p.bias, nB, p.out_dtype);
      }
    }
    return;
  }

  auto main_loop = [&](auto mode_tag) {
    constexpr int MODE = decltype(mode_tag)::value;
    DqConst cA, cB;
    cA.mz_lo = cA.mz_hi = MAGIC + uint32_t(p.zp_const) * 0x00010001u;
    cA.z2 = cA.s2 = cA.negz2 = 0;
    cB = cA;
    RowGroup<MODE, BITS> gA, gB;
    constexpr int EPB = 8 / BITS;
    gA.sc = reinterpret_cast<const uint16_t*>(p.scale) + size_t(nA) * p.G;
    gB.sc = reinterpret_cast<const uint16_t*>(p.scale) + size_t(nB) * p.G;
    gA.z = reinterpret_cast<const uint16_t*>(p.zeros) + size_t(nA) * p.G;
    gB.z = reinterpret_cast<const uint16_t*>(p.zeros) + size_t(nB) * p.G;
    gA.qz = reinterpret_cast<const uint8_t*>(p.zeros) + nA / EPB;
    gB.qz = reinterpret_cast<const uint8_t*>(p.zeros) + nB / EPB;
    gA.qz_stride = gB.qz_stride = size_t(p.N) * BITS / 8;
    gA.qz_shift = BITS * (nA % EPB);
    gB.qz_shift = BITS * (nB % EPB);
    const int kb_per_g = p.g / KB;
    int gi = kb0 / kb_per_g;                 // group of the next k-block
    int g_end = gi * kb_per_g - kb0;         // CTA-local k-block at which group gi starts (<= 0 for the first)
    if constexpr (MODE != 0) { gA.fetch(gi); gB.fetch(gi); }

    int st = 0;
    uint32_t full_par = 0;
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
      const uint32_t wofs = uint32_t(st * SM::kWBytes);
      if constexpr (INT8) {
        dequant_row_i8<BITS, IL>(srcA + wofs, t, fa, zp4);
        dequant_row_i8<BITS, IL>(srcB + wofs, t, fb, zp4);
      } else {
        dequant_row<TF, BITS, MODE, IL, FMT>(srcA + wofs, t, fa, cA, lut4, e5m2);
        dequant_row<TF, BITS, MODE, IL, FMT>(srcB + wofs, t, fb, cB, lut4, e5m2);
      }
      const uint64_t bdesc = make_sw128_desc(smem_u32(sA + st * SM::kActBytes));
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const uint32_t a[4] = {fa[2 * s], fb[2 * s], fa[2 * s + 1], fb[2 * s + 1]};
        if constexpr (INT8) {
          if (p.zp_const) Wgmma<BM>::template i8<true>(acc, a, bdesc + uint64_t(2 * s), 1u);
          else Wgmma<BM>::template i8<false>(acc, a, bdesc + uint64_t(2 * s), 1u);
        } else {
          Wgmma<BM>::template f16<TF>(acc, a, bdesc + uint64_t(2 * s), 1u);
        }
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
  };
  if constexpr (INT8) {
    main_loop(std::integral_constant<int, 0>{});
  } else if constexpr (FMT != 0) {   // table / fp8 formats: no zero points on the fast path (gemm_ts_supported)
    if (p.mode == 0) main_loop(std::integral_constant<int, 0>{}); else main_loop(std::integral_constant<int, 1>{});
  } else {
    switch (p.mode) {
      case 0: main_loop(std::integral_constant<int, 0>{}); break;
      case 1: main_loop(std::integral_constant<int, 1>{}); break;
      case 2: main_loop(std::integral_constant<int, 2>{}); break;
      case 3: main_loop(std::integral_constant<int, 3>{}); break;
      default: main_loop(std::integral_constant<int, 4>{}); break;
    }
  }

  // ----- epilogue: acc[4i + 2h + j] = C^T[row rA + 8h][column 8i + 2t + j] -> C[m, n] -----
  if constexpr (F == MatmulForm::SwiGLU) {
    if (p.splits == 1) {
      store_tile_swiglu<T, BM>(acc, p, reinterpret_cast<const T*>(p.bias), m0, p.M, nA, nB, t);
      return;
    }
  }
  if constexpr (F == MatmulForm::Scaled) {
    if (p.splits == 1) {
      const float swA = sc.w_scale[nA], swB = sc.w_scale[nB];
#pragma unroll
      for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int m = m0 + 8 * i + 2 * t + j;
          if (m >= p.M) continue;
          const float sa = sc.a_scale[m];
          store_out_scaled(p.out.ptr[0], size_t(m) * p.N + nA, int(acc[4 * i + j]), sa, swA, p.bias, nA, p.out_dtype);
          store_out_scaled(p.out.ptr[0], size_t(m) * p.N + nB, int(acc[4 * i + 2 + j]), sa, swB, p.bias, nB, p.out_dtype);
        }
      }
      return;
    }
  }
  float bias_f[2] = {0.f, 0.f};
  if (F != MatmulForm::Scaled && p.bias) {   // (a scaled call's bias is out_dtype, read by splitk_reduce_scaled)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = h ? nB : nA;
      if (p.a_dtype == BB_F16) bias_f[h] = __half2float(reinterpret_cast<const __half*>(p.bias)[n]);
      else if (p.a_dtype == BB_BF16) bias_f[h] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[n]);
      else bias_f[h] = float(reinterpret_cast<const int8_t*>(p.bias)[n]);
    }
  }
  void* const C0 = p.out.ptr[0];
  const int ndst = p.out.n;
  const size_t ld = size_t(p.out.ld), col0 = size_t(p.out.col0);
#pragma unroll
  for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + 8 * i + 2 * t + j;
      if (m >= p.M) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const Acc v = acc[4 * i + 2 * h + j];
        const int n = h ? nB : nA;
        if (p.splits > 1) {  // raw partial accumulator; bias / cast / scatter happen in splitk_reduce_kernel
          reinterpret_cast<Acc*>(p.ws)[(size_t(split) * p.M + m) * p.N + n] = v;
          continue;
        }
        const size_t o = size_t(m) * ld + col0 + size_t(n);
        // destination 0 (the local output, or this rank's own copy) takes the straight-line path; the peers' copies
        // (column-parallel scatter) follow in a loop that is empty otherwise
        if constexpr (INT8) {
          const int a = int(v);
          const int b = int(bias_f[h]);
          store_out_i32(C0, o, a, b, p.out_dtype);
          for (int d = 1; d < ndst; ++d) store_out_i32(p.out.ptr[d], o, a, b, p.out_dtype);
        } else {
          if (p.out_dtype == BB_F16) {
            __half r = __float2half_rn(v);
            if (p.bias) r = __hadd(r, __float2half_rn(bias_f[h]));
            reinterpret_cast<__half*>(C0)[o] = r;
            for (int d = 1; d < ndst; ++d) reinterpret_cast<__half*>(p.out.ptr[d])[o] = r;
          } else if (p.out_dtype == BB_BF16) {
            __nv_bfloat16 r = __float2bfloat16_rn(v);
            if (p.bias) r = __hadd(r, __float2bfloat16_rn(bias_f[h]));
            reinterpret_cast<__nv_bfloat16*>(C0)[o] = r;
            for (int d = 1; d < ndst; ++d) reinterpret_cast<__nv_bfloat16*>(p.out.ptr[d])[o] = r;
          } else {
            const float f = v + (p.bias ? bias_f[h] : 0.f);
            reinterpret_cast<float*>(C0)[o] = f;
            for (int d = 1; d < ndst; ++d) reinterpret_cast<float*>(p.out.ptr[d])[o] = f;
          }
        }
      }
    }
  }
}

// splitk_reduce_kernel of the SwiGLU instances: out[m, c] = silu(g) * u for the output columns c = 8b + i, with g and u the plain
// reduce's values of rows 16b + i and 16b + i + 8 (the same split order and rounding).  One thread = 4 consecutive c, which never
// straddle a block of 8 (N / 2 % 4 == 0): one 128-bit load of gate and one of up partials per split.
__device__ __forceinline__ void splitk_reduce_swiglu(const TsParams& p) {
  const unsigned n4 = unsigned(p.N) >> 3;                 // output quads per row (N / 2 columns)
  const unsigned total4 = unsigned(p.M) * n4;
  const size_t split_stride4 = size_t(p.M) * (unsigned(p.N) >> 2);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const unsigned m = i / n4, c = (i - m * n4) * 4u;
    const unsigned ng = (c >> 3) * 16u + (c & 7u);       // first gate row of the quad; its up rows are 8 further
    const size_t q = (size_t(m) * p.N + ng) >> 2;        // the gate quad's float4 index in one split's [M][N] partials
    float g[4] = {0.f, 0.f, 0.f, 0.f}, u[4] = {0.f, 0.f, 0.f, 0.f};
    for (int sp = 0; sp < p.splits; ++sp) {
      const float4* ws = reinterpret_cast<const float4*>(p.ws) + size_t(sp) * split_stride4 + q;
      const float4 vg = __ldcs(ws), vu = __ldcs(ws + 2);
      g[0] += vg.x; g[1] += vg.y; g[2] += vg.z; g[3] += vg.w;
      u[0] += vu.x; u[1] += vu.y; u[2] += vu.z; u[3] += vu.w;
    }
    const size_t o = size_t(m) * (p.N / 2) + c;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float bg = 0.f, bu = 0.f;
      if (p.bias) {
        if (p.a_dtype == BB_F16) {
          bg = __half2float(reinterpret_cast<const __half*>(p.bias)[ng + j]);
          bu = __half2float(reinterpret_cast<const __half*>(p.bias)[ng + 8 + j]);
        } else {
          bg = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[ng + j]);
          bu = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[ng + 8 + j]);
        }
      }
      store_swiglu(p.out.ptr[0], o + j, swiglu_operand(g[j], p.bias != nullptr, bg, p.out_dtype),
                   swiglu_operand(u[j], p.bias != nullptr, bu, p.out_dtype), p.out_dtype);
    }
  }
}

// splitk_reduce_kernel of the Scaled int8 instances: the exact int32 sum of the partials through store_out_scaled, so split and
// unsplit calls store the same bits
__device__ __forceinline__ void splitk_reduce_scaled(const TsParams& p, const ScaledArgs& sc) {
  const unsigned n4 = unsigned(p.N) >> 2;
  const unsigned total4 = unsigned(p.M) * n4;
  const size_t split_stride4 = size_t(p.M) * n4;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const unsigned m = i / n4, n = (i - m * n4) * 4u;
    int acc[4] = {0, 0, 0, 0};
    for (int sp = 0; sp < p.splits; ++sp) {
      const int4 v = __ldcs(reinterpret_cast<const int4*>(p.ws) + size_t(sp) * split_stride4 + i);
      acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
    }
    const float sa = sc.a_scale[m];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      store_out_scaled(p.out.ptr[0], size_t(m) * p.N + n + j, acc[j], sa, sc.w_scale[n + j], p.bias, n + j, p.out_dtype);
  }
}

// splitk_reduce_kernel of the W4A8 instances: S = the fp32 partials summed in split order (from 0), then round_out(S / a_scale[m])
// with the bias in out_dtype
__device__ __forceinline__ void splitk_reduce_w4a8(const TsParams& p, const ScaledArgs& sc) {
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
    const float sa = sc.a_scale[m];
#pragma unroll
    for (int j = 0; j < 4; ++j) store_out_dequant(p.out.ptr[0], size_t(m) * p.N + n + j, __fdiv_rn(S[j], sa), p.bias, n + j, p.out_dtype);
  }
}

// out[m, n] = cast(sum_s ws[s][m][n]) (+ bias), stored to every destination of the OutSpec.  One thread = 4 consecutive n
// (N is a multiple of 128 here): 128-bit loads of the partials, 32-bit index arithmetic, one vector store per destination.
// F = SwiGLU: splitk_reduce_swiglu; Scaled: splitk_reduce_scaled; W4A8: splitk_reduce_w4a8.
template <bool INT8, MatmulForm F>
__global__ void splitk_reduce_kernel(const TsParams p, const ScaledArgs sc) {
  if constexpr (F == MatmulForm::W4A8) {
    splitk_reduce_w4a8(p, sc);
    return;
  }
  if constexpr (F == MatmulForm::SwiGLU) {
    splitk_reduce_swiglu(p);
    return;
  }
  if constexpr (F == MatmulForm::Scaled) {
    splitk_reduce_scaled(p, sc);
    return;
  }
  const unsigned n4 = unsigned(p.N) >> 2;                 // quads per row
  const unsigned total4 = unsigned(p.M) * n4;             // m * N / 4 < 2^31 (m <= 128 on this path)
  const size_t split_stride4 = size_t(p.M) * n4;          // quads per split
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const unsigned m = i / n4, n = (i - m * n4) * 4u;
    float bias_f[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (p.a_dtype == BB_F16) bias_f[j] = __half2float(reinterpret_cast<const __half*>(p.bias)[n + j]);
        else if (p.a_dtype == BB_BF16) bias_f[j] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[n + j]);
        else bias_f[j] = float(reinterpret_cast<const int8_t*>(p.bias)[n + j]);
      }
    }
    const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
    if constexpr (INT8) {
      int acc[4] = {0, 0, 0, 0};
      for (int sp = 0; sp < p.splits; ++sp) {
        const int4 v = __ldcs(reinterpret_cast<const int4*>(p.ws) + size_t(sp) * split_stride4 + i);
        acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      }
      for (int d = 0; d < p.out.n; ++d) {
        void* Cd = p.out.ptr[d];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int b = int(bias_f[j]);
          switch (p.out_dtype) {
            case BB_I32: reinterpret_cast<int*>(Cd)[o + j] = acc[j] + b; break;
            case BB_I8: reinterpret_cast<int8_t*>(Cd)[o + j] = int8_t(int8_t(acc[j]) + b); break;
            case BB_F32: reinterpret_cast<float*>(Cd)[o + j] = float(acc[j]) + float(b); break;
            case BB_F16: reinterpret_cast<__half*>(Cd)[o + j] = __hadd(__int2half_rn(acc[j]), __int2half_rn(b)); break;
            default: reinterpret_cast<__nv_bfloat16*>(Cd)[o + j] = __hadd(__int2bfloat16_rn(acc[j]), __int2bfloat16_rn(b));
          }
        }
      }
    } else {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int sp = 0; sp < p.splits; ++sp) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(p.ws) + size_t(sp) * split_stride4 + i);
        acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      }
      if (p.out_dtype == BB_F16) {
        __half h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          h[j] = __float2half_rn(acc[j]);
          if (p.bias) h[j] = __hadd(h[j], __float2half_rn(bias_f[j]));
        }
        for (int d = 0; d < p.out.n; ++d) {
          __half* dst = reinterpret_cast<__half*>(p.out.ptr[d]) + o;
#pragma unroll
          for (int j = 0; j < 4; ++j) dst[j] = h[j];
        }
      } else if (p.out_dtype == BB_BF16) {
        __nv_bfloat16 h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          h[j] = __float2bfloat16_rn(acc[j]);
          if (p.bias) h[j] = __hadd(h[j], __float2bfloat16_rn(bias_f[j]));
        }
        for (int d = 0; d < p.out.n; ++d) {
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out.ptr[d]) + o;
#pragma unroll
          for (int j = 0; j < 4; ++j) dst[j] = h[j];
        }
      } else {
        for (int d = 0; d < p.out.n; ++d) {
          float* dst = reinterpret_cast<float*>(p.out.ptr[d]) + o;
#pragma unroll
          for (int j = 0; j < 4; ++j) dst[j] = acc[j] + (p.bias ? bias_f[j] : 0.f);
        }
      }
    }
  }
}

// split-K factor: only when the tile grid leaves most SMs idle; the k-range must split on k-block boundaries
int choose_splits(int tiles, int num_kb, int sms) {
  if (tiles >= sms) return 1;
  int best = 1;
  for (int sp = 2; sp <= 8; ++sp) {
    if (num_kb % sp || num_kb / sp < 8) continue;
    if (tiles * sp <= sms) best = sp;  // one CTA per SM
  }
  return best;
}

// Byte offset of the split-K partials in the workspace: past the m = 1 slab kernel's slot region, sized at the device's full SM
// count whatever bb_set_sm_count_cap says.  An operator hands one buffer to every m, and the slab requires its slots zero on entry.
size_t splitk_partials_offset() { return gemv_slab_slot_bytes(device_sm_count_uncapped()); }

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// BB_TILE_SLAB storage [N/32][row_bytes/512][32][512 B] as a 4-D tensor; box = {PRB bytes, 32 rows, 1 segment, 4 row blocks}
// lands in shared memory as the same dense [128 rows][PRB] tile the row-major 2-D box produces
int make_map_w_tiled(CUtensorMap* map, const void* base, uint64_t row_bytes, uint64_t rows, uint32_t prb) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 4; }
  const uint64_t upr = row_bytes / BB_TILE_ROW_BYTES;
  cuuint64_t dims[4] = {BB_TILE_ROW_BYTES, BB_TILE_ROWS, upr, rows / BB_TILE_ROWS};
  cuuint64_t strides[3] = {BB_TILE_ROW_BYTES, uint64_t(BB_TILE_ROW_BYTES) * BB_TILE_ROWS, uint64_t(BB_TILE_ROW_BYTES) * BB_TILE_ROWS * upr};
  cuuint32_t box[4] = {prb, BB_TILE_ROWS, 1, TS_ROWS / BB_TILE_ROWS};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (4-D, slab-tiled W) failed with CUresult %d", int(r)); return 4; }
  return 0;
}

// W4A8: the largest split factor up to the plain instance's that divides the group count, so every split starts on a group
// boundary (and needs no more workspace than the plain instance)
int choose_splits_w4a8(int tiles, int num_kb, int groups, int sms) {
  int sp = choose_splits(tiles, num_kb, sms);
  while (groups % sp) --sp;
  return sp;
}

template <typename T, int BITS, int BM, bool IL, int FMT, MatmulForm F>
int launch_ts_inst(const MatmulArgs& a, const TsParams& p0) {
  using SM = TsSmem<T, BITS, BM>;
  using EI = ElemInfo<T>;
  auto kernel = gemm_ts_kernel<T, BITS, BM, IL, FMT, F>;
  static KernelCache<> cache;
  if (!kernel_setup(cache, kernel, SM::kTotal)) {
    set_error("gemm_ts: cannot raise the kernel's dynamic shared memory to %d bytes on this device", SM::kTotal);
    return 2;
  }
  TsParams p = p0;
  p.m_tiles = (a.m + BM - 1) / BM;
  const int num_kb_total = a.d.K / EI::kKB;
  const int tiles = p.m_tiles * (a.d.N / TS_ROWS);
  if constexpr (F == MatmulForm::W4A8) p.splits = a.m <= 128 ? choose_splits_w4a8(tiles, num_kb_total, p.G, device_sm_count()) : 1;
  else p.splits = a.m <= 128 ? choose_splits(tiles, num_kb_total, device_sm_count()) : 1;
  const size_t ws_off = splitk_partials_offset();
  if (p.splits > 1 && a.workspace_bytes < ws_off + size_t(p.splits) * a.m * a.d.N * 4) p.splits = 1;  // no scratch given
  p.kb_per_split = num_kb_total / p.splits;
  p.ws = p.splits > 1 ? static_cast<char*>(a.workspace) + ws_off : a.workspace;
  const size_t smem_bytes = SM::kTotal;
  CUtensorMap tmA, tmW;
  const CUtensorMapDataType adt = EI::kInt8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                            : (std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                                                               : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  int rc = make_map_2d(&tmA, adt, a.A, uint64_t(a.d.K), uint64_t(a.m), uint64_t(a.d.K) * sizeof(T), EI::kKB, BM,
                       CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  const uint64_t wrow = uint64_t(a.d.K) * BITS / 8;
  p.w_tiled = a.d.w_tile == BB_TILE_SLAB ? 1 : 0;
  if (p.w_tiled) rc = make_map_w_tiled(&tmW, a.W, wrow, uint64_t(a.d.N), SM::kPRB);
  else rc = make_map_2d(&tmW, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.W, wrow, uint64_t(a.d.N), wrow, SM::kPRB, TS_ROWS,
                        CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  const int grid = tiles * p.splits;
  kernel<<<grid, TS_THREADS, smem_bytes, a.stream>>>(tmA, tmW, p, a.scaled);
  BB_LAUNCH_CHECK();
  if (p.splits > 1) {
    const size_t total = size_t(a.m) * a.d.N / (F == MatmulForm::SwiGLU ? 8 : 4);   // one thread per 4 consecutive output columns
    const int rthreads = 256;
    const int rblocks = int(std::min<size_t>((total + rthreads - 1) / rthreads, size_t(device_sm_count()) * 8));
    splitk_reduce_kernel<EI::kInt8, F><<<rblocks, rthreads, 0, a.stream>>>(p, a.scaled);
    BB_LAUNCH_CHECK();
  }
  return 0;
}

// activation rows per CTA: the wgmma N extent (m > 128 runs several 128-row tiles).  W4A8 stops at 64: at 128 its fp32 group sums
// do not fit beside the int32 accumulators (ptxas spills)
template <typename T, int BITS, bool IL, int FMT, MatmulForm F>
int launch_ts_bm(const MatmulArgs& a, const TsParams& p) {
  if (a.m <= 32) return launch_ts_inst<T, BITS, 32, IL, FMT, F>(a, p);
  if constexpr (F != MatmulForm::W4A8) {
    if (a.m > 64) return launch_ts_inst<T, BITS, 128, IL, FMT, F>(a, p);
  }
  return launch_ts_inst<T, BITS, 64, IL, FMT, F>(a, p);
}
// the forms built for each activation type: 16-bit ones run Plain and SwiGLU (bb_matmul_swiglu rejects int8 activations), int8
// ones Plain, Scaled and W4A8 (bb_matmul_scaled and bb_matmul_w4a8 reject 16-bit ones; bb_matmul_w4a8 takes 4-bit weights only)
template <typename T, int BITS, bool IL, int FMT>
int launch_ts_form(const MatmulArgs& a, const TsParams& p) {
  if constexpr (!std::is_same<T, int8_t>::value) {
    if (a.form == MatmulForm::SwiGLU) return launch_ts_bm<T, BITS, IL, FMT, MatmulForm::SwiGLU>(a, p);
  } else {
    if (a.form == MatmulForm::Scaled) return launch_ts_bm<T, BITS, IL, FMT, MatmulForm::Scaled>(a, p);
    if (a.form == MatmulForm::W4A8) return launch_ts_bm<T, 4, IL, FMT, MatmulForm::W4A8>(a, p);
  }
  return launch_ts_bm<T, BITS, IL, FMT, MatmulForm::Plain>(a, p);
}
template <typename T, int BITS>
int launch_ts_layout(const MatmulArgs& a, const TsParams& p) {
  return a.d.w_layout == BB_LAYOUT_COMPRESSED ? launch_ts_form<T, BITS, false, 0>(a, p) : launch_ts_form<T, BITS, true, 0>(a, p);
}

}  // namespace

bool gemm_ts_supported(const bb_matmul_desc& d, int m) {
  if (m < 1) return false;
  const bool table_fmt = d.w_fmt == BB_W_NF || d.w_fmt == BB_W_FP4;
  if (table_fmt) {   // 16-entry table formats: 4-bit compressed storage, scale only (a zero point has no fast path)
    if (d.w_bits != 4 || d.w_layout != BB_LAYOUT_COMPRESSED || d.with_zeros || d.a_dtype == BB_I8) return false;
  } else if (d.w_fmt == BB_W_FP8_E4M3 || d.w_fmt == BB_W_FP8_E5M2) {   // 8-bit float weights x 16-bit activations, scale only
    if (d.w_bits != 8 || d.w_layout != BB_LAYOUT_COMPRESSED || d.with_zeros || d.a_dtype == BB_I8) return false;
  } else if (d.w_fmt != BB_W_UINT && d.w_fmt != BB_W_INT) {
    return false;
  }
  if (d.w_bits != 4 && d.w_bits != 2 && !(d.w_bits == 8 && (d.w_fmt == BB_W_FP8_E4M3 || d.w_fmt == BB_W_FP8_E5M2))) return false;
  if (d.N % TS_ROWS) return false;
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if (d.a_dtype == BB_I8) {
    if (d.accum_dtype != BB_I32 || d.w_layout == BB_LAYOUT_INTERLEAVED_16) return false;
    if (d.with_scaling || d.with_zeros) return false;
    if (d.K % 128) return false;
    return true;
  }
  if (d.a_dtype != BB_F16 && d.a_dtype != BB_BF16) return false;
  if (d.w_layout == BB_LAYOUT_INTERLEAVED_8) return false;
  if (d.K % 64 || g % 64 || d.K % g) return false;
  if (d.with_zeros && !d.with_scaling) return false;
  if (d.w_fmt == BB_W_INT && d.with_zeros) return false;
  if (d.out_dtype != BB_F16 && d.out_dtype != BB_BF16 && d.out_dtype != BB_F32) return false;
  if (d.with_zeros && d.zeros_mode == BB_ZEROS_QUANTIZED && (d.N * d.w_bits) % 8) return false;
  return true;
}

int gemm_ts_splits(int tiles, int num_kb, int sms) { return choose_splits(tiles, num_kb, sms); }

size_t gemm_ts_workspace_bytes(const bb_matmul_desc& d, int m) {
  if (m > 128) return 0;
  const int kb = d.a_dtype == BB_I8 ? 128 : 64;
  const int bm = m <= 32 ? 32 : (m <= 64 ? 64 : 128);
  const int tiles = ((m + bm - 1) / bm) * (d.N / TS_ROWS);
  const int sp = choose_splits(tiles, d.K / kb, device_sm_count());
  return sp > 1 ? splitk_partials_offset() + size_t(sp) * m * d.N * 4 : 0;
}

int launch_gemm_ts(const MatmulArgs& a) {
  const bb_matmul_desc& d = a.d;
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15)) {
    set_error("gemm_ts: A and W must be 16-byte aligned");
    return 5;
  }
  const TsParams p = make_ts_params(d, a.scale, a.zeros, a.bias, a.lut, make_outspec(a), a.m);
  if (d.w_fmt == BB_W_NF || d.w_fmt == BB_W_FP4)
    return d.a_dtype == BB_F16 ? launch_ts_form<__half, 4, false, 1>(a, p) : launch_ts_form<__nv_bfloat16, 4, false, 1>(a, p);
  if (d.w_fmt == BB_W_FP8_E4M3 || d.w_fmt == BB_W_FP8_E5M2)
    return d.a_dtype == BB_F16 ? launch_ts_form<__half, 8, false, 2>(a, p) : launch_ts_form<__nv_bfloat16, 8, false, 2>(a, p);
  if (d.a_dtype == BB_I8) return d.w_bits == 4 ? launch_ts_layout<int8_t, 4>(a, p) : launch_ts_layout<int8_t, 2>(a, p);
  if (d.a_dtype == BB_F16) return d.w_bits == 4 ? launch_ts_layout<__half, 4>(a, p) : launch_ts_layout<__half, 2>(a, p);
  return d.w_bits == 4 ? launch_ts_layout<__nv_bfloat16, 4>(a, p) : launch_ts_layout<__nv_bfloat16, 2>(a, p);
}

}  // namespace bb
