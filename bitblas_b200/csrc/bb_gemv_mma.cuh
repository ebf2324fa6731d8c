// bb_gemv_mma.cuh -- the fp16 / bf16 streaming GEMV of bb_gemv.cu as a device function over one 16-row block of W.
// gemv_mma_kernel (bb_gemv.cu) runs it once per CTA; gemv_grouped_kernel (bb_grouped.cu) runs it for every (expert, row block,
// row chunk) work item a persistent CTA takes.  The design notes are at the top of bb_gemv.cu.
#pragma once
#include <algorithm>
#include <type_traits>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int MAX_KS = 8;  // warps per CTA = K splits per 16-row block
constexpr int PF = 4;      // weight steps in flight per warp (register queue of plain 128-bit ld.global.nc loads).
                           // tools/membench.cu compares this pattern (16 rows x 64 B per warp load, depth 4, 3 K-splits)
                           // with the linear-read rate, the same addresses through cp.async (LDGSTS) and deeper queues.

struct GemvParams {
  const void* A;
  const uint8_t* W;
  const void* scale;
  const void* zeros;
  const void* bias;
  OutSpec out;
  int M, N, K;
  int g;          // group size in elements (multiple of 128, or K)
  int G;          // groups per row
  int with_scaling;
  int zmode;      // 0 none, 1 original, 2 rescale, 3 quantized
  int zp_const;   // constant zero point of the "int" formats (2^(bits-1)), 0 for uint
  int out_dtype;
  int ks;         // warps per CTA
};

// the parameters of M rows of A against W (the launcher sets ks)
inline GemvParams make_params(const bb_matmul_desc& d, const void* A, const void* W, const void* scale, const void* zeros,
                              const void* bias, const OutSpec& out, int M) {
  GemvParams p;
  p.A = A; p.W = reinterpret_cast<const uint8_t*>(W); p.scale = d.with_scaling ? scale : nullptr;
  p.zeros = d.with_zeros ? zeros : nullptr; p.bias = d.with_bias ? bias : nullptr; p.out = out;
  p.M = M; p.N = d.N; p.K = d.K;
  p.g = d.group_size <= 0 ? d.K : d.group_size; p.G = d.K / p.g;
  p.with_scaling = d.with_scaling;
  p.zmode = d.with_zeros ? (d.zeros_mode + 1) : 0;
  p.zp_const = (d.w_fmt == BB_W_INT) ? (1 << (d.w_bits - 1)) : 0;
  p.out_dtype = d.out_dtype;
  p.ks = 1;
  return p;
}

// K splits per CTA (= warps per CTA) for a grid of `ctas` CTAs over rows of `steps` 128-k steps: the largest count up to max_ks
// for which EVERY CTA is resident at once (occupancy of this kernel instance, cached in `cache` per device and split).  When not
// even two warps per CTA fit in one wave (the decode GEMV at N >= ~24k rows), the full split is used and the grid runs in several
// waves rather than with one resident warp per CTA.
template <typename Kernel>
int pick_ks(KernelCache<MAX_KS + 1>& cache, Kernel kernel, int max_ks, int ctas, int steps) {
  const int full = std::max(1, std::min(max_ks, steps));
  const int dev = current_device(), sms = device_sm_count();
  for (int ks = full; ks >= 2; --ks)
    if (ctas <= sms * kernel_setup(cache, kernel, 0, ks * 32, 0, ks, dev)) return ks;
  return full;
}

// Programmatic dependent launch (PDL).  A decode step is a chain of dependent GEMVs (qkv -> o -> gate_up -> down); the
// weights, scales and zeros of the next one do not depend on the previous result, only its activations do.  Each streaming
// kernel therefore (1) lets the next kernel in the stream start once every CTA of its own has finished its weight stream
// (pdl_launch_dependents before the epilogue; triggered at kernel entry, the early CTAs of kernel i+1
// would compete with kernel i for the weight stream) and (2) starts its own weight prefetch immediately but
// executes pdl_wait -- which
// returns once the preceding kernel has completed and flushed -- before the first activation load.  Launch latency and the
// first DRAM round trip of kernel i+1 then overlap the tail of kernel i.  Both instructions are no-ops when the launch
// carries no programmatic-serialization attribute or the predecessor never triggers.  (pdl_launch_dependents / pdl_wait:
// bb_common.cuh.)

template <int BITS>
__device__ __forceinline__ void load_w(const uint8_t* p, uint32_t (&w)[BITS]) {
  if constexpr (BITS == 4) {
    uint4 v = ldg_nc_v4(p);
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
  } else {
    uint2 v = ldg_nc_v2(p);
    w[0] = v.x; w[1] = v.y;
  }
}

// split [0, total) into `parts` nearly equal contiguous ranges
__device__ __forceinline__ void split_range(int total, int parts, int idx, int& begin, int& end) {
  const int base = total / parts, rem = total % parts;
  begin = idx * base + min(idx, rem);
  end = begin + base + (idx < rem ? 1 : 0);
}

// register budget of one gemv_mma instance (NT batch tiles of 8 rows; "original" / "rescale" zeros carry more per-group state)
constexpr int gemv_mma_maxnreg(int nt, int zk) {
  return nt == 1 ? ((zk == 1 || zk == 2) ? 112 : 96) : (nt == 2 ? ((zk == 1 || zk == 2) ? 168 : 128) : ((zk == 1 || zk == 2) ? 232 : 192));
}
// most warps per CTA (K splits) of an instance with NT batch tiles: one batch tile splits K over at most 4 warps
constexpr int gemv_max_ks(int nt) { return nt == 1 ? 4 : MAX_KS; }

// The instance ladder of the streaming GEMV kernels.  gemv_nt: f(NT) with NT = 1, 2 or 4 batch tiles of 8 rows for `rows` rows of
// A.  gemv_mma_instance: f(NT, ZK, SC) with (ZK, SC) from p's scale / zero-point mode.  All as std::integral_constant tags.
template <typename F>
int gemv_nt(int rows, F&& f) {
  if (rows <= 8) return f(std::integral_constant<int, 1>{});
  if (rows <= 16) return f(std::integral_constant<int, 2>{});
  return f(std::integral_constant<int, 4>{});
}
template <typename F>
int gemv_mma_instance(const GemvParams& p, int rows, F&& f) {
  return gemv_nt(rows, [&](auto nt) {
    using std::integral_constant;
    if (!p.with_scaling) return f(nt, integral_constant<int, 0>{}, std::false_type{});
    if (p.zmode == 0) return f(nt, integral_constant<int, 0>{}, std::true_type{});
    if (p.zmode == 1) return f(nt, integral_constant<int, 1>{}, std::true_type{});
    if (p.zmode == 2) return f(nt, integral_constant<int, 2>{}, std::true_type{});
    return f(nt, integral_constant<int, 3>{}, std::true_type{});
  });
}

// ---------------------------------------------------------------------------------------------
// fp16 / bf16 activations
//   ZK: 0 no zeros (constant zero point of the "int" formats only), 1 "original", 2 "rescale", 3 "quantized"
//   SC: with_scaling
// ---------------------------------------------------------------------------------------------
// (Activations and group parameters are not staged in shared memory before the weight stream: the staging prologue of a
// short-lived CTA costs more than the in-order load stalls it removes.)
// One 16-row block `rb` of W against rows [0, p.M) of p.A (p.M <= 8 * NT), K split over the p.ks warps of the CTA and reduced
// through `red`.  PDL: the tile issues griddepcontrol.wait after its weight prologue and launch_dependents after its weight
// stream (gemv_mma_kernel); with PDL = false the caller owns both instructions.  SWIGLU: W holds gate/up interleaved (bb_common.cuh),
// and rows r and r + 8 of the block become column rb * 8 + r of p.out (row stride p.out.ld = N / 2), one destination only.
template <typename T, int BITS, bool IL, int NT, int ZK, bool SC, bool PDL, bool SWIGLU = false>
__device__ __forceinline__ void gemv_mma_tile(const GemvParams& p, const int rb, float (&red)[MAX_KS][16][8 * NT]) {
  constexpr bool RS = ZK == 2;
  constexpr int NP = 32 / BITS / 2;     // pairs per 32-bit word: 4 (4-bit) or 8 (2-bit)
  constexpr int WPS = BITS;             // 32-bit words per thread per row per step (32 k per thread)
  constexpr bool HI = std::is_same<T, __half>::value && BITS == 4;  // in-place odd-nibble extraction
  constexpr uint32_t MAGIC = TypeTraits<T>::kMagic;
  constexpr uint32_t NEGMAGIC = MAGIC | 0x80008000u;
  // odd nibbles sit at mantissa bits 4..7: with exponent 2^6 (0x5400) the fp16 value is exactly 64 + u
  constexpr uint32_t MAGIC_HI = 0x54005400u;
  constexpr uint32_t NEGMAGIC_HI = HI ? 0xd400d400u : NEGMAGIC;
  constexpr uint32_t ZMUL_HI = HI ? 0x00100010u : 0x00010001u;  // zero point scaled into the odd-nibble position
  constexpr int MAXZ = HI ? 47 : TypeTraits<T>::kMagicVal - (1 << BITS);  // largest zero point that folds exactly
  constexpr uint32_t ONE2 = std::is_same<T, __half>::value ? 0x3c003c00u : 0x3f803f80u;
  constexpr int EPB = 8 / BITS;
  constexpr int STEP_BYTES = 16 * BITS;  // packed bytes per row per step

  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // warp-uniform: keeps the loops below convergent
  const int r = lane >> 2, q = lane & 3;
  const int n_a = rb * 16 + r, n_b = n_a + 8;
  int step_begin, step_end;
  split_range(p.K / 128, p.ks, warp, step_begin, step_end);
  const int ns = step_end - step_begin;
  const int spg = p.g / 128;  // steps per group
  const size_t row_bytes = size_t(p.K) * BITS / 8;

  const uint8_t* wpa = p.W + size_t(n_a) * row_bytes + q * (4 * WPS) + size_t(step_begin) * STEP_BYTES;
  const uint8_t* wpb = wpa + 8 * row_bytes;
  // activations: this thread's 32-element slice of each step, as uint4 (8 elements each)
  const uint4* ap[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int m = min(8 * t + r, p.M - 1);
    ap[t] = reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.A) + size_t(m) * p.K) + step_begin * 16 + q * 4;
  }
  // running pointers to the NEXT group's parameters (scale / zeros rows are [N, G]; quantized zeros [G, N*bits/8])
  int gi = step_begin / spg;
  int grp_left = spg - (step_begin % spg);
  const uint16_t* sp_a = reinterpret_cast<const uint16_t*>(p.scale) + size_t(n_a) * p.G + gi;
  const uint16_t* zp_a = reinterpret_cast<const uint16_t*>(p.zeros) + size_t(n_a) * p.G + gi;
  const int row8 = 8 * p.G;
  const int qz_stride = p.N * BITS / 8;
  const uint8_t* qzp = reinterpret_cast<const uint8_t*>(p.zeros) + n_a / EPB + size_t(gi) * qz_stride;
  const uint32_t qsh_a = BITS * (n_a % EPB), qsh_b = BITS * (n_b % EPB);
  int groups_to_fetch = p.G - gi;

  // the 16 MMAs of a step are spread over NCH independent accumulator chains (weights / fold x j parity) so that the
  // per-warp step latency is 4 dependent HMMAs instead of 16
  constexpr int NCH = 2;
  float acc_t[NT][4], acc_c[NT][NCH][4], asum_g[RS ? NT : 1][4];
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc_t[t][j] = 0.f;
#pragma unroll
      for (int c = 0; c < NCH; ++c) acc_c[t][c][j] = 0.f;
    }
#pragma unroll
  for (int t = 0; t < (RS ? NT : 1); ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) asum_g[t][j] = 0.f;

  // per-group state
  float s_a = 1.f, s_b = 1.f, zc_a = 0.f, zc_b = 0.f;
  uint32_t dzf[4] = {0u, 0u, 0u, 0u};  // -(z - rint(z)) fragment for non-integer "original" zero points
  bool need_dz = false;
  uint32_t fold[4];  // -(magic + z) fragment: {row a even, row b even, row a odd, row b odd nibble positions}
  auto set_fold = [&](uint32_t za, uint32_t zb) {
    fold[0] = NEGMAGIC + za * 0x00010001u;
    fold[1] = NEGMAGIC + zb * 0x00010001u;
    fold[2] = NEGMAGIC_HI + za * ZMUL_HI;
    fold[3] = NEGMAGIC_HI + zb * ZMUL_HI;
  };
  set_fold(uint32_t(p.zp_const), uint32_t(p.zp_const));
  const uint32_t asum_frag[4] = {ONE2, ONE2, ONE2, ONE2};

  // group parameters are fetched one group ahead (raw bits) so their L2 latency overlaps a whole step
  uint16_t sr_a = 0, sr_b = 0, zr_a = 0, zr_b = 0;
  auto fetch_group = [&]() {
    if (groups_to_fetch > 0) {
      if constexpr (SC) {
        sr_a = __ldg(sp_a);
        sr_b = __ldg(sp_a + row8);
        ++sp_a;
      }
      if constexpr (ZK == 1 || ZK == 2) {
        zr_a = __ldg(zp_a);
        zr_b = __ldg(zp_a + row8);
        ++zp_a;
      }
      if constexpr (ZK == 3) {
        zr_a = __ldg(qzp);
        zr_b = __ldg(qzp + 8 / EPB);
        qzp += qz_stride;
      }
      --groups_to_fetch;
    }
  };
  auto begin_group = [&]() {
    if constexpr (SC) {
      s_a = raw_to_float<T>(sr_a);
      s_b = raw_to_float<T>(sr_b);
    }
    if constexpr (ZK == 2) {         // "rescale": w * s - z  ->  s * sum(w a) - z * sum(a)
      zc_a = raw_to_float<T>(zr_a);
      zc_b = raw_to_float<T>(zr_b);
    } else if constexpr (ZK == 1) {  // "original": (w - z) * s ; integer part folded, fraction via a third MMA
      const float za = raw_to_float<T>(zr_a), zb = raw_to_float<T>(zr_b);
      const float ia = rintf(za), ib = rintf(zb);
      const bool oka = ia >= 0.f && ia <= float(MAXZ), okb = ib >= 0.f && ib <= float(MAXZ);
      set_fold(oka ? uint32_t(int(ia)) : 0u, okb ? uint32_t(int(ib)) : 0u);
      const float da = oka ? za - ia : za, db = okb ? zb - ib : zb;
      need_dz = __any_sync(0xffffffffu, da != 0.f || db != 0.f);
      if (need_dz) {
        dzf[0] = dup2<T>(TypeTraits<T>::from_float(-da));
        dzf[1] = dup2<T>(TypeTraits<T>::from_float(-db));
        dzf[2] = dzf[0];
        dzf[3] = dzf[1];
      }
    } else if constexpr (ZK == 3) {
      set_fold((uint32_t(zr_a) >> qsh_a) & ((1u << BITS) - 1u), (uint32_t(zr_b) >> qsh_b) & ((1u << BITS) - 1u));
    }
    fetch_group();
  };
  auto end_group = [&]() {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float sj = (j < 2) ? s_a : s_b;
        if constexpr (RS) acc_t[t][j] = fmaf(-((j < 2) ? zc_a : zc_b), asum_g[t][j & 1], acc_t[t][j]);
        float g = acc_c[t][0][j];
#pragma unroll
        for (int c = 1; c < NCH; ++c) g += acc_c[t][c][j];
        acc_t[t][j] = SC ? fmaf(sj, g, acc_t[t][j]) : acc_t[t][j] + g;
#pragma unroll
        for (int c = 0; c < NCH; ++c) acc_c[t][c][j] = 0.f;
      }
      if constexpr (RS) {
#pragma unroll
        for (int j = 0; j < 4; ++j) asum_g[t][j] = 0.f;
      }
    }
  };

  constexpr int RPS = WPS * NP;  // activation registers per step per batch tile (32 k = 16 half2)
  constexpr int NBUF = 1;
  uint32_t Rbuf[NBUF][NT][RPS];
  // batch rows >= M read a clamped row: MMA output columns are independent and those are never stored
  auto load_acts = [&](uint32_t (&dst)[NT][RPS]) {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
#pragma unroll
      for (int x = 0; x < RPS / 4; ++x) {
        const uint4 v = __ldg(ap[t] + x);
        dst[t][4 * x] = v.x; dst[t][4 * x + 1] = v.y; dst[t][4 * x + 2] = v.z; dst[t][4 * x + 3] = v.w;
      }
      ap[t] += 16;
    }
  };
  auto process = [&](const uint32_t (&wa)[WPS], const uint32_t (&wb)[WPS], const uint32_t (&Rc)[NT][RPS]) {
    if (grp_left == 0) {
      end_group();
      grp_left = spg;
      begin_group();
    }
    --grp_left;
#pragma unroll
    for (int wi = 0; wi < WPS; ++wi) {
      uint32_t ha[NP], hb[NP];
      if constexpr (HI) {
        const uint32_t xa = wa[wi], ya = wa[wi] >> 8, xb = wb[wi], yb = wb[wi] >> 8;
        ha[0] = lop3_and_or(xa, 0x000f000fu, MAGIC); ha[1] = lop3_and_or(xa, 0x00f000f0u, MAGIC_HI);
        ha[2] = lop3_and_or(ya, 0x000f000fu, MAGIC); ha[3] = lop3_and_or(ya, 0x00f000f0u, MAGIC_HI);
        hb[0] = lop3_and_or(xb, 0x000f000fu, MAGIC); hb[1] = lop3_and_or(xb, 0x00f000f0u, MAGIC_HI);
        hb[2] = lop3_and_or(yb, 0x000f000fu, MAGIC); hb[3] = lop3_and_or(yb, 0x00f000f0u, MAGIC_HI);
      } else if constexpr (BITS == 4) {
        decode_u4x8_raw<T>(wa[wi], ha);
        decode_u4x8_raw<T>(wb[wi], hb);
      } else if constexpr (IL) {
        decode_u2x16_raw_interleaved<T>(wa[wi], ha);
        decode_u2x16_raw_interleaved<T>(wb[wi], hb);
      } else {
        decode_u2x16_raw_compressed<T>(wa[wi], ha);
        decode_u2x16_raw_compressed<T>(wb[wi], hb);
      }
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const uint32_t* R = &Rc[t][wi * NP];
#pragma unroll
        for (int j = 0; j < NP / 2; ++j) {
          const uint32_t af[4] = {ha[2 * j], hb[2 * j], ha[2 * j + 1], hb[2 * j + 1]};
          uint32_t b0, b1;
          if constexpr (IL) {
            b0 = R[2 * j]; b1 = R[2 * j + 1];
          } else {
            b0 = __byte_perm(R[j], R[j + NP / 2], 0x5410);
            b1 = __byte_perm(R[j], R[j + NP / 2], 0x7632);
          }
          constexpr int CW = 0, CF = NCH == 4 ? 2 : 1;   // chain bases: weights, fold
          const int par = NCH == 4 ? (j & 1) : 0;
          mma_16816<T>(acc_c[t][CW + par], af, b0, b1);
          mma_16816<T>(acc_c[t][CF + par], fold, b0, b1);
          if constexpr (ZK == 2) mma_16816<T>(asum_g[t], asum_frag, b0, b1);
          if constexpr (ZK == 1) {
            if (need_dz) mma_16816<T>(acc_c[t][CF + par], dzf, b0, b1);
          }
        }
      }
    }
  };

  if (ns > 0) {
    // register queue: wq[u] holds step (s + u); it is refilled with step (s + u + PF) right after being consumed
    uint32_t wq[PF][2][WPS];
    const uint8_t* wnext_a = wpa;
    const uint8_t* wnext_b = wpb;
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      if (u < ns) { load_w<BITS>(wnext_a, wq[u][0]); load_w<BITS>(wnext_b, wq[u][1]); }
      wnext_a += STEP_BYTES; wnext_b += STEP_BYTES;
    }
    fetch_group();   // first group's parameters: the only synchronous fetch, overlapped with the weight prologue
    if (PDL) pdl_wait();  // weights / scales / zeros above are not produced by the preceding kernel; the activations below may be
    begin_group();
    // GUARD = false: the chunk and all of its refills are inside the range (no per-step predicates)
    auto chunk = [&](auto guard_tag, int s, int buf) {
      constexpr bool GUARD = decltype(guard_tag)::value;
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        if (!GUARD || s + u < ns) {
          load_acts(Rbuf[0]);
          process(wq[u][0], wq[u][1], Rbuf[0]);
          if (!GUARD || s + u + PF < ns) { load_w<BITS>(wnext_a, wq[u][0]); load_w<BITS>(wnext_b, wq[u][1]); }
          wnext_a += STEP_BYTES; wnext_b += STEP_BYTES;
        }
      }
    };
    int s = 0, buf = 0;
#pragma unroll 1
    for (; s + 2 * PF <= ns; s += PF, buf ^= 1) chunk(std::false_type{}, s, buf);
#pragma unroll 1
    for (; s < ns; s += PF, buf ^= 1) chunk(std::true_type{}, s, buf);
    end_group();
  }

  // cross-warp reduction + epilogue
  if (PDL && ns <= 0) pdl_wait();   // (every path waits before it stores: the preceding kernel may still read what we overwrite)
  if (PDL) pdl_launch_dependents();   // the weight stream of this CTA is done: let the next kernel's CTAs take the freed slots
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    red[warp][r][8 * t + 2 * q] = acc_t[t][0];
    red[warp][r][8 * t + 2 * q + 1] = acc_t[t][1];
    red[warp][r + 8][8 * t + 2 * q] = acc_t[t][2];
    red[warp][r + 8][8 * t + 2 * q + 1] = acc_t[t][3];
  }
  __syncthreads();
  if constexpr (SWIGLU) {
    for (int idx = threadIdx.x; idx < 8 * 8 * NT; idx += blockDim.x) {
      const int row = idx & 7, m = idx >> 3;
      if (m >= p.M) continue;
      float vg = 0.f, vu = 0.f;
      for (int w = 0; w < p.ks; ++w) {
        vg += red[w][row][m];
        vu += red[w][row + 8][m];
      }
      const int n = rb * 16 + row;
      const T* bias = reinterpret_cast<const T*>(p.bias);
      const float g = swiglu_operand(vg, bias != nullptr, bias ? TypeTraits<T>::to_float(bias[n]) : 0.f, p.out_dtype);
      const float u = swiglu_operand(vu, bias != nullptr, bias ? TypeTraits<T>::to_float(bias[n + 8]) : 0.f, p.out_dtype);
      store_swiglu(p.out.ptr[0], size_t(m) * size_t(p.out.ld) + size_t(rb * 8 + row), g, u, p.out_dtype);
    }
  } else {
    for (int idx = threadIdx.x; idx < 16 * 8 * NT; idx += blockDim.x) {
      const int row = idx & 15, m = idx >> 4;
      if (m >= p.M) continue;
      float v = 0.f;
      for (int w = 0; w < p.ks; ++w) v += red[w][row][m];
      const int n = rb * 16 + row;
      const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
      const float bf = p.bias ? TypeTraits<T>::to_float(reinterpret_cast<const T*>(p.bias)[n]) : 0.f;
      if (p.out_dtype == BB_F16) {
        const __half h = round_out<__half>(v, p.bias, bf);
        for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__half*>(p.out.ptr[d])[o] = h;
      } else if (p.out_dtype == BB_BF16) {
        const __nv_bfloat16 h = round_out<__nv_bfloat16>(v, p.bias, bf);
        for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__nv_bfloat16*>(p.out.ptr[d])[o] = h;
      } else {
        for (int d = 0; d < p.out.n; ++d) reinterpret_cast<float*>(p.out.ptr[d])[o] = round_out<float>(v, p.bias, bf);
      }
    }
  }
}

}  // namespace

}  // namespace bb
