// bb_gemv.cu -- memory-bound streaming kernels for decode-sized M (1..32).
//
// Replaces the reference's generated SIMT GEMV (bitblas/ops/general_matmul/tilelang/dequantize/
// gemv_dequantize_simt.py:164-262: 128-bit A loads, 4-byte packed-B loads, LOP3 decode, fp16 FMA /
// __dp4a, shuffle all-reduce).  Design:
//   * the packed weights are the only HBM stream that matters (N*K*bits/8 bytes).  A warp owns 16 weight rows
//     and a contiguous K range; KS warps (one CTA) split K for a row block.  KS is chosen on the host so that
//     ~16 warps per SM are resident and EVERY CTA is resident at once: equal work per warp + a shared memory
//     system means all CTAs drain together and there is no tail wave.  Each warp keeps PF=4 steps (4 KB) of
//     128-bit ld.global.nc.L1::no_allocate loads in flight.
//   * LOP3 decode goes straight into mma.sync fragments (m16n8k16 f16/bf16, m16n8k32 u8.s8): 16 weight rows x
//     8 batch rows per instruction with fp32 / int32 accumulation, so the CUDA-core pipes only see the
//     decode.  The "+1024" decode magic and the zero point are NOT subtracted per element: a second MMA with
//     the constant fragment -(1024 + z[row]) against the same activations removes both inside the fp32
//     accumulator (1 HMMA instead of 4 HSUB2 per 16 weights x 2 rows).
//   * fp16 / 4-bit: odd nibbles are extracted in place (mask 0x00f000f0 -> 1024 + 16u) and paired with
//     activations pre-scaled by 1/16, which removes two of the three shifts per 32-bit word.
//   * k order inside a dot product is free, so the reference's interleaved storage layout AND the plain
//     compressed layout are both consumed with zero re-ordering cost (the B fragment is permuted instead).
//   * per-group scale is applied to the group's partial sum; non-integer zero points / "rescale" zeros use a
//     third MMA against a ones fragment to obtain sum(a) per group.
#include <cuda.h>

#include <atomic>
#include <algorithm>
#include <cstdlib>

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
__device__ __forceinline__ void mma_16832_u8s8(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <typename T>
__device__ __forceinline__ float raw_to_float(uint16_t b) {
  return TypeTraits<T>::to_float(*reinterpret_cast<const T*>(&b));
}

// Programmatic dependent launch (PDL).  A decode step is a chain of dependent GEMVs (qkv -> o -> gate_up -> down); the
// weights, scales and zeros of the next one do not depend on the previous result, only its activations do.  Each streaming
// kernel therefore (1) lets the next kernel in the stream start once every CTA of its own has finished its weight stream
// (pdl_launch_dependents before the epilogue; triggered at kernel entry, the early CTAs of kernel i+1
// would compete with kernel i for the weight stream) and (2) starts its own weight prefetch immediately but
// executes pdl_wait -- which
// returns once the preceding kernel has completed and flushed -- before the first activation load.  Launch latency and the
// first DRAM round trip of kernel i+1 then overlap the tail of kernel i.  Both instructions are no-ops when the launch
// carries no programmatic-serialization attribute or the predecessor never triggers.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

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

// ---------------------------------------------------------------------------------------------
// fp16 / bf16 activations
//   ZK: 0 no zeros (constant zero point of the "int" formats only), 1 "original", 2 "rescale", 3 "quantized"
//   SC: with_scaling
// ---------------------------------------------------------------------------------------------
// (Activations and group parameters are not staged in shared memory before the weight stream: the staging prologue of a
// short-lived CTA costs more than the in-order load stalls it removes.)
template <typename T, int BITS, bool IL, int NT, int ZK, bool SC>
__global__ void __launch_bounds__(NT == 1 ? 128 : MAX_KS * 32)
__maxnreg__(NT == 1 ? ((ZK == 1 || ZK == 2) ? 112 : 96) : (NT == 2 ? ((ZK == 1 || ZK == 2) ? 168 : 128) : ((ZK == 1 || ZK == 2) ? 232 : 192)))
gemv_mma_kernel(const GemvParams p) {
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
  __shared__ float red[MAX_KS][16][8 * NT];

  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // warp-uniform: keeps the loops below convergent
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
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
    pdl_wait();      // weights / scales / zeros above are not produced by the preceding kernel; the activations below may be
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
  if (ns <= 0) pdl_wait();   // (every path waits before it stores: the preceding kernel may still read what we overwrite)
  pdl_launch_dependents();   // the weight stream of this CTA is done: let the next kernel's CTAs take the freed slots
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    red[warp][r][8 * t + 2 * q] = acc_t[t][0];
    red[warp][r][8 * t + 2 * q + 1] = acc_t[t][1];
    red[warp][r + 8][8 * t + 2 * q] = acc_t[t][2];
    red[warp][r + 8][8 * t + 2 * q + 1] = acc_t[t][3];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 16 * 8 * NT; idx += blockDim.x) {
    const int row = idx & 15, m = idx >> 4;
    if (m >= p.M) continue;
    float v = 0.f;
    for (int w = 0; w < p.ks; ++w) v += red[w][row][m];
    const int n = rb * 16 + row;
    const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
    const float bf = p.bias ? TypeTraits<T>::to_float(reinterpret_cast<const T*>(p.bias)[n]) : 0.f;
    if (p.out_dtype == BB_F16) {
      __half h = __float2half_rn(v);
      if (p.bias) h = __hadd(h, __float2half_rn(bf));
      for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__half*>(p.out.ptr[d])[o] = h;
    } else if (p.out_dtype == BB_BF16) {
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      if (p.bias) h = __hadd(h, __float2bfloat16_rn(bf));
      for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__nv_bfloat16*>(p.out.ptr[d])[o] = h;
    } else {
      for (int d = 0; d < p.out.n; ++d) reinterpret_cast<float*>(p.out.ptr[d])[o] = v + bf;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Stream-K, TMA-fed streaming GEMV (m <= 2, fp16 / bf16 activations, 4-bit weights, group scales, no / quantized zeros).
//
// Same math as gemv_mma_kernel, different plumbing:
//  * work is cut into CHUNKS of [16 rows x 256 k] (2 KB of packed weights = two 128-k MMA steps).  The T = N/16 * K/256
//    chunks, ordered row block by row block, are split into equal contiguous ranges over ALL consumer warps of a persistent
//    grid (2 CTAs per SM): every SM streams the same number of bytes whatever N and K are -- no wave quantisation, no tail.
//  * every warp is its own TMA producer: per chunk, one elected lane requests one 128B-swizzled box of weights and the
//    matching 256 activations of each batch row into the warp's private 4-deep ring -- the request for chunk t + 4 is issued
//    as soon as chunk t sits in registers -- plus, whenever the stream enters a new window of 8 quantisation groups, the
//    scales [16 rows x 8 groups] and packed zeros [8 groups x 16 B] into a 2-deep window ring.  The warps therefore issue
//    NO global loads: nothing queues behind DRAM round trips (loads of a warp complete in order), all latency hiding is
//    the ring's, and there are no inter-warp barriers at all.  (A dedicated producer warp serving 8 consumers
//    would serialise the UTMALDG issue of the whole CTA.)
//  * a range whose FIRST segment starts inside a row block parks that segment's fp32 partial sums in its workspace slot and
//    raises a flag (a per-call 64-bit nonce, so undefined workspace contents cannot be mistaken for it).  The range that
//    holds the BEGINNING of a row block owns it: when it reaches the end of its share -- by then the other contributors,
//    who did theirs first, are long done, so nobody waits in steady state -- it adds their slots, the bias, and stores.
//    Ranges are handed out in REVERSE warp order, so an owner only ever waits for warps with lower ids (same or earlier
//    CTAs, dispatched no later than itself).  The summation order is fixed, so results are bit-reproducible; flags are reset
//    after use, so a replayed CUDA graph (same nonce) stays correct.
// ---------------------------------------------------------------------------------------------
constexpr int SK_CONSUMERS = 8;
constexpr int SK_DEPTH = 4;                 // weight / activation ring slots per consumer
constexpr int SK_THREADS = SK_CONSUMERS * 32;
constexpr int SK_WBYTES = 2048;             // weights per chunk
constexpr int SK_WIN_GROUPS = 8;
constexpr int SK_WIN_BYTES = 16 * SK_WIN_GROUPS * 2 + SK_WIN_GROUPS * 16;  // scales 256 B + zeros 128 B
constexpr int SK_WIN_SLOTS = 2;
constexpr int SK_MAX_M = 2;
constexpr int SK_SLOT_FLOATS = 128;         // per-warp partial slot: 32 lanes x 4 accumulators
constexpr int SK_NBARS = SK_CONSUMERS * (SK_DEPTH + SK_WIN_SLOTS);
constexpr int SK_MIN_CHUNKS = 4;            // do not spread a small problem thinner than this per warp

__host__ __device__ constexpr int sk_smem_bytes(int M, int depth) {
  return 1024 + SK_CONSUMERS * (depth * (SK_WBYTES + 512 * M) + SK_WIN_SLOTS * SK_WIN_BYTES) + SK_NBARS * 8;
}

struct SkParams {
  GemvParams g;
  int CPR;                       // chunks per row block = K / 256
  int WPR;                       // parameter windows per row = G / 8
  int lg_spg;                    // log2(steps per group); group sizes are 128 << lg_spg
  int depth;                     // ring slots in use per warp (1 .. SK_DEPTH)
  long long T;                   // chunks in total
  int Wtot;                      // consumer warps in the grid
  float* slots;                  // [Wtot][SK_SLOT_FLOATS]
  unsigned long long* flags;     // [Wtot]
  unsigned long long nonce;
};

__device__ __forceinline__ uint32_t sk_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sk_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void sk_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sk_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void sk_tma_2d(uint32_t dst, const void* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
__device__ __forceinline__ long long sk_range_begin(int ri, long long T, int Wtot) { return (long long)ri * T / Wtot; }

template <typename T>
__device__ __forceinline__ void sk_store(const GemvParams& p, int m, int n, float v) {
  const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
  const float bf = p.bias ? TypeTraits<T>::to_float(reinterpret_cast<const T*>(p.bias)[n]) : 0.f;
  if (p.out_dtype == BB_F16) {
    __half h = __float2half_rn(v);
    if (p.bias) h = __hadd(h, __float2half_rn(bf));
    for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__half*>(p.out.ptr[d])[o] = h;
  } else if (p.out_dtype == BB_BF16) {
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    if (p.bias) h = __hadd(h, __float2bfloat16_rn(bf));
    for (int d = 0; d < p.out.n; ++d) reinterpret_cast<__nv_bfloat16*>(p.out.ptr[d])[o] = h;
  } else {
    for (int d = 0; d < p.out.n; ++d) reinterpret_cast<float*>(p.out.ptr[d])[o] = v + bf;
  }
}

// c = a * b (+ 0): the first MMA of an accumulation chain, so accumulators never need zeroing
template <typename T>
__device__ __forceinline__ void mma_16816_z(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_16816_z<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=f"(c[0]), "=f"(c[1]), "=f"(c[2]), "=f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(0.f));
}
template <>
__device__ __forceinline__ void mma_16816_z<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=f"(c[0]), "=f"(c[1]), "=f"(c[2]), "=f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(0.f));
}

// GPC: quantisation groups per chunk -- 2 for group size 128 (one per MMA step), 1 for 256 << n
// MINB: CTAs per SM the kernel is compiled for.  2: both MMA steps of a chunk staged in registers, four interleaved HMMA chains
// (<= 128 registers); 3 / 4: one step at a time, two chains, <= 85 / 64 registers -- 24 / 32 warps per SM with a shallower ring.
template <typename T, bool IL, int ZK, int GPC, int MINB>
__global__ void __launch_bounds__(SK_THREADS, MINB)
gemv_sk_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA,
               const __grid_constant__ CUtensorMap tmS, const __grid_constant__ CUtensorMap tmZ, const SkParams sp) {
  constexpr int NP = 4, WPS = 4;
  constexpr bool HI = std::is_same<T, __half>::value;
  constexpr uint32_t MAGIC = TypeTraits<T>::kMagic;
  constexpr uint32_t NEGMAGIC = MAGIC | 0x80008000u;
  constexpr uint32_t MAGIC_HI = 0x54005400u;
  constexpr uint32_t NEGMAGIC_HI = HI ? 0xd400d400u : NEGMAGIC;
  constexpr uint32_t ZMUL_HI = HI ? 0x00100010u : 0x00010001u;
  constexpr uint32_t ZOFF = 16 * SK_WIN_GROUPS * 2;   // zeros follow the scales inside a window slot
  const GemvParams& p = sp.g;
  extern __shared__ uint8_t sk_raw[];
  const int lane = threadIdx.x & 31;
  const int c = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  // every warp is its own producer: barriers, ring and window slots are private to the warp
  const uint32_t abytes = 512u * uint32_t(p.M);
  const int DEPTH = sp.depth;   // ring slots per warp (1 .. SK_DEPTH); the shared-memory layout follows it
  const uint32_t smem0 = (sk_smem_u32(sk_raw) + 1023u) & ~1023u;
  const uint32_t wring_c = smem0 + uint32_t(c * DEPTH) * SK_WBYTES;
  const uint32_t aring_c = smem0 + uint32_t(SK_CONSUMERS * DEPTH) * SK_WBYTES + uint32_t(c * DEPTH) * abytes;
  const uint32_t wins_c = smem0 + uint32_t(SK_CONSUMERS * DEPTH) * (SK_WBYTES + abytes) + uint32_t(c * SK_WIN_SLOTS) * SK_WIN_BYTES;
  const uint32_t bars = smem0 + uint32_t(SK_CONSUMERS) * (uint32_t(DEPTH) * (SK_WBYTES + abytes) + SK_WIN_SLOTS * SK_WIN_BYTES);
  const uint32_t barF = bars + uint32_t(c * (SK_DEPTH + SK_WIN_SLOTS)) * 8u;   // full[DEPTH] then pfull[2]
  const uint32_t barP = barF + SK_DEPTH * 8u;
  const int lg_spg = sp.lg_spg;   // steps per group = 1 << lg_spg
  const int CPR = sp.CPR;
  const int cpw = 4 << lg_spg;    // chunks per parameter window (8 groups)
  const int Kb = p.K >> 1;        // packed bytes per weight row

  if (lane == 0) {
    for (int s = 0; s < SK_DEPTH + SK_WIN_SLOTS; ++s) sk_mbar_init(barF + s * 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();

  const int ri = sp.Wtot - 1 - (blockIdx.x * SK_CONSUMERS + c);   // ranges in reverse warp order
  const int r = lane >> 2, q = lane & 3;
  // MMA row r of the fragment is weight row rr of the 16-row block (and r + 8 -> rr + 8): with rr = (r >> 1) | ((r & 1) << 2)
  // the two rows met by one shared-memory phase (lanes 8i .. 8i+7: r = 2i, 2i+1) are rows i and i + 4, whose 128B-swizzle
  // masks differ in bit 2 -- the 8 lanes then cover all eight 16-byte columns and the tile reads are conflict-free.
  const int rr = (r >> 1) | ((r & 1) << 2);
  int t = int(sk_range_begin(ri, sp.T, sp.Wtot));
  const int t1 = int(sk_range_begin(ri + 1, sp.T, sp.Wtot));
  if (t >= t1) return;

  // ---- request side (lane 0 executes the TMA instructions; all lanes track the positions) ----
  int ti = t, islot = 0;
  int irb16 = (t / CPR) * 16, ic0 = (t - (t / CPR) * CPR) * 128;   // TMA coordinates of the next chunk to request
  auto issue_chunk = [&]() {
    if (lane == 0) {
      const uint32_t bar = barF + uint32_t(islot) * 8u;
      sk_mbar_expect_tx(bar, SK_WBYTES + abytes);
      sk_tma_2d(wring_c + uint32_t(islot) * SK_WBYTES, &tmW, ic0, irb16, bar);
      sk_tma_2d(aring_c + uint32_t(islot) * abytes, &tmA, 2 * ic0, 0, bar);
    }
    if (++islot == DEPTH) islot = 0;
    ++ti;
    ic0 += 128;
    if (ic0 == Kb) { ic0 = 0; irb16 += 16; }
  };
  int wrb = t / CPR, wwin = (t - wrb * CPR) / cpw, nwi = 0;   // next parameter window to request
  bool wmore = true;
  auto issue_window = [&]() {
    const int ps = nwi & 1;
    if (lane == 0) {
      const uint32_t dst = wins_c + uint32_t(ps) * SK_WIN_BYTES, bar = barP + uint32_t(ps) * 8u;
      sk_mbar_expect_tx(bar, ZK == 3 ? SK_WIN_BYTES : ZOFF);
      sk_tma_2d(dst, &tmS, wwin * SK_WIN_GROUPS, wrb * 16, bar);
      if constexpr (ZK == 3) sk_tma_2d(dst + ZOFF, &tmZ, (wrb * 8) & ~15, wwin * SK_WIN_GROUPS, bar);
    }
    ++nwi;
    if (++wwin == sp.WPR) { wwin = 0; ++wrb; }
    wmore = wrb * CPR + wwin * cpw < t1;
  };
  issue_window();
  if (wmore) issue_window();
#pragma unroll 1
  for (int i = 0; i < DEPTH && ti < t1; ++i) issue_chunk();

  // ---- consume side ----
  int cslot = 0, nwin = 0;
  uint32_t cphase = 0, wbase = 0;
  const uint32_t a_off = uint32_t(min(r, p.M - 1)) * 512u + uint32_t(q) * 64u;
  const uint32_t rowoff_a = rr * 128, rowoff_b = (rr + 8) * 128, sw = uint32_t(rr & 7);
  const uint32_t zsh = 4u * uint32_t(rr);   // nibble of row rr in the low word (rows 0..7), of row rr + 8 in the high word

  float parked[4] = {0.f, 0.f, 0.f, 0.f};
  bool has_parked = false;
  auto publish_parked = [&]() {
    if (has_parked) {
      reinterpret_cast<float4*>(sp.slots + size_t(ri) * SK_SLOT_FLOATS)[lane] = make_float4(parked[0], parked[1], parked[2], parked[3]);
      __threadfence();
      __syncwarp();
      if (lane == 0) asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(sp.flags + ri), "l"(sp.nonce) : "memory");
      has_parked = false;
    }
  };

  while (t < t1) {
    const int rb = t / CPR;
    int kc = t - rb * CPR;
    const int seg_n = min(t1 - t, CPR - kc);
    const bool seg_parks = kc != 0;   // a segment that starts inside the row block is a contribution, not the owner
    const bool seg_closes = kc + seg_n == CPR;
    const int n_a = rb * 16 + rr, n_b = n_a + 8;
    const uint32_t zrb8 = ZOFF + uint32_t(rb & 1) * 8u;
    float acc_t[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t fold[4];
    auto set_fold = [&](uint32_t za, uint32_t zb) {
      fold[0] = NEGMAGIC + za * 0x00010001u;
      fold[1] = NEGMAGIC + zb * 0x00010001u;
      fold[2] = NEGMAGIC_HI + za * ZMUL_HI;
      fold[3] = NEGMAGIC_HI + zb * ZMUL_HI;
    };
    set_fold(uint32_t(p.zp_const), uint32_t(p.zp_const));
    int win_left = 0, kw = 0;   // chunks left in the current parameter window; chunk index inside the window
#pragma unroll 1
    for (int i = 0; i < seg_n; ++i, ++kc) {
      if (win_left == 0) {   // warp-uniform: enter the next window of 8 groups
        const int ps = nwin & 1;
        sk_mbar_wait(barP + uint32_t(ps) * 8u, uint32_t(nwin >> 1) & 1u);
        wbase = wins_c + uint32_t(ps) * SK_WIN_BYTES;
        ++nwin;
        if (nwin >= 2 && wmore) {   // the other slot held the window before this one: all of it is in registers
          __syncwarp();
          issue_window();
        }
        kw = kc & (cpw - 1);
        win_left = cpw - kw;
      }
      --win_left;
      // raw group parameters of this chunk
      uint32_t sa2, sb2;
      uint2 z0 = make_uint2(0u, 0u), z1 = make_uint2(0u, 0u);
      if constexpr (GPC == 2) {
        const uint32_t po = uint32_t(kw) * 4u;   // groups 2 kw and 2 kw + 1: two fp16 scales per row in one word
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(sa2) : "r"(wbase + uint32_t(rr) * 16u + po));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(sb2) : "r"(wbase + uint32_t(rr + 8) * 16u + po));
        if constexpr (ZK == 3) {
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(z0.x), "=r"(z0.y) : "r"(wbase + zrb8 + po * 8u));
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(z1.x), "=r"(z1.y) : "r"(wbase + zrb8 + po * 8u + 16u));
        }
      } else {
        const uint32_t gl = uint32_t(2 * kw) >> lg_spg;
        asm volatile("ld.shared.u16 %0, [%1];" : "=r"(sa2) : "r"(wbase + uint32_t(rr) * 16u + gl * 2u));
        asm volatile("ld.shared.u16 %0, [%1];" : "=r"(sb2) : "r"(wbase + uint32_t(rr + 8) * 16u + gl * 2u));
        if constexpr (ZK == 3)
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(z0.x), "=r"(z0.y) : "r"(wbase + zrb8 + gl * 16u));
      }
      ++kw;
      sk_mbar_wait(barF + uint32_t(cslot) * 8u, cphase);
      const uint32_t tile = wring_c + uint32_t(cslot) * SK_WBYTES;
      const uint32_t atile = aring_c + uint32_t(cslot) * abytes + a_off;
      if (++cslot == DEPTH) { cslot = 0; cphase ^= 1u; }
      if constexpr (MINB == 2) {
        uint32_t wreg[2][2][4], R[2][16];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint32_t ch16 = ((uint32_t(j * 4 + q)) ^ sw) * 16;
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wreg[j][0][0]), "=r"(wreg[j][0][1]), "=r"(wreg[j][0][2]), "=r"(wreg[j][0][3]) : "r"(tile + rowoff_a + ch16));
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wreg[j][1][0]), "=r"(wreg[j][1][1]), "=r"(wreg[j][1][2]), "=r"(wreg[j][1][3]) : "r"(tile + rowoff_b + ch16));
#pragma unroll
          for (int x = 0; x < 4; ++x)
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(R[j][4 * x]), "=r"(R[j][4 * x + 1]), "=r"(R[j][4 * x + 2]), "=r"(R[j][4 * x + 3])
                         : "r"(atile + uint32_t(j * 256 + x * 16)));
        }
        // The whole chunk is in registers: request the chunk DEPTH ahead into this slot while we compute.  No proxy fence:
        // the ld.shared above were issued (in order, by every lane -- __syncwarp) before the request, complete within tens
        // of cycles, and the TMA write lands after an L2 / DRAM round trip; a fence.proxy.async here (MEMBAR.ALL.CTA +
        // FENCE.VIEW.ASYNC) would stall every chunk.
        if (ti < t1) {
          __syncwarp();
          issue_chunk();
        }
        // Group parameters of the two steps (GPC == 1: one group, both steps share it).
        float s_a[2], s_b[2];
        uint32_t fold2[2][4];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (GPC == 2 || j == 0) {
            if constexpr (ZK == 3) {
              const uint2 z = (GPC == 2 && j == 1) ? z1 : z0;
              set_fold((z.x >> zsh) & 15u, (z.y >> zsh) & 15u);
            }
            s_a[j] = raw_to_float<T>(uint16_t((GPC == 2 && j == 1) ? (sa2 >> 16) : sa2));
            s_b[j] = raw_to_float<T>(uint16_t((GPC == 2 && j == 1) ? (sb2 >> 16) : sb2));
          } else {
            s_a[j] = s_a[0]; s_b[j] = s_b[0];
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) fold2[j][u] = fold[u];
        }
        // The two MMA steps of the chunk are independent (separate accumulators), so their chains are interleaved: four
        // dependent HMMA chains per warp instead of two -- the kernel is latency-bound at 4 warps per scheduler.
        float acc_w[2][4], acc_f[2][4];
#pragma unroll
        for (int wi = 0; wi < WPS; ++wi) {
          uint32_t ha[2][NP], hb[2][NP];
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if constexpr (HI) {
              const uint32_t xa = wreg[j][0][wi], ya = wreg[j][0][wi] >> 8, xb = wreg[j][1][wi], yb = wreg[j][1][wi] >> 8;
              ha[j][0] = lop3_and_or(xa, 0x000f000fu, MAGIC); ha[j][1] = lop3_and_or(xa, 0x00f000f0u, MAGIC_HI);
              ha[j][2] = lop3_and_or(ya, 0x000f000fu, MAGIC); ha[j][3] = lop3_and_or(ya, 0x00f000f0u, MAGIC_HI);
              hb[j][0] = lop3_and_or(xb, 0x000f000fu, MAGIC); hb[j][1] = lop3_and_or(xb, 0x00f000f0u, MAGIC_HI);
              hb[j][2] = lop3_and_or(yb, 0x000f000fu, MAGIC); hb[j][3] = lop3_and_or(yb, 0x00f000f0u, MAGIC_HI);
            } else {
              decode_u4x8_raw<T>(wreg[j][0][wi], ha[j]);
              decode_u4x8_raw<T>(wreg[j][1][wi], hb[j]);
            }
          }
#pragma unroll
          for (int jj = 0; jj < NP / 2; ++jj) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const uint32_t af[4] = {ha[j][2 * jj], hb[j][2 * jj], ha[j][2 * jj + 1], hb[j][2 * jj + 1]};
              uint32_t b0, b1;
              if constexpr (IL) {
                b0 = R[j][wi * NP + 2 * jj]; b1 = R[j][wi * NP + 2 * jj + 1];
              } else {
                b0 = __byte_perm(R[j][wi * NP + jj], R[j][wi * NP + jj + NP / 2], 0x5410);
                b1 = __byte_perm(R[j][wi * NP + jj], R[j][wi * NP + jj + NP / 2], 0x7632);
              }
              if (wi == 0 && jj == 0) {   // first MMA of each chain: C = 0, accumulators never need zeroing
                mma_16816_z<T>(acc_w[j], af, b0, b1);
                mma_16816_z<T>(acc_f[j], fold2[j], b0, b1);
              } else {
                mma_16816<T>(acc_w[j], af, b0, b1);
                mma_16816<T>(acc_f[j], fold2[j], b0, b1);
              }
            }
          }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int u = 0; u < 4; ++u) acc_t[u] = fmaf((u < 2) ? s_a[j] : s_b[j], acc_w[j][u] + acc_f[j][u], acc_t[u]);
          } else {
        // ---- lean variant: one MMA step at a time (24 live data registers instead of 48), two chains ----
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint32_t wa[4], wb[4], Rj[16];
          const uint32_t ch16 = ((uint32_t(j * 4 + q)) ^ sw) * 16;
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wa[0]), "=r"(wa[1]), "=r"(wa[2]), "=r"(wa[3]) : "r"(tile + rowoff_a + ch16));
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wb[0]), "=r"(wb[1]), "=r"(wb[2]), "=r"(wb[3]) : "r"(tile + rowoff_b + ch16));
#pragma unroll
          for (int x = 0; x < 4; ++x)
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(Rj[4 * x]), "=r"(Rj[4 * x + 1]), "=r"(Rj[4 * x + 2]), "=r"(Rj[4 * x + 3])
                         : "r"(atile + uint32_t(j * 256 + x * 16)));
          if (j == 1 && ti < t1) {   // the second step has left the slot: request the chunk DEPTH ahead into it
            __syncwarp();
            issue_chunk();
          }
          float s_a, s_b;
          if (GPC == 2 || j == 0) {
            if constexpr (ZK == 3) {
              const uint2 z = (GPC == 2 && j == 1) ? z1 : z0;
              set_fold((z.x >> zsh) & 15u, (z.y >> zsh) & 15u);
            }
          }
          s_a = raw_to_float<T>(uint16_t((GPC == 2 && j == 1) ? (sa2 >> 16) : sa2));
          s_b = raw_to_float<T>(uint16_t((GPC == 2 && j == 1) ? (sb2 >> 16) : sb2));
          float acc_w[4], acc_f[4];
#pragma unroll
          for (int wi = 0; wi < WPS; ++wi) {
            uint32_t ha[NP], hb[NP];
            if constexpr (HI) {
              const uint32_t xa = wa[wi], ya = wa[wi] >> 8, xb = wb[wi], yb = wb[wi] >> 8;
              ha[0] = lop3_and_or(xa, 0x000f000fu, MAGIC); ha[1] = lop3_and_or(xa, 0x00f000f0u, MAGIC_HI);
              ha[2] = lop3_and_or(ya, 0x000f000fu, MAGIC); ha[3] = lop3_and_or(ya, 0x00f000f0u, MAGIC_HI);
              hb[0] = lop3_and_or(xb, 0x000f000fu, MAGIC); hb[1] = lop3_and_or(xb, 0x00f000f0u, MAGIC_HI);
              hb[2] = lop3_and_or(yb, 0x000f000fu, MAGIC); hb[3] = lop3_and_or(yb, 0x00f000f0u, MAGIC_HI);
            } else {
              decode_u4x8_raw<T>(wa[wi], ha);
              decode_u4x8_raw<T>(wb[wi], hb);
            }
#pragma unroll
            for (int jj = 0; jj < NP / 2; ++jj) {
              const uint32_t af[4] = {ha[2 * jj], hb[2 * jj], ha[2 * jj + 1], hb[2 * jj + 1]};
              uint32_t b0, b1;
              if constexpr (IL) {
                b0 = Rj[wi * NP + 2 * jj]; b1 = Rj[wi * NP + 2 * jj + 1];
              } else {
                b0 = __byte_perm(Rj[wi * NP + jj], Rj[wi * NP + jj + NP / 2], 0x5410);
                b1 = __byte_perm(Rj[wi * NP + jj], Rj[wi * NP + jj + NP / 2], 0x7632);
              }
              if (wi == 0 && jj == 0) {
                mma_16816_z<T>(acc_w, af, b0, b1);
                mma_16816_z<T>(acc_f, fold, b0, b1);
              } else {
                mma_16816<T>(acc_w, af, b0, b1);
                mma_16816<T>(acc_f, fold, b0, b1);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) acc_t[u] = fmaf((u < 2) ? s_a : s_b, acc_w[u] + acc_f[u], acc_t[u]);
        }
      }
    }
    t += seg_n;

    if (seg_parks) {
      // Contribution to a row block owned by another range (only the FIRST segment of a range can be one).  It is
      // published at the very end of the warp's life: a release fence here would wait for the TMA requests in flight.
#pragma unroll
      for (int u = 0; u < 4; ++u) { parked[u] = acc_t[u]; }
      has_parked = true;
    } else {
      // this range owns the row block: add the parked first segments of the ranges that cover the rest of it
      if (!seg_closes) {
        publish_parked();   // (this is the last segment of the range: nothing of mine is in flight any more)
        const long long rb_end = (long long)(rb + 1) * CPR;
        for (int rj = ri + 1; rj < sp.Wtot; ++rj) {
          const long long b = sk_range_begin(rj, sp.T, sp.Wtot), e = sk_range_begin(rj + 1, sp.T, sp.Wtot);
          if (b >= rb_end) break;
          if (b == e) continue;   // empty range
          unsigned long long f;
          do {
            asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(f) : "l"(sp.flags + rj) : "memory");
          } while (f != sp.nonce);
          asm volatile("fence.acq_rel.gpu;" ::: "memory");
          const float4 v = __ldcg(reinterpret_cast<const float4*>(sp.slots + size_t(rj) * SK_SLOT_FLOATS) + lane);
          acc_t[0] += v.x; acc_t[1] += v.y; acc_t[2] += v.z; acc_t[3] += v.w;
          __syncwarp();
          if (lane == 0) sp.flags[rj] = 0ull;
          if (e >= rb_end) break;
        }
      }
      if (2 * q < p.M) { sk_store<T>(p, 2 * q, n_a, acc_t[0]); sk_store<T>(p, 2 * q, n_b, acc_t[2]); }
      if (2 * q + 1 < p.M) { sk_store<T>(p, 2 * q + 1, n_a, acc_t[1]); sk_store<T>(p, 2 * q + 1, n_b, acc_t[3]); }
    }
  }
  publish_parked();
}

// ---------------------------------------------------------------------------------------------
// int8 activations (W2A8 / W4A8), exact int32 accumulation.  Weights are used as raw unsigned fields
// (mma .u8.s8); the constant zero point of the signed formats is removed with zp * sum_k(a), the sum
// produced on the tensor cores with an all-ones A fragment.
// ---------------------------------------------------------------------------------------------
template <int BITS, int NT>
__global__ void __launch_bounds__(NT == 1 ? 128 : MAX_KS * 32) __maxnreg__(NT == 1 ? 96 : (NT == 2 ? 128 : 208))
gemv_i8_kernel(const GemvParams p) {
  constexpr int WPS = BITS;            // words per thread per row per step (32 k)
  constexpr int STEP_BYTES = 16 * BITS;
  __shared__ int red[MAX_KS][16][8 * NT];
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
  const int n_a = rb * 16 + r;
  int step_begin, step_end;
  split_range(p.K / 128, p.ks, warp, step_begin, step_end);
  const int ns = step_end - step_begin;
  const size_t row_bytes = size_t(p.K) * BITS / 8;
  const uint8_t* wpa = p.W + size_t(n_a) * row_bytes + q * (4 * WPS) + size_t(step_begin) * STEP_BYTES;
  const uint8_t* wpb = wpa + 8 * row_bytes;
  const uint4* ap[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int m = min(8 * t + r, p.M - 1);
    ap[t] = reinterpret_cast<const uint4*>(reinterpret_cast<const int8_t*>(p.A) + size_t(m) * p.K) + step_begin * 8 + q * 2;
  }
  const uint32_t ones[4] = {0x01010101u, 0x01010101u, 0x01010101u, 0x01010101u};
  int acc[NT][4], asum[NT][4];
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[t][j] = asum[t][j] = 0;

  auto process = [&](const uint32_t (&wa)[WPS], const uint32_t (&wb)[WPS]) {
    uint32_t da[8], db[8];  // 8 byte-quads = 32 k per row, natural k order
#pragma unroll
    for (int wi = 0; wi < WPS; ++wi) {
      if constexpr (BITS == 2) {
        uint32_t ta[4], tb[4];
        decode_u2x16_to_u8(wa[wi], 0u, ta);
        decode_u2x16_to_u8(wb[wi], 0u, tb);
#pragma unroll
        for (int x = 0; x < 4; ++x) { da[4 * wi + x] = ta[x]; db[4 * wi + x] = tb[x]; }
      } else {
        uint32_t ta[2], tb[2];
        decode_u4x8_to_u8(wa[wi], 0u, ta);
        decode_u4x8_to_u8(wb[wi], 0u, tb);
#pragma unroll
        for (int x = 0; x < 2; ++x) { da[2 * wi + x] = ta[x]; db[2 * wi + x] = tb[x]; }
      }
    }
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const uint4 v0 = __ldg(ap[t]), v1 = __ldg(ap[t] + 1);
      const uint32_t R[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
      ap[t] += 8;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t af[4] = {da[2 * j], db[2 * j], da[2 * j + 1], db[2 * j + 1]};
        mma_16832_u8s8(acc[t], af, R[2 * j], R[2 * j + 1]);
        if (p.zp_const) mma_16832_u8s8(asum[t], ones, R[2 * j], R[2 * j + 1]);
      }
    }
  };

  if (ns > 0) {
    uint32_t wq[PF][2][WPS];
    const uint8_t* wnext_a = wpa;
    const uint8_t* wnext_b = wpb;
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      if (u < ns) { load_w<BITS>(wnext_a, wq[u][0]); load_w<BITS>(wnext_b, wq[u][1]); }
      wnext_a += STEP_BYTES; wnext_b += STEP_BYTES;
    }
    pdl_wait();
    auto chunk = [&](auto guard_tag, int s) {
      constexpr bool GUARD = decltype(guard_tag)::value;
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        if (!GUARD || s + u < ns) {
          process(wq[u][0], wq[u][1]);
          if (!GUARD || s + u + PF < ns) { load_w<BITS>(wnext_a, wq[u][0]); load_w<BITS>(wnext_b, wq[u][1]); }
          wnext_a += STEP_BYTES; wnext_b += STEP_BYTES;
        }
      }
    };
    int s = 0;
#pragma unroll 1
    for (; s + 2 * PF <= ns; s += PF) chunk(std::false_type{}, s);
#pragma unroll 1
    for (; s < ns; s += PF) chunk(std::true_type{}, s);
  }
  if (ns <= 0) pdl_wait();
  pdl_launch_dependents();
#pragma unroll
  for (int t = 0; t < NT; ++t) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[t][j] -= p.zp_const * asum[t][j & 1];
    red[warp][r][8 * t + 2 * q] = acc[t][0];
    red[warp][r][8 * t + 2 * q + 1] = acc[t][1];
    red[warp][r + 8][8 * t + 2 * q] = acc[t][2];
    red[warp][r + 8][8 * t + 2 * q + 1] = acc[t][3];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 16 * 8 * NT; idx += blockDim.x) {
    const int row = idx & 15, m = idx >> 4;
    if (m >= p.M) continue;
    int v = 0;
    for (int w = 0; w < p.ks; ++w) v += red[w][row][m];
    const int n = rb * 16 + row;
    const int b = p.bias ? int(reinterpret_cast<const int8_t*>(p.bias)[n]) : 0;
    const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
    for (int d = 0; d < p.out.n; ++d) {
      void* Cd = p.out.ptr[d];
      switch (p.out_dtype) {
        case BB_I32: reinterpret_cast<int*>(Cd)[o] = v + b; break;
        case BB_I8: reinterpret_cast<int8_t*>(Cd)[o] = int8_t(int8_t(v) + b); break;
        case BB_F32: reinterpret_cast<float*>(Cd)[o] = float(v) + float(b); break;
        case BB_F16: reinterpret_cast<__half*>(Cd)[o] = __hadd(__int2half_rn(v), __int2half_rn(b)); break;
        default: reinterpret_cast<__nv_bfloat16*>(Cd)[o] = __hadd(__int2bfloat16_rn(v), __int2bfloat16_rn(b));
      }
    }
  }
}

GemvParams make_params(const MatmulArgs& a) {
  GemvParams p;
  const bb_matmul_desc& d = a.d;
  p.A = a.A; p.W = (const uint8_t*)a.W; p.scale = d.with_scaling ? a.scale : nullptr;
  p.zeros = d.with_zeros ? a.zeros : nullptr; p.bias = d.with_bias ? a.bias : nullptr; p.out = make_outspec(a);
  p.M = a.m; p.N = d.N; p.K = d.K;
  p.g = a.gsize(); p.G = a.groups();
  p.with_scaling = d.with_scaling;
  p.zmode = d.with_zeros ? (d.zeros_mode + 1) : 0;
  p.zp_const = (d.w_fmt == BB_W_INT) ? (1 << (d.w_bits - 1)) : 0;
  p.out_dtype = d.out_dtype;
  p.ks = 1;
  return p;
}

// K splits per 16-row block (= warps per CTA): the largest count for which EVERY CTA of the grid is resident at once
// (occupancy queried from the runtime for this kernel instantiation, cached).  When not even two warps per CTA fit in one wave
// (N >= ~24k rows), the full split is used and the grid runs in several waves rather than with one resident warp per row
// block (`BB_GEMV_KS` sweeps it).
template <typename KernelT>
int pick_ks(KernelT kernel, int (&occ_cache)[MAX_KS + 1], int max_ks, int row_blocks, int steps, int stage_bytes) {
  const int sms = device_sm_count();
  const char* ks_e = getenv("BB_GEMV_KS");   // tuning / test hook, read per launch
  const int ks_env = ks_e ? atoi(ks_e) : 0;
  if (ks_env >= 1 && ks_env <= max_ks && ks_env <= steps) return ks_env;
  for (int ks = max_ks; ks >= 2; --ks) {
    if (ks > steps) continue;
    if (occ_cache[ks] < 0) {
      int occ = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, ks * 32, size_t(stage_bytes)) != cudaSuccess) occ = 0;
      occ_cache[ks] = occ;
    }
    if (row_blocks <= sms * occ_cache[ks]) return ks;
  }
  return std::max(1, std::min(max_ks, steps));
}

bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("BB_PDL"); return e ? atoi(e) != 0 : true; }();
  return on;
}

#define BB_GEMV_GO(KERNEL, MAXKS)                                              \
  {                                                                            \
    static int occ_cache_store[5][MAX_KS + 1];                                 \
    static bool occ_init = false;                                              \
    if (!occ_init) { for (auto& row : occ_cache_store) for (int& v : row) v = -1; occ_init = true; } \
    if (stage_bytes) for (int& v : occ_cache_store[1]) v = -1;  /* staged: smem depends on K -> recompute */ \
    int (&occ_cache)[MAX_KS + 1] = occ_cache_store[stage_bytes ? 1 : 0];       \
    p.ks = pick_ks(KERNEL, occ_cache, MAXKS, nb, p.K / 128, stage_bytes);      \
    cudaLaunchConfig_t cfg = {};                                               \
    cfg.gridDim = dim3(nb); cfg.blockDim = dim3(p.ks * 32);                    \
    cfg.dynamicSmemBytes = stage_bytes; cfg.stream = a.stream;                 \
    cudaLaunchAttribute attr[1];                                               \
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;           \
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0; \
    cfg.attrs = attr; cfg.numAttrs = 1;                                        \
    BB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, KERNEL, p));                        \
  }

typedef CUresult (*SkEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
SkEncodeFn sk_encode() {
  static SkEncodeFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
    return reinterpret_cast<SkEncodeFn>(f);
  }();
  return fn;
}

int sk_sm_count() { return device_sm_count(); }
constexpr int SK_MAX_MINB = 4;   // CTAs per SM of the densest variant (sizes the workspace)
size_t sk_workspace_bytes() { return size_t(SK_MAX_MINB * sk_sm_count() * SK_CONSUMERS) * (SK_SLOT_FLOATS * 4 + 8) + 256; }

bool gemv_sk_shape_ok(const bb_matmul_desc& d, int m) {
  if (m < 1 || m > SK_MAX_M || d.w_bits != 4 || !d.with_scaling) return false;
  if (d.with_zeros && d.zeros_mode != BB_ZEROS_QUANTIZED) return false;
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if (d.K % 256 || g % 128 || d.K % g || ((g / 128) & (g / 128 - 1))) return false;   // group size 128 << n
  const int G = d.K / g;
  if (G % SK_WIN_GROUPS) return false;
  if (d.N % 32) return false;
  return true;
}

template <typename T, bool IL>
int launch_gemv_sk(const MatmulArgs& a, const GemvParams& p) {
  SkEncodeFn enc = sk_encode();
  CUtensorMap tmW, tmA, tmS, tmZ;
  cuuint32_t estr[2] = {1, 1};
  CUresult r;
  {
    cuuint64_t dims[2] = {cuuint64_t(p.K) / 2, cuuint64_t(p.N)};
    cuuint64_t strides[1] = {cuuint64_t(p.K) / 2};
    cuuint32_t box[2] = {128, 16};
    r = enc(&tmW, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(p.W), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(W) failed with CUresult %d", int(r)); return 4; }
  }
  {
    cuuint64_t dims[2] = {cuuint64_t(p.K), cuuint64_t(p.M)};
    cuuint64_t strides[1] = {cuuint64_t(p.K) * 2};
    cuuint32_t box[2] = {256, cuuint32_t(p.M)};
    r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(p.A), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(A) failed with CUresult %d", int(r)); return 4; }
  }
  {
    cuuint64_t dims[2] = {cuuint64_t(p.G), cuuint64_t(p.N)};
    cuuint64_t strides[1] = {cuuint64_t(p.G) * 2};
    cuuint32_t box[2] = {SK_WIN_GROUPS, 16};
    r = enc(&tmS, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(p.scale), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(scale) failed with CUresult %d", int(r)); return 4; }
  }
  tmZ = tmS;
  if (p.zmode == 3) {
    cuuint64_t dims[2] = {cuuint64_t(p.N) / 2, cuuint64_t(p.G)};
    cuuint64_t strides[1] = {cuuint64_t(p.N) / 2};
    cuuint32_t box[2] = {16, SK_WIN_GROUPS};
    r = enc(&tmZ, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(p.zeros), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(zeros) failed with CUresult %d", int(r)); return 4; }
  }
  SkParams sp;
  sp.g = p;
  sp.CPR = p.K / 256;
  sp.WPR = p.G / SK_WIN_GROUPS;
  sp.lg_spg = 0;
  while ((128 << sp.lg_spg) < p.g) ++sp.lg_spg;
  static const int depth_env = [] { const char* e = getenv("BB_SK_DEPTH"); const int v = e ? atoi(e) : 0; return (v >= 1 && v <= SK_DEPTH) ? v : SK_DEPTH; }();
  sp.depth = depth_env;
  sp.T = (long long)(p.N / 16) * sp.CPR;
  static const int minb_env = [] { const char* e = getenv("BB_SK_MINB"); const int v = e ? atoi(e) : 0; return (v >= 2 && v <= SK_MAX_MINB) ? v : 2; }();
  const int smem = sk_smem_bytes(p.M, sp.depth);
  int grid = 0;
#define BB_SK_GO2(ZKV, GPCV, MB)                                                                                            \
  {                                                                                                                \
    auto k = gemv_sk_kernel<T, IL, ZKV, GPCV, MB>;                                                                 \
    static int occ_dev[BB_MAX_DEVICES][SK_MAX_M + 1] = {};   /* cudaFuncSetAttribute is per device */           \
    int (&occ)[SK_MAX_M + 1] = occ_dev[current_device()];                                                         \
    if (!occ[p.M]) {                                                                                               \
      BB_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, sk_smem_bytes(SK_MAX_M, SK_DEPTH))); \
      int o = 0;                                                                                                   \
      BB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k, SK_THREADS, size_t(smem)));               \
      occ[p.M] = o < 1 ? -1 : (o > MB ? MB : o);                                                                   \
    }                                                                                                              \
    if (occ[p.M] < 0) { set_error("gemv_sk: kernel does not fit on this device"); return 4; }                      \
    const long long want = (sp.T + SK_CONSUMERS * SK_MIN_CHUNKS - 1) / (SK_CONSUMERS * SK_MIN_CHUNKS);            \
    grid = int(std::min<long long>(want, (long long)occ[p.M] * sk_sm_count()));                                    \
    sp.Wtot = grid * SK_CONSUMERS;                                                                                 \
    k<<<grid, SK_THREADS, smem, a.stream>>>(tmW, tmA, tmS, tmZ, sp);                                               \
  }
  // workspace: flags then slots; sized for the largest grid (2 CTAs per SM)
  sp.flags = reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(a.workspace) + 15) & ~uintptr_t(15));
  sp.slots = reinterpret_cast<float*>(sp.flags + SK_MAX_MINB * sk_sm_count() * SK_CONSUMERS);
  static std::atomic<unsigned long long> counter{0x9e3779b97f4a7c15ull};
  unsigned long long z = counter.fetch_add(0x9e3779b97f4a7c15ull);   // splitmix64: never 0 in practice, distinct per call
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  sp.nonce = (z ^ (z >> 31)) | 1ull;
  if (sp.T >= (1ll << 31)) { set_error("gemv_sk: problem too large"); return 4; }
  // the denser variants are instantiated for the headline configuration only (fp16, interleaved, quantized zeros, g = 128)
#define BB_SK_GO(ZKV, GPCV)                                                                                       \
  if constexpr (std::is_same<T, __half>::value && IL && ZKV == 3 && GPCV == 2) {                                  \
    if (minb_env == 4) BB_SK_GO2(ZKV, GPCV, 4) else if (minb_env == 3) BB_SK_GO2(ZKV, GPCV, 3) else BB_SK_GO2(ZKV, GPCV, 2) \
  } else BB_SK_GO2(ZKV, GPCV, 2)
  if (p.zmode == 3) { if (sp.lg_spg == 0) BB_SK_GO(3, 2) else BB_SK_GO(3, 1) }
  else { if (sp.lg_spg == 0) BB_SK_GO(0, 2) else BB_SK_GO(0, 1) }
#undef BB_SK_GO
#undef BB_SK_GO2
  BB_LAUNCH_CHECK();
  return 0;
}

template <typename T, int BITS, bool IL>
int launch_mma_nt(const MatmulArgs& a, GemvParams p) {
  const int nb = p.N / 16;
  const int nt = (p.M + 7) / 8;
  const int stage_bytes = 0;
#define BB_GEMV_NT(ZKV, SCV)                                                             \
  if (nt <= 1) BB_GEMV_GO((gemv_mma_kernel<T, BITS, IL, 1, ZKV, SCV>), 4) \
  else if (nt == 2) BB_GEMV_GO((gemv_mma_kernel<T, BITS, IL, 2, ZKV, SCV>), MAX_KS) \
  else BB_GEMV_GO((gemv_mma_kernel<T, BITS, IL, 4, ZKV, SCV>), MAX_KS)
  if (!p.with_scaling) { BB_GEMV_NT(0, false) }
  else if (p.zmode == 0) { BB_GEMV_NT(0, true) }
  else if (p.zmode == 1) { BB_GEMV_NT(1, true) }
  else if (p.zmode == 2) { BB_GEMV_NT(2, true) }
  else { BB_GEMV_NT(3, true) }
#undef BB_GEMV_NT
  BB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

size_t gemv_streamk_workspace_bytes() { return sk_workspace_bytes(); }

bool gemv_mma_supported(const bb_matmul_desc& d, int m) {
  if (m < 1 || m > 32) return false;
  if (d.w_tile != BB_TILE_ROW_MAJOR) return false;   // this kernel streams whole rows with plain loads
  if (d.a_dtype != BB_F16 && d.a_dtype != BB_BF16) return false;
  if (d.w_fmt != BB_W_UINT && d.w_fmt != BB_W_INT) return false;
  if (d.w_bits != 4 && d.w_bits != 2) return false;
  if (d.w_layout == BB_LAYOUT_INTERLEAVED_8) return false;
  if (d.N % 16 || d.K % 128) return false;
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if (g % 128 || d.K % g) return false;
  if (d.with_zeros && !d.with_scaling) return false;
  if (d.w_fmt == BB_W_INT && d.with_zeros) return false;
  if (d.out_dtype != BB_F16 && d.out_dtype != BB_BF16 && d.out_dtype != BB_F32) return false;
  if (d.with_zeros && d.zeros_mode == BB_ZEROS_QUANTIZED && (d.N * d.w_bits) % 8) return false;
  return true;
}

int launch_gemv_mma(const MatmulArgs& a) {
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15)) {
    set_error("gemv: A and W must be 16-byte aligned");
    return 5;
  }
  const GemvParams p = make_params(a);
  const bool il = a.d.w_layout == BB_LAYOUT_INTERLEAVED_16;
  const bool f16 = a.d.a_dtype == BB_F16;
  const int bits = a.d.w_bits;
  if (f16) {
    if (bits == 4) return il ? launch_mma_nt<__half, 4, true>(a, p) : launch_mma_nt<__half, 4, false>(a, p);
    return il ? launch_mma_nt<__half, 2, true>(a, p) : launch_mma_nt<__half, 2, false>(a, p);
  }
  if (bits == 4) return il ? launch_mma_nt<__nv_bfloat16, 4, true>(a, p) : launch_mma_nt<__nv_bfloat16, 4, false>(a, p);
  return il ? launch_mma_nt<__nv_bfloat16, 2, true>(a, p) : launch_mma_nt<__nv_bfloat16, 2, false>(a, p);
}

bool gemv_streamk_supported(const bb_matmul_desc& d, int m) {
  if (!gemv_mma_supported(d, m) || !gemv_sk_shape_ok(d, m)) return false;
  return sk_encode() != nullptr;
}

int launch_gemv_streamk(const MatmulArgs& a) {
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15) ||
      (reinterpret_cast<uintptr_t>(a.scale) & 15) || (reinterpret_cast<uintptr_t>(a.zeros) & 15)) {
    set_error("gemv_streamk: A, W, scale and zeros must be 16-byte aligned (TMA)");
    return 5;
  }
  if (!a.workspace || a.workspace_bytes < sk_workspace_bytes()) {
    set_error("gemv_streamk needs a workspace of %zu bytes (bb_workspace_bytes)", sk_workspace_bytes());
    return 5;
  }
  const GemvParams p = make_params(a);
  const bool il = a.d.w_layout == BB_LAYOUT_INTERLEAVED_16;
  if (a.d.a_dtype == BB_F16) return il ? launch_gemv_sk<__half, true>(a, p) : launch_gemv_sk<__half, false>(a, p);
  return il ? launch_gemv_sk<__nv_bfloat16, true>(a, p) : launch_gemv_sk<__nv_bfloat16, false>(a, p);
}

bool gemv_i8_supported(const bb_matmul_desc& d, int m) {
  if (m < 1 || m > 32) return false;
  if (d.w_tile != BB_TILE_ROW_MAJOR) return false;
  if (d.a_dtype != BB_I8 || d.accum_dtype != BB_I32) return false;
  if (d.w_fmt != BB_W_UINT && d.w_fmt != BB_W_INT) return false;
  if (d.w_bits != 4 && d.w_bits != 2) return false;
  if (d.w_layout != BB_LAYOUT_INTERLEAVED_8) return false;
  if (d.with_scaling || d.with_zeros) return false;
  if (d.N % 16 || d.K % 128) return false;
  return true;
}

int launch_gemv_i8(const MatmulArgs& a) {
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15)) {
    set_error("gemv: A and W must be 16-byte aligned");
    return 5;
  }
  GemvParams p = make_params(a);
  const int nb = p.N / 16;
  const int nt = (p.M + 7) / 8;
  const int stage_bytes = 0;
  if (a.d.w_bits == 2) {
    if (nt <= 1) BB_GEMV_GO((gemv_i8_kernel<2, 1>), 4)
    else if (nt == 2) BB_GEMV_GO((gemv_i8_kernel<2, 2>), MAX_KS)
    else BB_GEMV_GO((gemv_i8_kernel<2, 4>), MAX_KS)
  } else {
    if (nt <= 1) BB_GEMV_GO((gemv_i8_kernel<4, 1>), 4)
    else if (nt == 2) BB_GEMV_GO((gemv_i8_kernel<4, 2>), MAX_KS)
    else BB_GEMV_GO((gemv_i8_kernel<4, 4>), MAX_KS)
  }
  BB_LAUNCH_CHECK();
  return 0;
}

}  // namespace bb
