// bb_gemv.cu -- memory-bound streaming kernels for decode-sized M: m <= 8 where the m = 1 slab kernel (bb_gemv_slab.cu) does
// not apply, and up to m = 32 where the wgmma kernel does not.
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
#include "bb_gemv_mma.cuh"

namespace bb {

namespace {

__device__ __forceinline__ void mma_16832_u8s8(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// SWIGLU: bb_matmul_swiglu (gate/up interleaved W, p.out = C [M, N / 2])
template <typename T, int BITS, bool IL, int NT, int ZK, bool SC, bool SWIGLU = false>
__global__ void __launch_bounds__(gemv_max_ks(NT) * 32) __maxnreg__(gemv_mma_maxnreg(NT, ZK))
gemv_mma_kernel(const GemvParams p) {
  __shared__ float red[MAX_KS][16][8 * NT];
  gemv_mma_tile<T, BITS, IL, NT, ZK, SC, true, SWIGLU>(p, blockIdx.x, red);
}

__device__ __forceinline__ void mma_16832_s8s8(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// register budget of one gemv_i8 instance (W4A8 also carries the fp32 group sums and the group parameters)
constexpr int gemv_i8_maxnreg(int nt, bool w4a8) {
  return w4a8 ? (nt == 1 ? 128 : (nt == 2 ? 168 : 232)) : (nt == 1 ? 96 : (nt == 2 ? 128 : 208));
}

// bb_matmul_w4a8 on the streaming GEMV: 4-bit weights (interleaved-8), per-group fp32 scales sc.w_scale [N, G] and zero points.
// Warp w of the CTA owns whole groups (split_range over the G groups); each 128-k step decodes u - z into signed bytes for an
// s8.s8 MMA, and at a group's last step the exact int32 sums are promoted into fp32 with the group's scale (fetched one group
// ahead).  The CTA then sums the warps' fp32 partials in warp order and stores round_out(S / a_scale[m]) (+ bias).
template <int NT>
__device__ __forceinline__ void gemv_i8_w4a8(const GemvParams& p, const ScaledArgs& sc, int (&red)[MAX_KS][16][8 * NT]) {
  constexpr int BITS = 4, WPS = BITS, STEP_BYTES = 16 * BITS;
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
  const int n_a = rb * 16 + r, n_b = n_a + 8;
  const int spg = p.g / 128;   // steps per group
  int g_begin, g_end;
  split_range(p.G, p.ks, warp, g_begin, g_end);
  const int step_begin = g_begin * spg;
  const int ns = (g_end - g_begin) * spg;
  const size_t row_bytes = size_t(p.K) * BITS / 8;
  const uint8_t* wpa = p.W + size_t(n_a) * row_bytes + q * (4 * WPS) + size_t(step_begin) * STEP_BYTES;
  const uint8_t* wpb = wpa + 8 * row_bytes;
  const uint4* ap[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int m = min(8 * t + r, p.M - 1);
    ap[t] = reinterpret_cast<const uint4*>(reinterpret_cast<const int8_t*>(p.A) + size_t(m) * p.K) + step_begin * 8 + q * 2;
  }
  const uint8_t* qz = reinterpret_cast<const uint8_t*>(p.zeros);
  const float* scA = sc.w_scale + size_t(n_a) * p.G;
  const float* scB = sc.w_scale + size_t(n_b) * p.G;
  int acc[NT][4];
  float facc[NT][4];
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[t][j] = 0; facc[t][j] = 0.f; }
  // group gi's zero bytes / scales (z, s) and group gi + 1's (nz, ns_)
  int gi = g_begin, left = spg;
  uint32_t zA = 0, zB = 0, nzA = 0, nzB = 0;
  float sA = 0.f, sB = 0.f, nsA = 0.f, nsB = 0.f;
  auto fetch = [&](int g) {
    nzA = uint32_t(w4a8_zero(qz, p.N, g, n_a, p.zp_const)) * 0x01010101u;
    nzB = uint32_t(w4a8_zero(qz, p.N, g, n_b, p.zp_const)) * 0x01010101u;
    nsA = __ldg(scA + g);
    nsB = __ldg(scB + g);
  };
  auto enter = [&]() {   // group gi begins: its fetched parameters become current; fetch the next group's
    zA = nzA; zB = nzB; sA = nsA; sB = nsB;
    if (gi + 1 < g_end) fetch(gi + 1);
  };

  auto process = [&](const uint32_t (&wa)[WPS], const uint32_t (&wb)[WPS]) {
    uint32_t da[8], db[8];  // 8 byte-quads = 32 k per row, natural k order: u - z as signed bytes
#pragma unroll
    for (int wi = 0; wi < WPS; ++wi) {
      uint32_t ta[2], tb[2];
      decode_u4x8_to_u8(wa[wi], 0x80808080u, ta);
      decode_u4x8_to_u8(wb[wi], 0x80808080u, tb);
#pragma unroll
      for (int x = 0; x < 2; ++x) { da[2 * wi + x] = bytes_sub_zp(ta[x], zA); db[2 * wi + x] = bytes_sub_zp(tb[x], zB); }
    }
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const uint4 v0 = __ldg(ap[t]), v1 = __ldg(ap[t] + 1);
      const uint32_t R[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
      ap[t] += 8;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t af[4] = {da[2 * j], db[2 * j], da[2 * j + 1], db[2 * j + 1]};
        mma_16832_s8s8(acc[t], af, R[2 * j], R[2 * j + 1]);
      }
    }
    if (--left == 0) {   // the group's last step: promote (acc[t][0..1] are row n_a, acc[t][2..3] row n_b) and restart
#pragma unroll
      for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          facc[t][j] = w4a8_promote(facc[t][j], acc[t][j], j < 2 ? sA : sB);
          acc[t][j] = 0;
        }
      left = spg;
      ++gi;
      if (gi < g_end) enter();
    }
  };

  if (ns > 0) {
    fetch(gi);
    enter();
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
    red[warp][r][8 * t + 2 * q] = __float_as_int(facc[t][0]);
    red[warp][r][8 * t + 2 * q + 1] = __float_as_int(facc[t][1]);
    red[warp][r + 8][8 * t + 2 * q] = __float_as_int(facc[t][2]);
    red[warp][r + 8][8 * t + 2 * q + 1] = __float_as_int(facc[t][3]);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 16 * 8 * NT; idx += blockDim.x) {
    const int row = idx & 15, m = idx >> 4;
    if (m >= p.M) continue;
    float S = 0.f;
    for (int w = 0; w < p.ks; ++w) S = __fadd_rn(S, __int_as_float(red[w][row][m]));
    const int n = rb * 16 + row;
    store_out_dequant(p.out.ptr[0], size_t(m) * size_t(p.out.ld) + n, __fdiv_rn(S, sc.a_scale[m]), p.bias, n, p.out_dtype);
  }
}

// ---------------------------------------------------------------------------------------------
// int8 activations (W2A8 / W4A8), exact int32 accumulation.  Weights are used as raw unsigned fields
// (mma .u8.s8); the constant zero point of the signed formats is removed with zp * sum_k(a), the sum
// produced on the tensor cores with an all-ones A fragment.
// Scaled: bb_matmul_scaled -- the epilogue divides by sc.a_scale[m] (read after the PDL wait) and sc.w_scale[n] (store_out_scaled;
// bias in out_dtype).  The scales are a parameter of their own: GemvParams is also the grouped GEMV's, whose layout stays put.
// ---------------------------------------------------------------------------------------------
// W4A8 (BITS = 4): bb_matmul_w4a8, gemv_i8_w4a8 (red then holds fp32 bits).
template <int BITS, int NT, MatmulForm F>
__global__ void __launch_bounds__(gemv_max_ks(NT) * 32) __maxnreg__(gemv_i8_maxnreg(NT, F == MatmulForm::W4A8))
gemv_i8_kernel(const GemvParams p, const ScaledArgs sc) {
  constexpr int WPS = BITS;            // words per thread per row per step (32 k)
  constexpr int STEP_BYTES = 16 * BITS;
  __shared__ int red[MAX_KS][16][8 * NT];
  if constexpr (F == MatmulForm::W4A8) {
    gemv_i8_w4a8<NT>(p, sc, red);
    return;
  }
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
    if constexpr (F == MatmulForm::Scaled) {
      store_out_scaled(p.out.ptr[0], size_t(m) * size_t(p.out.ld) + n, v, sc.a_scale[m], sc.w_scale[n], p.bias, n,
                       p.out_dtype);
      continue;
    }
    const int b = p.bias ? int(reinterpret_cast<const int8_t*>(p.bias)[n]) : 0;
    const size_t o = size_t(m) * size_t(p.out.ld) + size_t(p.out.col0) + n;
    for (int d = 0; d < p.out.n; ++d) store_out_i32(p.out.ptr[d], o, v, b, p.out_dtype);
  }
}

// one CTA per 16-row block, the K split from pick_ks; `extra` follows p in the kernel's parameters
template <int NT, typename Kernel, typename... Extra>
int launch_gemv_kernel(Kernel kernel, KernelCache<MAX_KS + 1>& cache, GemvParams p, cudaStream_t stream, const Extra&... extra) {
  const int nb = p.N / 16;
  p.ks = pick_ks(cache, kernel, gemv_max_ks(NT), nb, p.K / 128);
  return launch_pdl(kernel, nb, p.ks * 32, 0, stream, pdl_enabled(), p, extra...);
}

template <typename T, int BITS, bool IL, bool SWIGLU>
int launch_mma_nt(const MatmulArgs& a, const GemvParams& p) {
  return gemv_mma_instance(p, p.M, [&](auto nt, auto zk, auto sc) {
    constexpr int NT = decltype(nt)::value;
    static KernelCache<MAX_KS + 1> cache;
    return launch_gemv_kernel<NT>(gemv_mma_kernel<T, BITS, IL, NT, decltype(zk)::value, decltype(sc)::value, SWIGLU>, cache, p,
                                  a.stream);
  });
}

// W4A8: the warps split the groups, not the steps (ks <= G)
template <int BITS, int NT, MatmulForm F>
int launch_i8_inst(const MatmulArgs& a, GemvParams p) {
  auto kernel = gemv_i8_kernel<BITS, NT, F>;
  static KernelCache<MAX_KS + 1> cache;
  p.ks = pick_ks(cache, kernel, gemv_max_ks(NT), p.N / 16, F == MatmulForm::W4A8 ? p.G : p.K / 128);
  return launch_pdl(kernel, p.N / 16, p.ks * 32, 0, a.stream, pdl_enabled(), p, a.scaled);
}

GemvParams make_params(const MatmulArgs& a) { return make_params(a.d, a.A, a.W, a.scale, a.zeros, a.bias, make_outspec(a), a.m); }

}  // namespace

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
  return dispatch_t_bits_il(a.d, [&](auto t, auto bits, auto il) {
    using T = typename decltype(t)::type;
    constexpr int BITS = decltype(bits)::value;
    constexpr bool IL = decltype(il)::value;
    return a.form == MatmulForm::SwiGLU ? launch_mma_nt<T, BITS, IL, true>(a, p) : launch_mma_nt<T, BITS, IL, false>(a, p);
  });
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
  const GemvParams p = make_params(a);
  return gemv_nt(p.M, [&](auto nt) {
    constexpr int NT = decltype(nt)::value;
    switch (a.form) {   // (bb_matmul_swiglu rejects int8 activations; bb_matmul_w4a8 takes 4-bit weights only)
      case MatmulForm::W4A8: return launch_i8_inst<4, NT, MatmulForm::W4A8>(a, p);
      case MatmulForm::Scaled:
        return a.d.w_bits == 2 ? launch_i8_inst<2, NT, MatmulForm::Scaled>(a, p) : launch_i8_inst<4, NT, MatmulForm::Scaled>(a, p);
      default:
        return a.d.w_bits == 2 ? launch_i8_inst<2, NT, MatmulForm::Plain>(a, p) : launch_i8_inst<4, NT, MatmulForm::Plain>(a, p);
    }
  });
}

}  // namespace bb
