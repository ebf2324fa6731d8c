// bb_gemm_ts.cuh -- the per-tile pieces of the wgmma GEMM (bb_gemm_ts.cu): PTX wrappers, shared-memory layout, the LOP3
// decode into wgmma A fragments and per-row group parameters.  gemm_ts_kernel (bb_gemm_ts.cu) runs one tile per
// CTA; gemm_ts_grouped_kernel (bb_grouped_gemm.cu) runs every (expert, m-tile, n-tile) tile a persistent CTA takes.  Each kernel
// keeps its own k-loop and epilogue: sharing them as device functions changes gemm_ts_kernel's register allocation.  The
// design notes are at the top of bb_gemm_ts.cu.
#pragma once
#include <type_traits>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int TS_ROWS = 128;               // weight rows per CTA = two wgmma M = 64 warpgroups
constexpr int TS_CONSUMER_WARPS = 8;       // warps 0-7: two consumer warpgroups (wgmma needs warpgroup-aligned warps)
constexpr int TS_THREADS = (TS_CONSUMER_WARPS + 1) * 32;   // + warp 8: TMA producer

// ---------------------------------------------------------------------------------------------
// PTX wrappers (the shared-memory, mbarrier and 2-D TMA ones are in bb_common.cuh)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// K-major, 128B-swizzled shared-memory operand descriptor (rows of 128 B, 8-row swizzle atoms = 1024 B); the tile is
// 1024-byte aligned, so the base-offset field stays 0.  Advancing k by 32 bytes inside the atom adds 2 to the address field.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr & 0x3FFFFu) >> 4);  // start address, 16-byte units
  d |= uint64_t(1) << 16;                      // leading byte offset: unused for swizzled K-major
  d |= uint64_t(1024 >> 4) << 32;              // stride byte offset: 8 rows * 128 B
  d |= uint64_t(1) << 62;                      // SWIZZLE_128B
  return d;
}

// D[64 x N] (+)= A[64 x 16] (registers) * B[N x 16] (smem descriptor), and the int8 m64nNk32 variant (A unsigned or signed,
// B = int8 activations).  acc = 0 overwrites D.
template <int N>
struct Wgmma;
#include "bb_wgmma.inc"

// ---- the block-scaled FP8 GEMMs' PTX wrapper (gemm_fp8_kernel, bb_gemm_fp8.cu; gemm_fp8_grouped_kernel, bb_grouped_fp8.cu) ----
constexpr int FP8_KB = 128;   // k per block: one 128-byte swizzle row, one scale block

// D[64 x N] (+)= A[64 x 32] * B[N x 32], both e4m3 K-major 128B-swizzled shared-memory descriptors; acc = 0 overwrites D
template <int N>
struct WgmmaFp8;

template <>
struct WgmmaFp8<32> {
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(acc));
  }
};

template <>
struct WgmmaFp8<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(adesc), "l"(bdesc), "r"(acc));
  }
};

template <>
struct WgmmaFp8<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc), "r"(acc));
  }
};


// ---------------------------------------------------------------------------------------------
struct TsParams {
  const void* scale;
  const void* zeros;
  const void* bias;
  OutSpec out;
  int M, N, K;
  int g, G;
  int mode;       // 0 none, 1 scale, 2 original, 3 rescale, 4 quantized
  int zp_const;
  int out_dtype;
  int a_dtype;
  int m_tiles;
  int splits;        // split-K factor (>1: fp32 / int32 partials go to `ws`, reduced by splitk_reduce_kernel)
  int kb_per_split;  // k-blocks per split
  void* ws;          // [splits][M][N] partials
  const void* lut;   // NF4 table (16 x A_dtype), null otherwise
  int w_fmt;         // bb_wfmt (the table formats run the FMT = 1 instances)
  int w_tiled;       // BB_TILE_SLAB weight storage: tmW is the 4-D map {512 B, 32 rows, segments per row, row blocks}
};

// the parameters of M rows of A against W, up to the split-K fields and w_tiled (set by the launcher)
inline TsParams make_ts_params(const bb_matmul_desc& d, const void* scale, const void* zeros, const void* bias, const void* lut,
                               const OutSpec& out, int M) {
  TsParams p;
  p.scale = d.with_scaling ? scale : nullptr;
  p.zeros = d.with_zeros ? zeros : nullptr;
  p.bias = d.with_bias ? bias : nullptr;
  p.out = out; p.M = M; p.N = d.N; p.K = d.K;
  p.g = d.group_size <= 0 ? d.K : d.group_size; p.G = d.K / p.g;
  p.mode = !d.with_scaling ? 0 : (!d.with_zeros ? 1 : 2 + d.zeros_mode);
  p.zp_const = d.w_fmt == BB_W_INT ? (1 << (d.w_bits - 1)) : 0;
  p.out_dtype = d.out_dtype; p.a_dtype = d.a_dtype; p.m_tiles = 1;
  p.lut = d.w_fmt == BB_W_NF ? lut : nullptr;
  p.w_fmt = d.w_fmt;
  return p;
}

template <typename T>
struct ElemInfo {
  static constexpr bool kInt8 = false;
  static constexpr int kKB = 64;  // elements per 128-byte swizzle row
};
template <>
struct ElemInfo<int8_t> {
  static constexpr bool kInt8 = true;
  static constexpr int kKB = 128;
};

template <typename T, int BITS, int BM>
struct TsSmem {
  static constexpr int kPRB = ElemInfo<T>::kKB * BITS / 8;  // packed bytes per row per k-block
  static constexpr int kActBytes = BM * 128;
  static constexpr int kWBytes = TS_ROWS * kPRB;
  static constexpr int kStageBytes = kActBytes + kWBytes;
  static constexpr int kStagesRaw = (200 * 1024) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kBarBytes = 256;   // full[8] + empty[8]
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + 1024;  // + alignment slack
};

// byte t of each of four words: (w0.t, w1.t, w2.t, w3.t)
__device__ __forceinline__ uint32_t gather_byte(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t sel) {
  return __byte_perm(__byte_perm(w0, w1, sel), __byte_perm(w2, w3, sel), 0x5410);
}

// One weight row's share of a k-block in wgmma A-fragment order.  Thread t (= lane % 4) of a quad owns, per 16-element k
// step s (32 for int8), the element pairs (quads) at k = 2t (4t) and k = 2t + 8 (4t + 16):  out[2s] and out[2s + 1].  `src` is
// the shared address of the row's packed k-block.  16-bit targets return dequantised A_dtype pairs; int8 returns signed or
// unsigned bytes.  MODE: 0 none, 1 scale, 2 original, 3 rescale, 4 quantized.  IL = LOP3-interleaved storage (fast_decoding);
// !IL = plain compressed storage.  FMT: 0 integer, 1 16-entry table (NF4 / fp4), 2 8-bit float.
template <typename T, int BITS, int MODE, bool IL, int FMT>
__device__ __forceinline__ void dequant_row(uint32_t src, int t, uint32_t (&out)[8], const DqConst& c, const Lut4& lut,
                                            bool e5m2) {
  constexpr uint32_t M = TypeTraits<T>::kMagic;
  constexpr uint32_t MBYTES = ((M >> 8) & 0xffu) * 0x01010101u;  // magic high byte (0x64 / 0x43)
  auto fin = [&](uint32_t x) -> uint32_t { return dq_finish<T, MODE, BITS>(x, c.mz_lo, c); };
  const uint32_t bsel = uint32_t(t) | (uint32_t(t + 4) << 4);
  if constexpr (FMT == 2) {
    // 8-bit floats: the pair at k = 16s + 2t is half (t & 1) of word 4s + t/2.  e5m2 is the top byte of an fp16
    // (quantization.py:179-182); e4m3 follows the reference's bit trick (quantization.py:169-176); bf16 widens exactly.
    const uint32_t hsel = (t & 1) ? 0x3424u : 0x1404u;   // (byte 2j) << 8 | (byte 2j+1) << 24
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t w = lds32(src + uint32_t((j >> 1) * 4 + (j & 1) * 2 + (t >> 1)) * 4u);
      const uint32_t x = __byte_perm(w, 0u, hsel);
      uint32_t h = x;
      if (!e5m2) h = ((x & 0xC000C000u) | ((x >> 1) & 0x3F803F80u)) ^ 0x20002000u;
      if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        const float2 f = __half22float2(u32_as_h2(h));
        h = b2_as_u32(__floats2bfloat162_rn(f.x, f.y));
      }
      out[j] = MODE == 1 ? mul2<T>(h, c.s2) : h;
    }
  } else if constexpr (BITS == 4) {
    const uint4 p0 = lds128(src), p1 = lds128(src + 16);
    const uint32_t w[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};   // word j = k 8j .. 8j + 7
    if constexpr (IL && FMT == 0) {
      // interleaved: the pair (2t, 2t+1) of a word is nibble t of its low and high half
#pragma unroll
      for (int j = 0; j < 8; ++j) out[j] = fin(lop3_and_or(w[j] >> (4 * t), 0x000f000fu, M));
    } else {
      // compressed: the pair (2t, 2t+1) of a word is its byte t (low nibble first)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t pk = gather_byte(w[4 * h], w[4 * h + 1], w[4 * h + 2], w[4 * h + 3], bsel);
        if constexpr (FMT == 1) {
          uint32_t v[4];
          lut4_decode8(pk, lut, v);
#pragma unroll
          for (int i = 0; i < 4; ++i) out[4 * h + i] = MODE == 1 ? mul2<T>(v[i], c.s2) : v[i];
        } else {
          const uint32_t lo = pk & 0x0f0f0f0fu, hi = (pk >> 4) & 0x0f0f0f0fu;
          const uint32_t x = __byte_perm(lo, hi, 0x5140), y = __byte_perm(lo, hi, 0x7362);
          out[4 * h + 0] = fin(__byte_perm(x, MBYTES, 0x4140));
          out[4 * h + 1] = fin(__byte_perm(x, MBYTES, 0x4342));
          out[4 * h + 2] = fin(__byte_perm(y, MBYTES, 0x4140));
          out[4 * h + 3] = fin(__byte_perm(y, MBYTES, 0x4342));
        }
      }
    }
  } else {
    const uint4 pk = lds128(src);
    const uint32_t w[4] = {pk.x, pk.y, pk.z, pk.w};   // word s = k 16s .. 16s + 15
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      if constexpr (IL) {
        // interleaved: bytes (even 0-7, odd 0-7, even 8-15, odd 8-15) -- decode_u2x16_raw_interleaved
        const uint32_t lo = __byte_perm(w[s], 0, 0x4140), hi = __byte_perm(w[s], 0, 0x4342);
        out[2 * s] = fin(lop3_and_or(lo >> (2 * t), 0x00030003u, M));
        out[2 * s + 1] = fin(lop3_and_or(hi >> (2 * t), 0x00030003u, M));
      } else {
        // compressed: e_{2t}, e_{2t+1} at bits 4t, 4t + 2; e_{2t+8}, e_{2t+9} 16 bits up
        const uint32_t x = w[s] >> (4 * t);
        const uint32_t L = lop3_and_or(x, 0x00030003u, M), H = lop3_and_or(x >> 2, 0x00030003u, M);
        out[2 * s] = fin(__byte_perm(L, H, 0x5410));
        out[2 * s + 1] = fin(__byte_perm(L, H, 0x7632));
      }
    }
  }
}

// int8 activations (k32 steps): the quad at k = 32s + 4t of word (4-bit: 4s + t/2; 2-bit: 2s), and 16 further.
template <int BITS, bool IL>
__device__ __forceinline__ void dequant_row_i8(uint32_t src, int t, uint32_t (&out)[8], uint32_t zp4) {
  const uint32_t orv = zp4 ? 0x80808080u : 0u;
  if constexpr (BITS == 4) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t w = lds32(src + uint32_t((j >> 1) * 4 + (j & 1) * 2 + (t >> 1)) * 4u);
      uint32_t h;
      if constexpr (IL) {
        h = lop3_and_or(w >> (4 * (t & 1)), 0x0f0f0f0fu, orv);   // elements 0-3: low nibbles, 4-7: high nibbles
      } else {
        const uint32_t x = w >> (16 * (t & 1));
        h = __byte_perm(lop3_and_or(x, 0x0f0f0f0fu, orv), lop3_and_or(x >> 4, 0x0f0f0f0fu, orv), 0x5140);
      }
      out[j] = zp4 ? bytes_sub_zp(h, zp4) : h;
    }
  } else {
    const uint4 p0 = lds128(src), p1 = lds128(src + 16);
    const uint32_t w[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};   // word j = k 16j .. 16j + 15
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t h;
      if constexpr (IL) {
        h = lop3_and_or(w[j] >> (2 * t), 0x03030303u, orv);          // decode_u2x16_to_u8
      } else {
        const uint32_t v = __byte_perm(w[j], 0, uint32_t(t) * 0x1111u);  // byte t (elements 4t .. 4t + 3) in every byte
        h = (v & 0x03u) | ((v >> 2) & 0x0300u) | ((v >> 4) & 0x030000u) | ((v >> 6) & 0x03000000u) | orv;
      }
      out[j] = zp4 ? bytes_sub_zp(h, zp4) : h;
    }
  }
}

// Per-row group parameters, fetched one group ahead so their latency never sits in front of a decode.
template <int MODE, int BITS>
struct RowGroup {
  const uint16_t* sc;
  const uint16_t* z;
  const uint8_t* qz;
  size_t qz_stride;
  uint32_t qz_shift;
  uint16_t s_raw = 0, z_raw = 0;
  uint32_t qz_raw = 0;
  __device__ __forceinline__ void fetch(int gi) {
    if constexpr (MODE != 0) s_raw = __ldg(sc + gi);
    if constexpr (MODE == 2 || MODE == 3) z_raw = __ldg(z + gi);
    if constexpr (MODE == 4) qz_raw = __ldg(qz + size_t(gi) * qz_stride);
  }
  __device__ __forceinline__ void apply(DqConst& c, uint32_t magic) const {
    c.s2 = uint32_t(s_raw) * 0x00010001u;
    if constexpr (MODE == 2 || MODE == 3) {
      c.z2 = uint32_t(z_raw) * 0x00010001u;
      c.negz2 = c.z2 ^ 0x80008000u;
    }
    if constexpr (MODE == 4) c.mz_lo = magic + ((qz_raw >> qz_shift) & ((1u << BITS) - 1u)) * 0x00010001u;
  }
};

// The SwiGLU epilogue of the wgmma GEMMs (gemm_ts_kernel without split-K, gemm_ts_grouped_kernel): acc[4i + 2h + j] = C^T[row
// rA + 8h][column 8i + 2t + j], and the thread's rows nA = 16b + i and nB = nA + 8 (i < 8) are gate and up of
// C[m, 8b + i] = silu(gate) * up (row stride N / 2), for the rows m < m_end; bias is A_dtype [N] or null
template <typename T, int BM>
__device__ __forceinline__ void store_tile_swiglu(const float (&acc)[BM / 2], const TsParams& p, const T* bias, int m0, int m_end,
                                                  int nA, int nB, int t) {
  const float bg = bias ? TypeTraits<T>::to_float(bias[nA]) : 0.f, bu = bias ? TypeTraits<T>::to_float(bias[nB]) : 0.f;
  const size_t col = size_t(nA >> 4) * 8 + size_t(nA & 7);
#pragma unroll
  for (int i = 0; i < BM / 8; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + 8 * i + 2 * t + j;
      if (m >= m_end) continue;
      const float g = swiglu_operand(acc[4 * i + j], bias != nullptr, bg, p.out_dtype);
      const float u = swiglu_operand(acc[4 * i + 2 + j], bias != nullptr, bu, p.out_dtype);
      store_swiglu(p.out.ptr[0], size_t(m) * size_t(p.N / 2) + col, g, u, p.out_dtype);
    }
  }
}

}  // namespace

}  // namespace bb
