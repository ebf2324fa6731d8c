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
#include <cuda.h>

#include <algorithm>
#include <mutex>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int TS_ROWS = 128;               // weight rows per CTA = two wgmma M = 64 warpgroups
constexpr int TS_CONSUMER_WARPS = 8;       // warps 0-7: two consumer warpgroups (wgmma needs warpgroup-aligned warps)
constexpr int TS_THREADS = (TS_CONSUMER_WARPS + 1) * 32;   // + warp 8: TMA producer

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
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
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
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

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

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

// FMT: 0 = integer formats (LOP3 magic-number decode), 1 = 16-entry table formats (NF4 / fp4; BITS = 4, compressed storage),
//      2 = 8-bit float weights (e4m3 / e5m2; BITS = 8)
template <typename T, int BITS, int BM, bool IL, int FMT = 0>
__global__ void __launch_bounds__(TS_THREADS, 1)
gemm_ts_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const TsParams p) {
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
  float bias_f[2] = {0.f, 0.f};
  if (p.bias) {
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
          auto put = [&](void* Cd) {
            switch (p.out_dtype) {
              case BB_I32: reinterpret_cast<int*>(Cd)[o] = a + b; break;
              case BB_I8: reinterpret_cast<int8_t*>(Cd)[o] = int8_t(int8_t(a) + b); break;
              case BB_F32: reinterpret_cast<float*>(Cd)[o] = float(a) + float(b); break;
              case BB_F16: reinterpret_cast<__half*>(Cd)[o] = __hadd(__int2half_rn(a), __int2half_rn(b)); break;
              default: reinterpret_cast<__nv_bfloat16*>(Cd)[o] = __hadd(__int2bfloat16_rn(a), __int2bfloat16_rn(b));
            }
          };
          put(C0);
          for (int d = 1; d < ndst; ++d) put(p.out.ptr[d]);
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

// out[m, n] = cast(sum_s ws[s][m][n]) (+ bias), stored to every destination of the OutSpec.  One thread = 4 consecutive n
// (N is a multiple of 128 here): 128-bit loads of the partials, 32-bit index arithmetic, one vector store per destination.
template <bool INT8>
__global__ void splitk_reduce_kernel(const TsParams p) {
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

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
std::once_flag g_encode_once;

EncodeTiledFn get_encode() {
  std::call_once(g_encode_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  });
  return g_encode;
}

int make_map_2d(CUtensorMap* map, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 4; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", int(r)); return 4; }
  return 0;
}

// BB_TILE_SLAB storage [N/32][row_bytes/512][32][512 B] as a 4-D tensor; box = {PRB bytes, 32 rows, 1 segment, 4 row blocks}
// lands in shared memory as the same dense [128 rows][PRB] tile the row-major 2-D box produces
int make_map_w_tiled(CUtensorMap* map, const void* base, uint64_t row_bytes, uint64_t rows, uint32_t prb) {
  EncodeTiledFn enc = get_encode();
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

template <typename T, int BITS, int BM, bool IL, int FMT = 0>
int launch_ts_inst(const MatmulArgs& a, const TsParams& p0) {
  using SM = TsSmem<T, BITS, BM>;
  using EI = ElemInfo<T>;
  auto kernel = gemm_ts_kernel<T, BITS, BM, IL, FMT>;
  static bool attr_set[BB_MAX_DEVICES] = {};   // cudaFuncSetAttribute is per device
  const int dev = current_device();
  if (!attr_set[dev]) {
    BB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kTotal));
    attr_set[dev] = true;
  }
  TsParams p = p0;
  p.m_tiles = (a.m + BM - 1) / BM;
  const int num_kb_total = a.d.K / EI::kKB;
  const int tiles = p.m_tiles * (a.d.N / TS_ROWS);
  p.splits = a.m <= 128 ? choose_splits(tiles, num_kb_total, device_sm_count()) : 1;
  if (p.splits > 1 && a.workspace_bytes < size_t(p.splits) * a.m * a.d.N * 4) p.splits = 1;  // no scratch given
  p.kb_per_split = num_kb_total / p.splits;
  p.ws = a.workspace;
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
  kernel<<<grid, TS_THREADS, smem_bytes, a.stream>>>(tmA, tmW, p);
  BB_LAUNCH_CHECK();
  if (p.splits > 1) {
    const size_t total = size_t(a.m) * a.d.N / 4;   // one thread per 4 consecutive n
    const int rthreads = 256;
    const int rblocks = int(std::min<size_t>((total + rthreads - 1) / rthreads, size_t(device_sm_count()) * 8));
    if (EI::kInt8) splitk_reduce_kernel<true><<<rblocks, rthreads, 0, a.stream>>>(p);
    else splitk_reduce_kernel<false><<<rblocks, rthreads, 0, a.stream>>>(p);
    BB_LAUNCH_CHECK();
  }
  return 0;
}

// activation rows per CTA: the wgmma N extent (m > 128 runs several 128-row tiles)
template <typename T, int BITS, bool IL, int FMT>
int launch_ts_bm(const MatmulArgs& a, const TsParams& p) {
  if (a.m <= 32) return launch_ts_inst<T, BITS, 32, IL, FMT>(a, p);
  if (a.m <= 64) return launch_ts_inst<T, BITS, 64, IL, FMT>(a, p);
  return launch_ts_inst<T, BITS, 128, IL, FMT>(a, p);
}
template <typename T, int BITS>
int launch_ts_layout(const MatmulArgs& a, const TsParams& p) {
  return a.d.w_layout == BB_LAYOUT_COMPRESSED ? launch_ts_bm<T, BITS, false, 0>(a, p) : launch_ts_bm<T, BITS, true, 0>(a, p);
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

size_t gemm_ts_workspace_bytes(const bb_matmul_desc& d, int m) {
  if (m > 128) return 0;
  const int kb = d.a_dtype == BB_I8 ? 128 : 64;
  const int bm = m <= 32 ? 32 : (m <= 64 ? 64 : 128);
  const int tiles = ((m + bm - 1) / bm) * (d.N / TS_ROWS);
  const int sp = choose_splits(tiles, d.K / kb, device_sm_count());
  return sp > 1 ? size_t(sp) * m * d.N * 4 : 0;
}

int gemm_ts_init(int) { return get_encode() ? 0 : 0; }

int launch_gemm_ts(const MatmulArgs& a) {
  const bb_matmul_desc& d = a.d;
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15)) {
    set_error("gemm_ts: A and W must be 16-byte aligned");
    return 5;
  }
  TsParams p;
  p.scale = d.with_scaling ? a.scale : nullptr;
  p.zeros = d.with_zeros ? a.zeros : nullptr;
  p.bias = d.with_bias ? a.bias : nullptr;
  p.out = make_outspec(a); p.M = a.m; p.N = d.N; p.K = d.K; p.g = a.gsize(); p.G = a.groups();
  p.mode = !d.with_scaling ? 0 : (!d.with_zeros ? 1 : 2 + d.zeros_mode);
  p.zp_const = d.w_fmt == BB_W_INT ? (1 << (d.w_bits - 1)) : 0;
  p.out_dtype = d.out_dtype; p.a_dtype = d.a_dtype; p.m_tiles = 1;
  p.lut = d.w_fmt == BB_W_NF ? a.lut : nullptr;
  p.w_fmt = d.w_fmt;
  if (d.w_fmt == BB_W_NF || d.w_fmt == BB_W_FP4)
    return d.a_dtype == BB_F16 ? launch_ts_bm<__half, 4, false, 1>(a, p) : launch_ts_bm<__nv_bfloat16, 4, false, 1>(a, p);
  if (d.w_fmt == BB_W_FP8_E4M3 || d.w_fmt == BB_W_FP8_E5M2)
    return d.a_dtype == BB_F16 ? launch_ts_bm<__half, 8, false, 2>(a, p) : launch_ts_bm<__nv_bfloat16, 8, false, 2>(a, p);
  if (d.a_dtype == BB_I8) return d.w_bits == 4 ? launch_ts_layout<int8_t, 4>(a, p) : launch_ts_layout<int8_t, 2>(a, p);
  if (d.a_dtype == BB_F16) return d.w_bits == 4 ? launch_ts_layout<__half, 4>(a, p) : launch_ts_layout<__half, 2>(a, p);
  return d.w_bits == 4 ? launch_ts_layout<__nv_bfloat16, 4>(a, p) : launch_ts_layout<__nv_bfloat16, 2>(a, p);
}

}  // namespace bb
