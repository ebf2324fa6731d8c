// bb_gemv_slab.cu -- m = 1 decode GEMV, W4A16 (fp16 / bf16 activations x 4-bit weights), the HBM-bound headline kernel.
//
// Replaces the reference's generated SIMT GEMV (bitblas/ops/general_matmul/tilelang/dequantize/gemv_dequantize_simt.py:164-262)
// and supersedes the round-1 register-queue kernel (bb_gemv.cu: 0.40 of the HBM roofline, bound by instruction issue and by
// DRAM round trips sitting on the warps' scoreboards).  Design, top down:
//
//   * WORK UNIT = [32 weight rows] x [1024 k] = 16 KB of packed weights out of the unchanged [N, K/2] storage, fetched by ONE TMA
//     request: box {128 x u32 = 512 B, 32 rows}, no swizzle.  The TMA engine pays per request and per box row, so one box
//     with long rows streams closer to the linear-read rate than a GEMM-style 128B-swizzled box or many small bulk copies
//     (tools/slabbench.cu compares them); bandwidth then depends only on the bytes in flight.  Units are ordered (row-block group, k, member) and cut into equal contiguous ranges over a persistent grid
//     (CTA-level stream-K): every SM streams the same number of bytes whatever N, K are; a 1024-row tensor-parallel shard
//     still fills all 132 SMs of an H100.
//   * a CTA = NG = 2 consumer GROUPS of 4 warps + an issuer warp + NF = 1 finisher warp around an S = 4-stage mbarrier ring, two
//     CTAs per SM.  Group g
//     consumes the units whose row block is g (mod NG) -- whole row blocks per group, so a group reduces, exchanges stream-K
//     partials and stores on its own, with a 128-thread named barrier; nothing ever synchronises the whole CTA.  The
//     consumers issue NO global loads: weights, activations, group parameters and activation sums are all in the stage when its
//     barrier flips, so nothing but ld.shared latency ever sits on a consumer scoreboard.
//   * consumer warp ws of a group owns K-slice ws of the unit (32 rows x 128 B = two 128-k steps): ld.shared.v4 -> LOP3 decode
//     into mma.sync.m16n8k16 A fragments (fp16: even nibbles as 1024+u, odd nibbles in place as 64+u) -> 8 HMMA per step and
//     16-row tile, the activations as the n8 side and shared by the warp's two row tiles.  The decode magic and the zero point
//     are never subtracted per element and never folded through extra MMAs (round 1 spent half its HMMAs on that): per step
//         acc += c1[row] * (partial - SM) + c2[row] * S,    SM = sum_k magic(k) a[k],  S = sum_k a[k]   (per 128-k step)
//     with (c1, c2) = (s, -s*z) for "original" / quantized zeros, (s, -z) for "rescale", (s, -s*2^(b-1)) for int formats.
//     This is exact in fp32 for ANY zero point (no integer / fraction split) and is three FMAs per output row per step.
//   * the ISSUER requests, the moment a ring slot is free, everything the unit needs: the weight box, the activation slab
//     (bulk copy) and the RAW group parameters (cp.async, 16 B per row); a FINISHER turns the slab into (SM, S) per step on the
//     tensor cores and the raw parameters into fp32 (c1, c2) pairs, then completes the stage barrier.  The DRAM system runs
//     saturated, so by Little's law EVERY request -- also a 1-byte parameter load -- takes (bytes in flight)/bandwidth, microseconds:
//     anything fetched with plain loads "a few units ahead" stalls its warp on every unit.
//   * L2 policy: the weight requests carry evict_first (each byte is read once).  Without it the weight stream pushes the
//     parameter sectors out of L2 between the two units that share one, and the parameters cost 0.65-2.5 us per launch on top of
//     the weights; tools/slab_stream.cu measures this (DESIGN.md 3.2).  Neither evict_last on the activation slab nor one L2
//     prefetch of a row block's contiguous scale run paid in that replay, so neither is used.
//   * stream-K fix-up: a range that starts inside a row block parks its group-reduced partial row sums in tagged 64-bit
//     workspace slots {call nonce, fp32}; the range holding the block's first unit adds them in fixed order (bit-reproducible)
//     and stores.  Ranges are handed out in reverse CTA order so an owner only waits for CTAs dispatched before it.
//   * programmatic dependent launch: weights and parameters of the first S units are requested before griddepcontrol.wait,
//     activations after it; launch_dependents is raised at kernel entry -- the grid is persistent and fully resident, so the
//     next kernel's CTAs can only take slots that this kernel's CTAs have vacated, and its prefetch overlaps our tail.
#include <atomic>
#include <algorithm>
#include <cstring>
#include <mutex>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int GS_ROWS = 32;                         // weight rows per unit (two 16-row MMA tiles)
constexpr int GS_GW = 4;                            // consumer warps per group = K-slices per unit
constexpr int GS_SLICE_BYTES = 128;                 // packed bytes per row per consumer warp per unit
constexpr int GS_ROW_BYTES = GS_GW * GS_SLICE_BYTES;   // packed bytes per row per unit: 512 B = one box row of the TMA request
constexpr int GS_KU = GS_ROW_BYTES * 2;             // k per unit (4-bit): 1024
constexpr int GS_STEPS = GS_KU / 128;               // 128-k steps per unit: 8
constexpr int GS_WBYTES = GS_ROWS * GS_ROW_BYTES;   // 16 KB, dense [32 rows][512 B]
constexpr int GS_ABYTES = GS_KU * 2;                // activation slab (one batch row): 2 KB
constexpr int GS_PBYTES = GS_STEPS * GS_ROWS * 8;   // (c1, c2) fp32 pairs [step][row]: 2 KB
constexpr int GS_SBYTES = GS_STEPS * 8;             // (SM, S) fp32 pairs [step]
constexpr int GS_RAWBYTES = 1024;                   // raw scales [32 rows][8 groups] fp16 + raw zeros (fp16 [32][8] or packed [8 groups][16 B])
constexpr int GS_RED_GROUP_BYTES = 2 * (2 * GS_GW) * GS_ROWS * 4;   // per group: two buffers x (4 warps x 2 k-halves) partials x 32 rows
constexpr int GS_NG = 2;                            // consumer groups per CTA
constexpr int GS_MINB = 2;                          // CTAs per SM
constexpr int GS_STAGES = 4;                        // ring depth
constexpr int GS_NF = 1;                            // finisher warps; finisher f serves the units i = f (mod GS_NF) of the range
// slot s of the ring always belongs to group s % GS_NG (and finisher s % GS_NF), which therefore sees every phase of the slot's
// barriers (a group that skipped a phase would mistake the parity of a later one for its own)
static_assert(GS_STAGES % GS_NG == 0 && GS_STAGES % GS_NF == 0, "the ring depth must be a multiple of the group and finisher counts");
constexpr int GS_THREADS = (GS_GW * GS_NG + 1 + GS_NF) * 32;   // consumers + issuer + finishers
constexpr int GS_SMEM_BYTES = 1024 + GS_STAGES * (GS_WBYTES + GS_ABYTES + GS_PBYTES + GS_RAWBYTES + GS_SBYTES) +
                              GS_NG * GS_RED_GROUP_BYTES + 32 * GS_STAGES + 64;
constexpr uint32_t GS_SUSPEND_NS = 20000;   // try_wait suspend-time hint: a waiting warp sleeps in hardware until the phase flips
                                             // instead of re-issuing the probe (the default limit re-issued it ~12 times per wait: 14 %
                                             // of all issued instructions were wait-loop instructions)

struct SlabParams {
  const void* A;
  const void* scale;
  const void* zeros;
  const void* bias;
  OutSpec out;
  int N, K;
  int G;            // groups per row
  int g128;         // group size / 128
  int with_scaling;
  int zmode;        // 0 none, 1 original, 2 rescale, 3 quantized
  int zp_const;
  int out_dtype;
  int UPR;          // units per 32-row block = ceil(K / 1024)
  int NRB;          // 32-row blocks = ceil(N / 32)
  int T;            // units in total, padded to whole row-block groups
  unsigned long long* ws;   // [grid][NG][32] tagged partial slots, zero-tagged on entry and on exit
  unsigned int nonce;
  const void* lut;   // NF4 table (16 x A_dtype) for the FMT = 1 instances, else null
  int w_fmt;         // bb_wfmt
  const uint8_t* Wt; // BB_TILE_SLAB storage (else null): unit (rb, ku) is the contiguous 16 KB block number rb * UPR + ku
  int fast_params;  // group size 128, 8-aligned group count, N % 32 == 0, aligned pointers: 16-byte async copies of the parameters
};

// the PTX wrappers only this kernel uses (the shared ones are in bb_common.cuh)
__device__ __forceinline__ void gs_mbar_expect_tx_only(uint32_t bar, uint32_t bytes) {   // no arrival
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gs_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "GS_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra GS_DONE_%=;\n"
      "bra GS_WAIT_%=;\n"
      "GS_DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity), "r"(GS_SUSPEND_NS) : "memory");
}
// (No nanosleep back-off between the helper warps' barrier probes: the schedulers are not short of issue slots, the consumer warps
//  are bound by their own dependent-instruction latency.)
__device__ __forceinline__ void gs_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ float2 gs_lds64f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
// the mbarrier receives one arrival from this thread when all its cp.async issued so far have landed
__device__ __forceinline__ void gs_cp_async_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t gs_lds8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void gs_sts64f(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void gs_sts32f(uint32_t addr, float a) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory"); }
__device__ __forceinline__ float gs_lds32f(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

template <typename T>
__device__ __forceinline__ void gs_store(const SlabParams& p, int n, float v) {
  const size_t o = size_t(p.out.col0) + n;   // m == 0
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

// bb_matmul_swiglu: C[0, col] = silu(g) * u of gate row n and up row n + 8, each rounded as gs_store rounds it (row stride N / 2)
template <typename T>
__device__ __forceinline__ void gs_store_swiglu(const SlabParams& p, int n, int col, float vg, float vu) {
  const T* bias = reinterpret_cast<const T*>(p.bias);
  const float g = swiglu_operand(vg, bias != nullptr, bias ? TypeTraits<T>::to_float(bias[n]) : 0.f, p.out_dtype);
  const float u = swiglu_operand(vu, bias != nullptr, bias ? TypeTraits<T>::to_float(bias[n + 8]) : 0.f, p.out_dtype);
  store_swiglu(p.out.ptr[0], size_t(col), g, u, p.out_dtype);
}

__device__ __forceinline__ int gs_range_begin(int ri, int T, int R) { return int((long long)ri * T / R); }


// FMT: 0 = uint4 / int4 (LOP3 magic decode, magic and zero point removed through the activation sums), 1 = 16-entry table formats
// (NF4 / fp4, compressed storage: PRMT table decode to exact A_dtype values, scale only -- the sums are not needed).
// SWIGLU: bb_matmul_swiglu (gate/up interleaved W, p.out = C [1, N / 2]); only the final store differs
template <typename T, bool IL, int FMT, bool SWIGLU = false>
__global__ void __launch_bounds__(GS_THREADS, GS_MINB)
gemv_slab_kernel(const __grid_constant__ CUtensorMap tmW, const SlabParams p) {
  constexpr bool F16 = std::is_same<T, __half>::value;
  constexpr bool HI = F16 && FMT == 0;   // odd nibbles decoded in place (mantissa bits 4..7 under exponent 2^6: exactly 64 + u)
  constexpr uint32_t MAGIC = TypeTraits<T>::kMagic;
  constexpr uint32_t MAGIC_HI = 0x54005400u;
  constexpr int NG = GS_NG, NF = GS_NF, S = GS_STAGES;
  constexpr int NCW = GS_GW * NG;            // consumer warps
  extern __shared__ uint8_t gs_raw[];
  const uint32_t base = (smem_u32(gs_raw) + 1023u) & ~1023u;
  const uint32_t Wb = base;                                   // [S][32 rows][512 B]
  const uint32_t Ab = Wb + uint32_t(S) * GS_WBYTES;           // [S][1024 halves]
  const uint32_t Pb = Ab + uint32_t(S) * GS_ABYTES;           // [S][8 steps][32 rows] (c1, c2)
  const uint32_t RAWb = Pb + uint32_t(S) * GS_PBYTES;         // [S] raw parameters: 512 B scales + 512 B zeros
  const uint32_t Sb = RAWb + uint32_t(S) * GS_RAWBYTES;       // [S][8 steps] (SM, S)
  const uint32_t Rb = Sb + uint32_t(S) * GS_SBYTES;           // [NG] group reduction buffers
  const uint32_t Bb = Rb + uint32_t(NG) * GS_RED_GROUP_BYTES; // wfull[S], pfull[S], praw[S], empty[S]
  const int lane = threadIdx.x & 31;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(Bb + 8u * s, 1);             // wfull: the weight box and the activation slab have landed (issuer arrival + transaction bytes)
      mbar_init(Bb + 8u * (S + s), 1);       // pfull: the finisher has written the unit's sums and (c1, c2) pairs
      mbar_init(Bb + 8u * (2 * S + s), 32);  // praw: the 32 issuer lanes' parameter copies landed
      mbar_init(Bb + 8u * (3 * S + s), GS_GW);   // empty: the four warps of the group that consumed the unit
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const int R = gridDim.x;
  const int ri = R - 1 - int(blockIdx.x);   // ranges in reverse CTA order: an owner waits only for CTAs dispatched before it
  const int t0 = gs_range_begin(ri, p.T, R), t1 = gs_range_begin(ri + 1, p.T, R);
  const int n_units = t1 - t0;
  const int UPR = p.UPR;
  const int Kb = p.K >> 1;                  // packed bytes per row
  const int steps_total = p.K >> 7;         // 128-k steps per row
  const int npre = min(S, n_units);
  // unit t -> (row block rb, k index ku): t = (q * UPR + ku) * NG + g, rb = q * NG + g
  auto unit_of = [&](int t, int& rb, int& ku) {
    const int g = t % NG, rest = t / NG;
    const int q = rest / UPR;
    ku = rest - q * UPR;
    rb = q * NG + g;
  };

  // ---- helper warps ----------------------------------------------------------------------------------------------------
  const uint16_t* scale16 = reinterpret_cast<const uint16_t*>(p.scale);
  const uint16_t* zeros16 = reinterpret_cast<const uint16_t*>(p.zeros);
  const uint8_t* zeros8 = reinterpret_cast<const uint8_t*>(p.zeros);
  auto unit_fast = [&](int rb, int ku) { return p.fast_params != 0 && (ku + 1) * GS_STEPS <= steps_total && rb < p.NRB; };

  if (warp == NCW) {
    // =========================== issuer warp ===========================
    // one weight TMA box {128 x u32 = 512 B, 32 rows} -> dense [32][512 B] (rows past N / columns past K/2 are zero-filled and
    // never stored / consumed; the transaction count is always the full box), the activation slab, the raw parameters
    // every weight byte is read exactly once: evict_first keeps the stream from displacing the parameter sectors and activation
    // slabs that later units read again (tools/slab_stream.cu, DESIGN.md 3.2)
    auto unit_w = [&](int rb, int ku, int slot) {   // lane 0
      if (p.Wt) bulk_g2s_hint(Wb + uint32_t(slot) * GS_WBYTES, p.Wt + (size_t(rb) * UPR + ku) * GS_WBYTES, GS_WBYTES, Bb + 8u * slot, l2_policy_evict_first());
      else tma_load_2d_hint(Wb + uint32_t(slot) * GS_WBYTES, &tmW, ku * (GS_ROW_BYTES / 4), rb * GS_ROWS, Bb + 8u * slot, l2_policy_evict_first());
    };
    auto unit_params = [&](int rb, int ku, int slot) {   // all 32 lanes: lane = row of the unit
      const uint32_t bar = Bb + 8u * (2 * S + slot);
      if (unit_fast(rb, ku)) {
        const uint32_t raw = RAWb + uint32_t(slot) * GS_RAWBYTES;
        const size_t off = size_t(rb * GS_ROWS + lane) * p.G + ku * GS_STEPS;   // g = 128: group index = step index
        if (p.with_scaling) cp_async16(raw + uint32_t(lane) * 16u, scale16 + off);
        if (p.zmode == 1 || p.zmode == 2) cp_async16(raw + 512u + uint32_t(lane) * 16u, zeros16 + off);
        else if (p.zmode == 3 && lane < GS_STEPS)
          cp_async16(raw + 512u + uint32_t(lane) * 16u, zeros8 + size_t(ku * GS_STEPS + lane) * (p.N >> 1) + rb * (GS_ROWS / 2));
        gs_cp_async_arrive_noinc(bar);
      } else {
        mbar_arrive(bar);   // slow path: the finisher loads the parameters itself
      }
    };
    // weights and group parameters do not depend on the preceding kernel: request the first ring-full before waiting for it
    int q0, ku0, g0;   // the range's first unit
    {
      const int rest = t0 / NG;
      g0 = t0 - rest * NG; q0 = rest / UPR; ku0 = rest - q0 * UPR;
    }
    auto next_unit = [&](int& qq, int& kk, int& gg) {   // t -> t + 1 in (q, ku, g) coordinates: no division per unit
      if (++gg == NG) { gg = 0; if (++kk == UPR) { kk = 0; ++qq; } }
    };
    {
      int qq = q0, kk = ku0, gg = g0;
      for (int u = 0; u < npre; ++u) {
        const int rb = qq * NG + gg;
        if (lane == 0 && rb < p.NRB) { gs_mbar_expect_tx_only(Bb + 8u * u, GS_WBYTES); unit_w(rb, kk, u); }
        unit_params(rb, kk, u);
        next_unit(qq, kk, gg);
      }
    }
    pdl_wait();   // the activations depend on the preceding kernel
    int slot = 0, qq = q0, ku = ku0, gg = g0;
    uint32_t ephase = 1u;   // parity trick: the first pass over the ring finds every slot free
#pragma unroll 1
    for (int i = 0; i < n_units; ++i) {
      const int rb = qq * NG + gg;
      gs_mbar_wait(Bb + 8u * (3 * S + slot), ephase);
      const int k0 = ku * GS_KU;
      const uint32_t abytes = uint32_t(min(GS_KU, p.K - k0)) * 2u;
      if (lane == 0) {
        // (the weight bytes of the first ring-full were registered with the pre-wait request; the padding units past the last
        //  row block -- they exist when NRB % NG != 0 -- carry no weights)
        const bool w_now = i >= npre && rb < p.NRB;
        mbar_arrive_expect_tx(Bb + 8u * slot, abytes + (w_now ? uint32_t(GS_WBYTES) : 0u));
        if (w_now) unit_w(rb, ku, slot);
        gs_bulk_g2s(Ab + uint32_t(slot) * GS_ABYTES, reinterpret_cast<const uint8_t*>(p.A) + size_t(k0) * 2, abytes, Bb + 8u * slot);
      }
      if (i >= npre) unit_params(rb, ku, slot);
      if (++slot == S) { slot = 0; ephase ^= 1u; }
      next_unit(qq, ku, gg);
    }
    return;
  }
  pdl_wait();   // (our stores and workspace traffic must follow the preceding kernel)

  if (warp > NCW) {
    // =========================== finisher warp f: units i = f, f + NF, ... of the range ===========================
    // when the slab has landed: the activation sums of the unit's 8 steps on the tensor cores (A fragment = [ones; the decode
    // magic of element k mod 8], B column g8 = step g8); when the raw parameters have landed: fp32 (c1, c2) pairs [step][row]
    // (lane = row); then the second arrival on full[s]
    const int f = warp - NCW - 1;
    const int g8 = lane >> 2, t4 = lane & 3;
    uint32_t sfrag[4] = {0u, 0u, 0u, 0u};
    {
      const uint32_t one2 = F16 ? 0x3c003c00u : 0x3f803f80u;
      uint32_t pat;
      if (FMT == 1) pat = 0u;                                  // table formats decode to the exact value: nothing to remove
      else if (!HI) pat = MAGIC;                               // (magic, magic)
      else if (IL) pat = (t4 & 1) ? MAGIC_HI : MAGIC;          // elements {2,3,6,7} of a word sit in odd nibbles
      else pat = 0x54006400u;                                  // (even element: 1024, odd element: 64)
      if (g8 == 0) { sfrag[0] = one2; sfrag[2] = one2; }
      if (g8 == 1) { sfrag[0] = pat; sfrag[2] = pat; }
    }
    const uint32_t zsh = 4u * uint32_t(lane & 1);
    int rb, ku, gg, slot = f;
    uint32_t phase = 0u;
    unit_of(t0 + f, rb, ku);   // (one division per kernel; the loop advances the coordinates incrementally)
    gg = (t0 + f) % NG;
#pragma unroll 1
    for (int i = f; i < n_units; i += NF) {
      // ---- activation sums ----
      gs_mbar_wait(Bb + 8u * slot, phase);
      const uint32_t abase = Ab + uint32_t(slot) * GS_ABYTES;
      // column g8 of the B operand = step g8; its 16-k blocks are visited in an order rotated by g8 (bank spread) -- any order
      // is fine as long as (physical k) = (MMA k slot) mod 8, which the magic-pattern row relies on; two independent chains
      uint32_t bf[8][2];
#pragma unroll
      for (int ms = 0; ms < 8; ++ms) {
        const uint32_t a = abase + uint32_t(g8 * 128 + ((ms + g8) & 7) * 16 + 2 * t4) * 2u;
        bf[ms][0] = lds32(a);
        bf[ms][1] = lds32(a + 16u);
      }
      float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int ms = 0; ms < 4; ++ms) {
        mma_16816<T>(c0, sfrag, bf[ms][0], bf[ms][1]);
        mma_16816<T>(c1, sfrag, bf[ms + 4][0], bf[ms + 4][1]);
      }
      if (g8 < 2) {   // row 0: S -> .y, row 1: SM -> .x
        const uint32_t d = Sb + uint32_t(slot) * GS_SBYTES + uint32_t(2 * t4) * 8u + (g8 == 0 ? 4u : 0u);
        gs_sts32f(d, c0[0] + c1[0]);
        gs_sts32f(d + 8u, c0[1] + c1[1]);
      }
      // ---- group parameters -> fp32 (c1, c2) pairs ----
      gs_mbar_wait(Bb + 8u * (2 * S + slot), phase);
      uint32_t sc[8], zc[8];   // raw 16-bit scales; raw fp16 zeros or (quantized) the byte holding this row's zero point
      if (unit_fast(rb, ku)) {
        const uint32_t raw = RAWb + uint32_t(slot) * GS_RAWBYTES;
        const uint4 s4 = lds128(raw + uint32_t(lane) * 16u);
        const uint32_t sw[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
        for (int st = 0; st < 8; ++st) sc[st] = (st & 1) ? (sw[st >> 1] >> 16) : (sw[st >> 1] & 0xffffu);
        if (p.zmode == 3) {
#pragma unroll
          for (int st = 0; st < 8; ++st) zc[st] = gs_lds8(raw + 512u + uint32_t(st) * 16u + uint32_t(lane >> 1));
        } else {
          const uint4 z4 = lds128(raw + 512u + uint32_t(lane) * 16u);
          const uint32_t zw[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
          for (int st = 0; st < 8; ++st) zc[st] = (st & 1) ? (zw[st >> 1] >> 16) : (zw[st >> 1] & 0xffffu);
        }
      } else {
        // slow path (group size != 128, unaligned parameter tensors, N % 32 != 0, a row block's ragged last unit): synchronous loads
        const int n = rb * GS_ROWS + lane;
        const int kstep = ku * GS_STEPS;
        int gi = kstep / p.g128, rem = kstep - gi * p.g128;
#pragma unroll
        for (int st = 0; st < 8; ++st) {
          sc[st] = 0u; zc[st] = 0u;
          if (kstep + st < steps_total && n < p.N) {
            if (p.with_scaling) sc[st] = __ldg(scale16 + size_t(n) * p.G + gi);
            if (p.zmode == 1 || p.zmode == 2) zc[st] = __ldg(zeros16 + size_t(n) * p.G + gi);
            else if (p.zmode == 3) zc[st] = __ldg(zeros8 + size_t(gi) * (p.N >> 1) + (n >> 1));
          }
          if (++rem == p.g128) { rem = 0; ++gi; }
        }
      }
      const uint32_t pbase = Pb + uint32_t(slot) * GS_PBYTES + uint32_t(lane) * 8u;
      // the zero-point mode is hoisted out of the per-step loop (a switch inside it compiles to eight indirect branches)
      auto body = [&](auto zm_tag, auto sc_tag) {
        constexpr int ZM = decltype(zm_tag)::value;
        constexpr bool SC = decltype(sc_tag)::value;
#pragma unroll
        for (int st = 0; st < 8; ++st) {
          const float c1 = SC ? raw_to_float<T>(sc[st]) : 1.f;
          float c2;
          if constexpr (ZM == 0) c2 = -c1 * float(p.zp_const);
          else if constexpr (ZM == 1) c2 = -c1 * raw_to_float<T>(zc[st]);
          else if constexpr (ZM == 2) c2 = -raw_to_float<T>(zc[st]);
          else c2 = -c1 * float((zc[st] >> zsh) & 15u);
          gs_sts64f(pbase + uint32_t(st) * (GS_ROWS * 8u), c1, c2);
        }
      };
      using std::integral_constant;
      if (!p.with_scaling) body(integral_constant<int, 0>{}, std::false_type{});   // (zeros need scaling: gemv_slab_supported)
      else if (p.zmode == 0) body(integral_constant<int, 0>{}, std::true_type{});
      else if (p.zmode == 1) body(integral_constant<int, 1>{}, std::true_type{});
      else if (p.zmode == 2) body(integral_constant<int, 2>{}, std::true_type{});
      else body(integral_constant<int, 3>{}, std::true_type{});
      __syncwarp();
      if (lane == 0) mbar_arrive(Bb + 8u * (S + slot));
      slot += NF;                       // S % NF == 0: the slot sequence of this warp closes on itself
      if (slot >= S) { slot -= S; phase ^= 1u; }
      gg += NF; rb += NF;               // t -> t + NF
      if (gg >= NG) { gg -= NG; rb -= NG; if (++ku == UPR) { ku = 0; rb += NG; } }
    }
    return;
  }

  // =========================== consumer groups ===========================
  // The slab is dense ([32 rows][512 B]): a 128-bit shared load is conflict-free only if the 8 lanes of one phase read 128
  // contiguous bytes of ONE row.  So lane L = 8 i + c loads chunk c (16 B = 32 k) of this warp's 128-byte slice for rows
  // i, 4+i, ..., 28+i.  In mma.sync terms (row slot r = L >> 2 = 2 i + b, t = L & 3) the slots with b = 0 then hold the
  // slice's first 128 k (step 2 ws) and the slots with b = 1 its second 128 k (step 2 ws + 1) OF THE SAME weight rows --
  // different k in one MMA.  That is legal here because m = 1 leaves 7 of the 8 B-operand columns free: column 0 carries the
  // activations of step 2 ws, column 1 those of step 2 ws + 1; slot r's result is valid in column b only (lane (r, t = 0),
  // register c[b]).  The B fragments are loaded once per unit and serve both 16-row tiles.
  const int grp = warp / GS_GW, ws = warp % GS_GW;
  const int li = lane >> 3, lc = lane & 7, lb = lc >> 2, q = lane & 3;
  const uint32_t woff = uint32_t(li) * GS_ROW_BYTES + uint32_t(ws) * GS_SLICE_BYTES + uint32_t(lc) * 16u;   // + 4 x rows per load
  const uint32_t aoff = uint32_t(ws) * 512u + uint32_t(lc) * 64u;     // lanes 0..7: the 32 activations of their own chunk
  const int step_l = 2 * ws + lb;                                        // this lane's 128-k step inside the unit
  const uint32_t poff = uint32_t(step_l * GS_ROWS + li) * 8u;            // (c1, c2) of rows li (+4, +8, ...)
  const uint32_t soff = uint32_t(step_l) * 8u;
  const uint32_t redg = Rb + uint32_t(grp) * GS_RED_GROUP_BYTES;
  const int nsl_last = (Kb - (UPR - 1) * GS_ROW_BYTES) / GS_SLICE_BYTES;   // valid K-slices of a row block's last unit

  Lut4 lut4;
  if constexpr (FMT == 1) lut4_init(lut4, p.w_fmt, !F16, p.lut);
  uint32_t Rv[4][4];   // activations of the lane's chunk (lanes 0..7); other lanes feed unused MMA columns
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) Rv[x][y] = 0u;
  float acc[8];        // rows 16 tl + 4 ph + li and + 8 (pair index pr = 2 tl + ph): this lane's k-half, column lb
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;

  // this group's first unit: the first t >= t0 with t % NG == grp; afterwards t -> t + NG is ku -> ku + 1 (wrapping into the next
  // row block of the group), and -- S % NG == 0 -- the group's slot sequence closes on itself: no division per unit
  int i = (grp - t0 % NG + NG) % NG;
  int rb = 0, ku = 0;
  if (i < n_units) unit_of(t0 + i, rb, ku);
  int slot = i, rbuf = 0;
  uint32_t fphase = 0u;
  bool seg_from0 = false, seg_open = false;
#pragma unroll 1
  for (; i < n_units; i += NG) {
    if (!seg_open) { seg_from0 = (ku == 0); seg_open = true; }
    const bool closes = (ku == UPR - 1);
    gs_mbar_wait(Bb + 8u * slot, fphase);   // weights + activations have landed
    // (p.UPR > 0 always holds; the run-time term keeps ptxas's register allocation of the fp16 compressed-word instance: without it
    //  that instance spills 38 / 64 B instead of 16 / 24 B, partly inside this loop, and runs 3-5 % slower on an H100.  Which term
    //  does it depends on the rest of the kernel: since the weight copies carry an L2 policy, p.N > 0 no longer does, p.UPR > 0 does)
    const bool active = (!closes || ws < nsl_last) && rb < p.NRB && p.UPR > 0;
    float cc[4][4];
    if (active) {
      const uint32_t wst = Wb + uint32_t(slot) * GS_WBYTES + woff;
      uint4 wv[8];
#pragma unroll
      for (int x = 0; x < 8; ++x) wv[x] = lds128(wst + uint32_t(x) * (4u * GS_ROW_BYTES));
      if (lane < 8) {   // one divergent region per unit
        const uint32_t ast = Ab + uint32_t(slot) * GS_ABYTES + aoff;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const uint4 v = lds128(ast + uint32_t(x) * 16u);
          Rv[x][0] = v.x; Rv[x][1] = v.y; Rv[x][2] = v.z; Rv[x][3] = v.w;
        }
      }
      __syncwarp();
      auto decode_pair = [&](uint32_t xw, uint32_t yw, uint32_t (&ha)[4], uint32_t (&hb)[4]) {
        if constexpr (FMT == 1) {
          lut4_decode8(xw, lut4, ha);      // natural pairs (e0,e1) .. (e6,e7): the activation registers pair up as stored
          lut4_decode8(yw, lut4, hb);
        } else if constexpr (HI) {
          const uint32_t xa = xw, ya = xw >> 8, xb = yw, yb = yw >> 8;
          ha[0] = lop3_and_or(xa, 0x000f000fu, MAGIC); ha[1] = lop3_and_or(xa, 0x00f000f0u, MAGIC_HI);
          ha[2] = lop3_and_or(ya, 0x000f000fu, MAGIC); ha[3] = lop3_and_or(ya, 0x00f000f0u, MAGIC_HI);
          hb[0] = lop3_and_or(xb, 0x000f000fu, MAGIC); hb[1] = lop3_and_or(xb, 0x00f000f0u, MAGIC_HI);
          hb[2] = lop3_and_or(yb, 0x000f000fu, MAGIC); hb[3] = lop3_and_or(yb, 0x00f000f0u, MAGIC_HI);
        } else {
          decode_u4x8_raw<T>(xw, ha);
          decode_u4x8_raw<T>(yw, hb);
        }
      };
      auto word_of = [&](int idx, int wi) -> uint32_t {
        return wi == 0 ? wv[idx].x : (wi == 1 ? wv[idx].y : (wi == 2 ? wv[idx].z : wv[idx].w));
      };
      auto mma_pair = [&](float (&c)[4], const uint32_t (&ha)[4], const uint32_t (&hb)[4], int wi) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const uint32_t af[4] = {ha[2 * jj], hb[2 * jj], ha[2 * jj + 1], hb[2 * jj + 1]};
          uint32_t b0, b1;
          if constexpr (IL || FMT == 1) {
            b0 = Rv[wi][2 * jj]; b1 = Rv[wi][2 * jj + 1];
          } else {
            b0 = __byte_perm(Rv[wi][jj], Rv[wi][jj + 2], 0x5410);
            b1 = __byte_perm(Rv[wi][jj], Rv[wi][jj + 2], 0x7632);
          }
          mma_16816<T>(c, af, b0, b1);
        }
      };
#pragma unroll
      for (int pr = 0; pr < 4; ++pr)
#pragma unroll
        for (int j = 0; j < 4; ++j) cc[pr][j] = 0.f;
      // fragment rows r <- weight row 16 tl + 4 ph + li, rows r + 8 <- that row + 8   (pr = 2 tl + ph)
#pragma unroll
      for (int pr = 0; pr < 4; ++pr) {
        const int ia = 4 * (pr >> 1) + (pr & 1);
#pragma unroll
        for (int wi = 0; wi < 4; ++wi) {
          uint32_t ha[4], hb[4];
          decode_pair(word_of(ia, wi), word_of(ia + 2, wi), ha, hb);
          mma_pair(cc[pr], ha, hb, wi);
        }
      }
    }
    // the group parameters and activation sums are needed only now: the finisher works on THIS unit while we decode it, so its
    // latency is off the critical path (with everything behind one barrier the consumers would wait for the slowest part of the
    // feed)
    gs_mbar_wait(Bb + 8u * (S + slot), fphase);
    if (active) {
      const uint32_t pst = Pb + uint32_t(slot) * GS_PBYTES + poff;
      const float2 su = gs_lds64f(Sb + uint32_t(slot) * GS_SBYTES + soff);
#pragma unroll
      for (int pr = 0; pr < 4; ++pr) {
        const int tl = pr >> 1, ph = pr & 1;
        const float2 pa = gs_lds64f(pst + uint32_t(16 * tl + 4 * ph) * 8u);
        const float2 pb = gs_lds64f(pst + uint32_t(16 * tl + 4 * ph + 8) * 8u);
        const float va = lb ? cc[pr][1] : cc[pr][0], vb = lb ? cc[pr][3] : cc[pr][2];   // column lb of fragment rows r / r + 8 (valid in lanes t = 0)
        acc[2 * pr] = fmaf(pa.x, va - su.x, acc[2 * pr]);
        acc[2 * pr] = fmaf(pa.y, su.y, acc[2 * pr]);
        acc[2 * pr + 1] = fmaf(pb.x, vb - su.x, acc[2 * pr + 1]);
        acc[2 * pr + 1] = fmaf(pb.y, su.y, acc[2 * pr + 1]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(Bb + 8u * (3 * S + slot));

    if (closes || i + NG >= n_units) {
      // ---- end of this range's segment of row block rb: group reduction over 4 K-slices x 2 k-halves, then store / park / collect ----
      const uint32_t rbase = redg + uint32_t(rbuf) * (2 * GS_GW * GS_ROWS * 4);
      if (q == 0) {
        const uint32_t rw = rbase + uint32_t(2 * ws + lb) * (GS_ROWS * 4u) + uint32_t(li) * 4u;
#pragma unroll
        for (int pr = 0; pr < 4; ++pr) {
          gs_sts32f(rw + uint32_t(16 * (pr >> 1) + 4 * (pr & 1)) * 4u, acc[2 * pr]);
          gs_sts32f(rw + uint32_t(16 * (pr >> 1) + 4 * (pr & 1) + 8) * 4u, acc[2 * pr + 1]);
        }
      }
      asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(GS_GW * 32) : "memory");
      if (ws == 0) {
        const int row = lane;
        const int n = rb * GS_ROWS + row;
        float v = 0.f;
#pragma unroll
        for (int ww = 0; ww < 2 * GS_GW; ++ww) v += gs_lds32f(rbase + uint32_t(ww) * (GS_ROWS * 4u) + uint32_t(row) * 4u);
        unsigned long long* myslot = p.ws + (size_t(ri) * NG + grp) * GS_ROWS + row;
        if (!seg_from0) {
          // contribution to a row block owned by a later range (only the first segment of a group's range can be one)
          const unsigned long long pk = (static_cast<unsigned long long>(p.nonce) << 32) | __float_as_uint(v);
          asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(myslot), "l"(pk) : "memory");
        } else {
          if (!closes) {
            // this range owns the block but does not reach its end: add the parked sums of the ranges that cover the rest.
            // the block's last unit is t_last; range rj contributes iff it holds a unit of this row block
            const int t_first = (t0 + i) - ku * NG;                 // the block's unit with ku = 0
            const int t_last = t_first + (UPR - 1) * NG;
            for (int rj = ri + 1; rj < R; ++rj) {
              const int bj = gs_range_begin(rj, p.T, R), ej = gs_range_begin(rj + 1, p.T, R);
              if (bj > t_last) break;
              // first unit of this row block (t = t_first mod NG) inside [bj, ej)
              const int tf = bj + ((t_first - bj) % NG + NG) % NG;
              if (tf >= ej || tf > t_last) { if (ej > t_last) break; continue; }
              unsigned long long* sl = p.ws + (size_t(rj) * NG + grp) * GS_ROWS + row;
              unsigned long long pk;
              do {
                asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(pk) : "l"(sl) : "memory");
              } while (static_cast<unsigned int>(pk >> 32) != p.nonce);
              v += __uint_as_float(static_cast<unsigned int>(pk));
              asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(sl), "l"(0ull) : "memory");
              if (ej > t_last) break;
            }
          }
          if constexpr (SWIGLU) {
            // lane l holds row rb * 32 + l: the gate rows of the block's two 16-row halves are lanes 0-7 and 16-23, their up rows
            // the lanes 8 above.  The whole warp takes this branch (seg_from0 and closes are uniform over the group), so all 32
            // lanes join the shuffle; a gate row below N has its up row below N too (N % 16 == 0)
            const float vu = __shfl_down_sync(0xffffffffu, v, 8);
            if ((lane & 8) == 0 && n < p.N) gs_store_swiglu<T>(p, n, rb * 16 + 8 * (lane >> 4) + (lane & 7), v, vu);
          } else {
            if (n < p.N) gs_store<T>(p, n, v);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      rbuf ^= 1;
      seg_open = false;
    }
    slot += NG;
    if (slot >= S) { slot -= S; fphase ^= 1u; }
    if (++ku == UPR) { ku = 0; rb += NG; }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// a tensor map is a pure function of (device pointer, N, K): cached, so a steady-state launch makes no driver call
struct MapEntry { const void* W; int N, K; CUtensorMap map; unsigned long long stamp; };
constexpr int GS_MAP_CACHE = 256;
std::mutex g_map_mu;
MapEntry g_maps[GS_MAP_CACHE];
int g_map_count = 0;
unsigned long long g_map_clock = 0;

bool get_w_map(CUtensorMap* tm, const void* W, int N, int K) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  ++g_map_clock;
  for (int i = 0; i < g_map_count; ++i)
    if (g_maps[i].W == W && g_maps[i].N == N && g_maps[i].K == K) { g_maps[i].stamp = g_map_clock; *tm = g_maps[i].map; return true; }
  CUtensorMap m;
  const uint64_t Kb = uint64_t(K) / 2;
  if (make_map_2d(&m, CU_TENSOR_MAP_DATA_TYPE_UINT32, W, Kb / 4, uint64_t(N), Kb, GS_ROW_BYTES / 4, GS_ROWS,
                  CU_TENSOR_MAP_SWIZZLE_NONE))
    return false;
  int idx = g_map_count;
  if (g_map_count < GS_MAP_CACHE) ++g_map_count;
  else {
    idx = 0;
    for (int i = 1; i < GS_MAP_CACHE; ++i) if (g_maps[i].stamp < g_maps[idx].stamp) idx = i;
  }
  g_maps[idx] = MapEntry{W, N, K, m, g_map_clock};
  *tm = m;
  return true;
}


template <typename T, bool IL, int FMT, bool SWIGLU>
int launch_slab_inst(const MatmulArgs& a, const CUtensorMap& tm, const SlabParams& p) {
  auto kernel = gemv_slab_kernel<T, IL, FMT, SWIGLU>;
  static KernelCache<> cache;
  const int occ = kernel_setup(cache, kernel, kSmemOptinMax, GS_THREADS, GS_SMEM_BYTES);
  if (occ < 1) { set_error("gemv_slab: kernel does not fit on this device"); return 4; }
  const int grid = std::max(1, std::min(p.T, std::min(occ, GS_MINB) * device_sm_count()));
  return launch_pdl(kernel, grid, GS_THREADS, GS_SMEM_BYTES, a.stream, pdl_enabled(), tm, p);
}
template <typename T, bool IL, int FMT>
int launch_slab(const MatmulArgs& a, const CUtensorMap& tm, const SlabParams& p) {
  return a.form == MatmulForm::SwiGLU ? launch_slab_inst<T, IL, FMT, true>(a, tm, p) : launch_slab_inst<T, IL, FMT, false>(a, tm, p);
}

}  // namespace

// tagged exchange slots: [CTAs][consumer groups][32 rows], at most GS_MINB CTAs per SM
size_t gemv_slab_slot_bytes(int sms) { return size_t(GS_MINB * GS_NG) * size_t(sms) * GS_ROWS * 8 + 256; }
size_t gemv_slab_workspace_bytes() { return gemv_slab_slot_bytes(device_sm_count()); }

bool gemv_slab_supported(const bb_matmul_desc& d, int m) {
  if (m != 1) return false;
  if (d.a_dtype != BB_F16 && d.a_dtype != BB_BF16) return false;
  const bool table_fmt = d.w_fmt == BB_W_NF || d.w_fmt == BB_W_FP4;
  if (table_fmt) {   // NF4 / fp4: compressed storage, scale only
    if (d.w_layout != BB_LAYOUT_COMPRESSED || d.with_zeros) return false;
  } else if (d.w_fmt != BB_W_UINT && d.w_fmt != BB_W_INT) {
    return false;
  }
  if (d.w_bits != 4) return false;
  if (d.w_layout == BB_LAYOUT_INTERLEAVED_8) return false;
  if (d.N % 16 || d.K % 256) return false;
  if (d.w_tile == BB_TILE_SLAB && (d.N % GS_ROWS || d.K % GS_KU)) return false;   // whole units only
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if (g % 128 || d.K % g) return false;
  if (d.with_zeros && !d.with_scaling) return false;
  if (d.w_fmt == BB_W_INT && d.with_zeros) return false;
  if (d.out_dtype != BB_F16 && d.out_dtype != BB_BF16 && d.out_dtype != BB_F32) return false;
  if (d.with_zeros && d.zeros_mode == BB_ZEROS_QUANTIZED && (d.N % 2)) return false;
  if ((long long)((d.N + GS_ROWS - 1) / GS_ROWS + 4) * ((d.K + GS_KU - 1) / GS_KU) >= (1ll << 30)) return false;
  return true;   // (a missing cuTensorMapEncodeTiled entry point is reported loudly at launch, not hidden behind a fallback)
}

int launch_gemv_slab(const MatmulArgs& a) {
  const bb_matmul_desc& d = a.d;
  if ((reinterpret_cast<uintptr_t>(a.A) & 15) || (reinterpret_cast<uintptr_t>(a.W) & 15)) {
    set_error("gemv_slab: A and W must be 16-byte aligned (TMA)");
    return 5;
  }
  if (!a.workspace || a.workspace_bytes < gemv_slab_workspace_bytes()) {
    set_error("gemv_slab needs a zero-initialised workspace of %zu bytes (bb_workspace_bytes)", gemv_slab_workspace_bytes());
    return 5;
  }
  SlabParams p;
  p.A = a.A; p.scale = d.with_scaling ? a.scale : nullptr; p.zeros = d.with_zeros ? a.zeros : nullptr;
  p.bias = d.with_bias ? a.bias : nullptr; p.out = make_outspec(a);
  p.N = d.N; p.K = d.K; p.G = a.groups(); p.g128 = a.gsize() / 128;
  p.with_scaling = d.with_scaling;
  p.zmode = d.with_zeros ? (d.zeros_mode + 1) : 0;
  p.zp_const = (d.w_fmt == BB_W_INT) ? (1 << (d.w_bits - 1)) : 0;
  p.out_dtype = d.out_dtype;
  p.UPR = (d.K + GS_KU - 1) / GS_KU;
  p.NRB = (d.N + GS_ROWS - 1) / GS_ROWS;
  p.T = ((p.NRB + GS_NG - 1) / GS_NG) * p.UPR * GS_NG;
  p.lut = d.w_fmt == BB_W_NF ? a.lut : nullptr;
  p.w_fmt = d.w_fmt;
  CUtensorMap tm;
  p.Wt = nullptr;
  if (d.w_tile == BB_TILE_SLAB) {
    // slab-tiled storage: a unit is one contiguous 16 KB block -- a single bulk copy, no tensor map
    p.Wt = reinterpret_cast<const uint8_t*>(a.W);
    memset(&tm, 0, sizeof(tm));
  } else if (!get_w_map(&tm, a.W, d.N, d.K)) { set_error("gemv_slab: cuTensorMapEncodeTiled failed"); return 4; }
  p.fast_params = (p.g128 == 1 && (p.G & 7) == 0 && (d.N % GS_ROWS) == 0 &&
                   (!d.with_scaling || (reinterpret_cast<uintptr_t>(a.scale) & 15) == 0) &&
                   (!d.with_zeros || (reinterpret_cast<uintptr_t>(a.zeros) & 15) == 0)) ? 1 : 0;
  p.ws = reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(a.workspace) + 15) & ~uintptr_t(15));
  static std::atomic<unsigned int> counter{0x9e3779b9u};
  unsigned int nz = counter.fetch_add(0x9e3779b9u);
  p.nonce = nz | 1u;
  const bool il = d.w_layout == BB_LAYOUT_INTERLEAVED_16;
  const bool f16 = d.a_dtype == BB_F16;
  if (d.w_fmt == BB_W_NF || d.w_fmt == BB_W_FP4)   // table formats: compressed storage only
    return f16 ? launch_slab<__half, false, 1>(a, tm, p) : launch_slab<__nv_bfloat16, false, 1>(a, tm, p);
  if (f16) return il ? launch_slab<__half, true, 0>(a, tm, p) : launch_slab<__half, false, 0>(a, tm, p);
  return il ? launch_slab<__nv_bfloat16, true, 0>(a, tm, p) : launch_slab<__nv_bfloat16, false, 0>(a, tm, p);
}

}  // namespace bb
