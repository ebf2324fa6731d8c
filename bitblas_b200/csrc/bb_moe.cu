// bb_moe.cu -- the two ends of a mixture-of-experts expert block around the grouped matmuls (bb_moe_route, bb_moe_combine), and
// the top-k gating that produces the block's router output (bb_moe_topk).
//
// Routing (moe_route_kernel): slot s = t * k + j of a [T, k] top-k id table goes to expert ids[s]; rows are sorted by expert and,
// within an expert, by slot, so the order is stable and independent of the grid.  One persistent launch, no workspace:
//   * every CTA owns a contiguous slot range [s0, s1) and histograms ALL n = T * k ids in shared memory (E <= 256 counters; warp
//     aggregation with match.any keeps a routing that sends every slot to one expert from serialising on one shared atomic).  It
//     counts the ids before s0 separately, so it knows each expert's first sorted row and how many of its rows precede the range.
//   * it then walks its range in chunks of one slot per thread: match.any ranks the slots of an expert inside a warp, per-warp
//     counts in shared memory rank them across the warps of the chunk, and a running count per expert carries on to the next
//     chunk.  The chunk's rows of x are copied with 16-byte vectors.
//   * ids outside [0, E) are dropped (slot_rows[s] = -1); sorted rows offsets[E] .. n - 1 are not written.
//   * PDL: griddepcontrol.wait before the first read of ids and x; launch_dependents after the copy.
//   * INDEX instance (bb_moe_route_index): the same offsets and slot_rows, but instead of copying x it writes the token of each
//     sorted row, row_token[slot_rows[s]] = s / k, which the gathering grouped GEMM reads its A rows through.
//
// Combine (moe_combine_kernel): out[t, :] = sum_j w[t, j] * Y[slot_rows[t * k + j], :], accumulated in fp32 in j order and rounded
// once; slots whose row is outside [0, T * k) add nothing.  One thread per 8 output elements, no atomics: deterministic.
//
// Top-k gating (moe_topk_kernel): router logits [T, E] -> the [T, k] ids and fp32 weights routing and combine read.  One warp per
// token, lane l holding the scores of experts l, l + 32, ... (E <= 256: 8 per lane) in registers; softmax or sigmoid scores, the
// optional selection bias, the optional group limit (one lane per group over the warp's values in shared memory), then k rounds
// of warp arg-max, each removing its winner.  Ties go to the lower expert index and a NaN ranks below every number, so the ids,
// their order and the weights are a function of the logits alone.  PDL: griddepcontrol.wait before the first read,
// launch_dependents after the stores.
#include <algorithm>
#include <climits>
#include <type_traits>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int ROUTE_THREADS = 256;
constexpr int ROUTE_WARPS = ROUTE_THREADS / 32;
constexpr int ROUTE_MIN_SLOTS = 8;   // slots per CTA below which more CTAs only repeat the histogram
constexpr int ROUTE_CTAS_PER_SM = 2;  // every CTA reads all T * k ids: more CTAs than this per SM cost more than their copy gains

struct RouteParams {
  const int32_t* ids;
  const uint4* x;       // [T, K / 8] 16-byte vectors
  int32_t* offsets;     // [E + 1]
  int32_t* slot_rows;   // [n]
  uint4* x_sorted;      // [n, K / 8]
  int n, k, E, vecs;    // slots, top-k, experts, 16-byte vectors per row
  int32_t* row_token;   // [n] (INDEX)
};

__device__ __forceinline__ int route_expert(const RouteParams& r, long long s) {
  if (s >= r.n) return -1;
  const int e = r.ids[s];
  return (e >= 0 && e < r.E) ? e : -1;
}

template <bool INDEX>
__global__ void __launch_bounds__(ROUTE_THREADS) moe_route_kernel(const RouteParams r) {
  __shared__ int cnt_s[BB_GROUPED_MAX_GROUPS];      // slots of each expert (all n)
  __shared__ int run_s[BB_GROUPED_MAX_GROUPS];      // first sorted row of each expert's next slot in this CTA
  __shared__ int warp_s[ROUTE_WARPS][BB_GROUPED_MAX_GROUPS];   // slots of each expert per warp of the current chunk
  __shared__ int dst_s[ROUTE_THREADS];              // sorted row of each slot of the chunk (-1: dropped)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt = (1u << lane) - 1u;
  int s0, s1;
  {
    const int base = r.n / gridDim.x, rem = r.n % gridDim.x, b = blockIdx.x;
    s0 = b * base + min(b, rem);
    s1 = s0 + base + (b < rem ? 1 : 0);
  }
  for (int e = tid; e < BB_GROUPED_MAX_GROUPS; e += ROUTE_THREADS) {
    cnt_s[e] = 0;
    run_s[e] = 0;
    for (int w = 0; w < ROUTE_WARPS; ++w) warp_s[w][e] = 0;
  }
  __syncthreads();
  pdl_wait();   // ids and x are the preceding kernels' output

  // histogram: all slots into cnt_s, the slots before s0 into run_s
  for (long long base = 0; base < r.n; base += ROUTE_THREADS) {
    const long long s = base + tid;
    const int e = route_expert(r, s);
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    if (e >= 0 && (peers & lt) == 0) atomicAdd(&cnt_s[e], __popc(peers));
    if (base < s0) {
      const int eb = s < s0 ? e : -1;
      const unsigned pb = __match_any_sync(0xffffffffu, eb);
      if (eb >= 0 && (pb & lt) == 0) atomicAdd(&run_s[eb], __popc(pb));
    }
  }
  __syncthreads();
  // exclusive prefix sum of the counts by warp 0 (8 consecutive experts per lane): offsets, and run_s += each expert's start
  if (warp == 0) {
    constexpr int PER = BB_GROUPED_MAX_GROUPS / 32;
    int c[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = lane * PER + i;
      c[i] = e < r.E ? cnt_s[e] : 0;
      sum += c[i];
    }
    int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    int start = incl - sum;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = lane * PER + i;
      if (e < r.E) {
        if (blockIdx.x == 0) r.offsets[e] = start;
        run_s[e] += start;
      }
      start += c[i];
    }
    if (blockIdx.x == 0 && lane == 31) r.offsets[r.E] = incl;
  }
  __syncthreads();

  for (long long c0 = s0; c0 < s1; c0 += ROUTE_THREADS) {
    const long long s = c0 + tid;
    const int e = s < s1 ? route_expert(r, s) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    const bool leader = e >= 0 && (peers & lt) == 0;
    if (leader) warp_s[warp][e] = __popc(peers);
    __syncthreads();
    int row = -1;
    if (e >= 0) {
      row = run_s[e] + __popc(peers & lt);
      for (int w = 0; w < warp; ++w) row += warp_s[w][e];
    }
    if (s < s1) r.slot_rows[s] = row;
    if constexpr (INDEX) {
      if (row >= 0) r.row_token[row] = int(s / r.k);
    } else {
      dst_s[tid] = row;
    }
    __syncthreads();
    if (leader) {
      atomicAdd(&run_s[e], __popc(peers));
      warp_s[warp][e] = 0;
    }
    if constexpr (!INDEX) {
      // copy the chunk's rows: x[s / k] -> x_sorted[row]
      const int len = int(min((long long)ROUTE_THREADS, s1 - c0));
      const long long total = (long long)len * r.vecs;
      for (long long idx = tid; idx < total; idx += ROUTE_THREADS) {
        const int i = int(idx / r.vecs), v = int(idx - (long long)i * r.vecs);
        const int dst = dst_s[i];
        if (dst >= 0) r.x_sorted[size_t(dst) * r.vecs + v] = r.x[size_t((c0 + i) / r.k) * r.vecs + v];
      }
    }
    __syncthreads();   // run_s, warp_s and dst_s are final for the next chunk
  }
  pdl_launch_dependents();
}

struct CombineParams {
  const int32_t* slot_rows;   // [T * k]
  const float* w;             // [T * k]
  const void* Y;              // [T * k, N]
  void* out;                  // [T, N]
  int k, cols8;               // top-k, N / 8
  long long T, n;             // tokens, slots = T * k
  int out_dtype;
};

template <typename OT>
__device__ __forceinline__ void load8(const void* base, size_t elem, float (&v)[8]) {
  if constexpr (std::is_same<OT, float>::value) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem);
    const float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const OT*>(base) + elem);
    const OT* h = reinterpret_cast<const OT*>(&q);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = TypeTraits<OT>::to_float(h[i]);
  }
}

template <typename OT>
__device__ __forceinline__ void store8(void* base, size_t elem, const float (&v)[8]) {
  if constexpr (std::is_same<OT, float>::value) {
    float4* p = reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem);
    p[0] = make_float4(v[0], v[1], v[2], v[3]);
    p[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint4 q;
    OT* h = reinterpret_cast<OT*>(&q);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = TypeTraits<OT>::from_float(v[i]);
    *reinterpret_cast<uint4*>(reinterpret_cast<OT*>(base) + elem) = q;
  }
}

template <typename OT>
__global__ void __launch_bounds__(256) moe_combine_kernel(const CombineParams c) {
  pdl_wait();   // Y is the preceding kernel's output
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < c.T * c.cols8) {
    const long long t = idx / c.cols8;
    const int col = int(idx - t * c.cols8) * 8;
    const size_t N = size_t(c.cols8) * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < c.k; ++j) {
      const long long s = t * c.k + j;
      const int row = c.slot_rows[s];
      if (row < 0 || row >= c.n) continue;
      const float w = c.w[s];
      float y[8];
      load8<OT>(c.Y, size_t(row) * N + col, y);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(w, y[i], acc[i]);
    }
    store8<OT>(c.out, size_t(t) * N + col, acc);
  }
  pdl_launch_dependents();
}

constexpr int TOPK_WARPS = 4;                                  // tokens per CTA
constexpr int TOPK_PER_LANE = BB_GROUPED_MAX_GROUPS / 32;      // experts per lane

struct TopkParams {
  const void* logits;   // [T, E]
  const float* bias;    // [E] or null
  int32_t* ids;         // [T, k]
  float* weights;       // [T, k]
  int T, E, k;
  bool sigmoid, top2, renormalize;
  int groups, topk_group;   // groups <= 1: no group limit
  float scale;
};

// (a, ia) ranks before (b, ib): the larger value first, a NaN below every number, ties to the lower index
__device__ __forceinline__ bool topk_before(float a, int ia, float b, int ib) {
  if (isnan(a)) return isnan(b) && ia < ib;
  if (isnan(b)) return true;
  return a > b || (a == b && ia < ib);
}

template <typename LT>
__device__ __forceinline__ float logit_to_float(LT v) {
  if constexpr (std::is_same<LT, float>::value) return v;
  else return TypeTraits<LT>::to_float(v);
}

template <typename LT>
__global__ void __launch_bounds__(TOPK_WARPS * 32) moe_topk_kernel(const TopkParams p) {
  __shared__ float v_s[TOPK_WARPS][BB_GROUPED_MAX_GROUPS];   // selection values of each warp's token (group limit only)
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long t = (long long)blockIdx.x * TOPK_WARPS + warp;
  pdl_wait();   // the logits are the preceding kernel's output
  if (t < p.T) {
    const LT* row = reinterpret_cast<const LT*>(p.logits) + size_t(t) * p.E;
    float s[TOPK_PER_LANE], v[TOPK_PER_LANE];
    unsigned live = 0;   // bit i: expert lane + 32 i exists and can still be chosen
#pragma unroll
    for (int i = 0; i < TOPK_PER_LANE; ++i) {
      const int e = lane + 32 * i;
      s[i] = 0.f;
      if (e < p.E) {
        s[i] = logit_to_float(row[e]);
        live |= 1u << i;
      }
    }
    if (p.sigmoid) {
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i) s[i] = 1.f / (1.f + expf(-s[i]));
    } else {
      // softmax over the experts; NaN logits stay NaN and add nothing to the max or the sum.  The xor butterflies give every lane
      // the same bits (fmaxf and + are commutative).
      float m = -INFINITY;
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i)
        if ((live >> i) & 1) m = fmaxf(m, s[i]);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, d));
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i) {
        if (((live >> i) & 1) && !isnan(s[i])) {
          s[i] = expf(s[i] - m);
          sum += s[i];
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(FULL, sum, d);
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i) s[i] = s[i] / sum;
    }
#pragma unroll
    for (int i = 0; i < TOPK_PER_LANE; ++i) {
      const int e = lane + 32 * i;
      v[i] = (p.bias && e < p.E) ? s[i] + p.bias[e] : s[i];
    }

    if (p.groups > 1) {
      // lane g scores group g (experts [g * gs, (g + 1) * gs)) from shared memory, ranks it against the other groups, and the
      // experts of groups outside the topk_group best leave `live`
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i)
        if (lane + 32 * i < p.E) v_s[warp][lane + 32 * i] = v[i];
      __syncwarp();
      const int gs = p.E / p.groups;
      float score = __int_as_float(0x7fffffff);
      if (lane < p.groups) {
        float b1 = __int_as_float(0x7fffffff), b2 = b1;   // the two best values of the group
        int i1 = INT_MAX, i2 = INT_MAX;
        // lane g starts at offset g % gs of its group and wraps around, so that with gs a multiple of 32 the lanes read 32
        // different banks; the two best are the same in any scan order (topk_before is a strict total order)
        const int e0 = lane * gs, e1 = e0 + gs;
        int e = e0 + lane % gs;
        for (int n = 0; n < gs; ++n, e = e + 1 == e1 ? e0 : e + 1) {
          const float x = v_s[warp][e];
          if (topk_before(x, e, b1, i1)) {
            b2 = b1; i2 = i1; b1 = x; i1 = e;
          } else if (topk_before(x, e, b2, i2)) {
            b2 = x; i2 = e;
          }
        }
        score = p.top2 ? b1 + b2 : b1;
      }
      int rank = 0;
      for (int g = 0; g < p.groups; ++g) {
        const float o = __shfl_sync(FULL, score, g);
        if (topk_before(o, g, score, lane)) ++rank;
      }
      const unsigned kept = __ballot_sync(FULL, lane < p.groups && rank < p.topk_group);
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i) {
        const int e = lane + 32 * i;
        if (e < p.E && !((kept >> (e / gs)) & 1)) live &= ~(1u << i);
      }
    }

    // k rounds of warp arg-max; lane j keeps the j-th choice.  The weights' sum runs in j order.
    int my_id = 0;
    float my_w = 0.f, wsum = 0.f;
    for (int j = 0; j < p.k; ++j) {
      float bv = __int_as_float(0x7fffffff);
      int bi = INT_MAX;
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i) {
        if (((live >> i) & 1) && topk_before(v[i], lane + 32 * i, bv, bi)) {
          bv = v[i];
          bi = lane + 32 * i;
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {   // topk_before is a strict total order: every lane ends with the same winner
        const float ov = __shfl_xor_sync(FULL, bv, d);
        const int oi = __shfl_xor_sync(FULL, bi, d);
        if (topk_before(ov, oi, bv, bi)) {
          bv = ov;
          bi = oi;
        }
      }
      // the validated k leaves a live expert for every round, so bi < E
      const int owner = bi & 31, slot = bi >> 5;
      float mine = 0.f;
#pragma unroll
      for (int i = 0; i < TOPK_PER_LANE; ++i)
        if (i == slot) mine = s[i];
      if (lane == owner) live &= ~(1u << slot);
      const float w = __shfl_sync(FULL, mine, owner);
      wsum += w;
      if (lane == j) {
        my_id = bi;
        my_w = w;
      }
    }
    if (lane < p.k) {
      float w = my_w;
      if (p.renormalize) w = wsum != 0.f ? w / wsum : 0.f;
      const size_t o = size_t(t) * p.k + lane;
      p.ids[o] = my_id;
      p.weights[o] = w * p.scale;
    }
  }
  pdl_launch_dependents();
}

}  // namespace

// x_sorted == nullptr: the INDEX instance, which writes row_token instead of copying x
int launch_moe_route(const int32_t* topk_ids, int n_slots, int top_k, int num_experts, const void* x, int K, int32_t* offsets,
                     int32_t* slot_rows, void* x_sorted, int32_t* row_token, cudaStream_t stream) {
  const bool index = x_sorted == nullptr;
  auto kernel = index ? moe_route_kernel<true> : moe_route_kernel<false>;
  static KernelCache<> cache[2];   // [index]
  const int occ = kernel_setup(cache[index], kernel, 0, ROUTE_THREADS);
  if (occ <= 0) { set_error("moe route: the kernel cannot be resident on this device"); return 2; }
  RouteParams r;
  r.ids = topk_ids; r.x = reinterpret_cast<const uint4*>(x); r.offsets = offsets; r.slot_rows = slot_rows;
  r.x_sorted = reinterpret_cast<uint4*>(x_sorted); r.n = n_slots; r.k = top_k; r.E = num_experts; r.vecs = K / 8;
  r.row_token = row_token;
  const int resident = std::min(occ, ROUTE_CTAS_PER_SM) * device_sm_count();
  const int grid = std::max(1, std::min((n_slots + ROUTE_MIN_SLOTS - 1) / ROUTE_MIN_SLOTS, resident));
  return launch_pdl(kernel, grid, ROUTE_THREADS, 0, stream, pdl_enabled(), r);
}

int launch_moe_combine(const int32_t* slot_rows, const float* topk_weights, const void* Y, int out_dtype, void* out,
                       int num_tokens, int top_k, int N, cudaStream_t stream) {
  CombineParams c;
  c.slot_rows = slot_rows; c.w = topk_weights; c.Y = Y; c.out = out; c.k = top_k; c.cols8 = N / 8;
  c.T = num_tokens; c.n = (long long)num_tokens * top_k; c.out_dtype = out_dtype;
  const long long threads = c.T * c.cols8;
  auto kernel = out_dtype == BB_F16 ? moe_combine_kernel<__half>
                                    : (out_dtype == BB_BF16 ? moe_combine_kernel<__nv_bfloat16> : moe_combine_kernel<float>);
  return launch_pdl(kernel, unsigned((threads + 255) / 256), 256, 0, stream, pdl_enabled(), c);
}

int launch_moe_topk(const void* logits, int logits_dtype, int num_tokens, int num_experts, int top_k, int scoring,
                    const float* correction_bias, int num_expert_group, int topk_group, int group_score, int renormalize,
                    float routed_scaling_factor, int32_t* topk_ids, float* topk_weights, cudaStream_t stream) {
  TopkParams p;
  p.logits = logits; p.bias = correction_bias; p.ids = topk_ids; p.weights = topk_weights;
  p.T = num_tokens; p.E = num_experts; p.k = top_k;
  p.sigmoid = scoring == 1; p.top2 = group_score == 1; p.renormalize = renormalize != 0;
  p.groups = num_expert_group > 1 ? num_expert_group : 1; p.topk_group = topk_group;
  p.scale = routed_scaling_factor;
  auto kernel = logits_dtype == BB_F16 ? moe_topk_kernel<__half>
                                       : (logits_dtype == BB_BF16 ? moe_topk_kernel<__nv_bfloat16> : moe_topk_kernel<float>);
  return launch_pdl(kernel, unsigned((num_tokens + TOPK_WARPS - 1) / TOPK_WARPS), TOPK_WARPS * 32, 0, stream, pdl_enabled(), p);
}

}  // namespace bb
