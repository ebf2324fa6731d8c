// bb_grouped.cu -- grouped low-bit matmul for mixture-of-experts layers (bb_matmul_grouped): ONE launch over E experts,
//   C[offsets[e] : offsets[e+1]] = A[offsets[e] : offsets[e+1]] x dequant(W[e])^T (+ bias[e])     for every e,
// with the row offsets read on the device.
//
// Design:
//   * the per-expert arithmetic is the decode GEMV's (gemv_mma_tile, bb_gemv_mma.cuh): LOP3 decode into mma.sync fragments,
//     per-group scale / zero corrections, K split over the warps of a CTA and reduced in shared memory.  Numerics are those of
//     bb_matmul for the same descriptor.
//   * the grid is persistent and sized to what is resident on the device (an upper bound of the work, capped at one wave), not to
//     E: with 128 experts of which 8 are active, no CTA is spent on an empty expert.  Every CTA stages the (clamped) offsets in
//     shared memory, derives each group's count of work items -- (16-row block of W, chunk of 8 * NT rows of A) -- with one
//     warp-wide prefix sum, and walks the items blockIdx.x, blockIdx.x + gridDim.x, ...  An item's expert is found by binary
//     search over the prefix sums; items run expert by expert, row chunk by row chunk, row block by row block.
//   * rows per pass (NT batch tiles of 8) are chosen on the host from the mean rows per active expert.  A group with more
//     rows than 8 * NT is served by several passes over its weights (the later passes mostly hit L2).
//   * programmatic dependent launch: the offsets and the sorted activations are written by the routing kernels right before
//     this one, and which experts' weights to stream is not known before the offsets are.  So griddepcontrol.wait is the first
//     instruction; unlike the single-matrix GEMV no weight is prefetched before it.  launch_dependents follows the CTA's last item.
//   * the offsets are untrusted: each is clamped to [0, T] and a group whose end is below its start is empty, so a malformed
//     table never reads or writes outside A[0:T] / C[0:T]; rows that no group claims are not written.
//   * SWIGLU instances (bb_matmul_grouped_swiglu): W holds gate/up interleaved and the tile epilogue writes silu(gate) * up into
//     C [T, N / 2] (gemv_mma_tile, bb_gemv_mma.cuh; DESIGN.md §3.2.1).
#include <algorithm>
#include <climits>

#include "bb_gemv_mma.cuh"

namespace bb {

namespace {

struct GroupedParams {
  GemvParams p;               // the problem of group 0 (p.M unused; p.out: C with row stride N)
  const int32_t* offsets;     // [E + 1], device
  int E;                      // groups
  int T;                      // rows of A and C
  long long w_stride;         // bytes per group: W, scale, zeros, bias
  long long s_stride, z_stride, b_stride;
  int out_bytes;              // bytes per element of C
};

template <typename T, int BITS, bool IL, int NT, int ZK, bool SC, bool SWIGLU = false>
__global__ void __launch_bounds__(gemv_max_ks(NT) * 32) __maxnreg__(gemv_mma_maxnreg(NT, ZK))
gemv_grouped_kernel(const GroupedParams g) {
  constexpr int R = 8 * NT;   // rows of A per pass over a 16-row block of W
  __shared__ float red[MAX_KS][16][8 * NT];
  __shared__ int row0_s[BB_GROUPED_MAX_GROUPS];       // clamped first row of each group
  __shared__ int rows_s[BB_GROUPED_MAX_GROUPS];       // rows of each group (0: empty)
  __shared__ int item0_s[BB_GROUPED_MAX_GROUPS + 1];  // first work item of each group; item0_s[E] = all items

  pdl_wait();   // offsets and A are the preceding kernels' output; nothing is read before this (see the header)
  const int nb = g.p.N / 16;
  if (threadIdx.x < 32) grouped_schedule(g, R, nb, row0_s, rows_s, item0_s);
  __syncthreads();
  const int total = item0_s[g.E];

  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    const int e = grouped_find(item0_s, g.E, item);
    const int local = item - item0_s[e];
    const int chunk = local / nb, rb = local - chunk * nb;
    const int r0 = row0_s[e] + chunk * R;
    GemvParams p = g.p;
    p.out.n = 1;   // one destination: the epilogue's loop over out.ptr then indexes it statically
    p.M = min(R, rows_s[e] - chunk * R);
    p.A = reinterpret_cast<const T*>(g.p.A) + size_t(r0) * p.K;
    p.W = g.p.W + size_t(e) * size_t(g.w_stride);
    if (SC) p.scale = reinterpret_cast<const uint8_t*>(g.p.scale) + size_t(e) * size_t(g.s_stride);
    if (ZK) p.zeros = reinterpret_cast<const uint8_t*>(g.p.zeros) + size_t(e) * size_t(g.z_stride);
    if (g.p.bias) p.bias = reinterpret_cast<const uint8_t*>(g.p.bias) + size_t(e) * size_t(g.b_stride);
    p.out.ptr[0] = reinterpret_cast<uint8_t*>(g.p.out.ptr[0]) + size_t(r0) * size_t(SWIGLU ? p.N / 2 : p.N) * size_t(g.out_bytes);
    if (item != int(blockIdx.x)) __syncthreads();   // the previous item's epilogue has finished reading `red`
    gemv_mma_tile<T, BITS, IL, NT, ZK, SC, false, SWIGLU>(p, rb, red);
  }
  pdl_launch_dependents();
}

// K splits (warps per CTA) as the decode GEMV picks them, for an upper bound of the work items as the CTA count; the grid is
// that bound, capped at the resident CTAs.
template <typename KernelT>
int launch_grouped_kernel(KernelT kernel, KernelCache<MAX_KS + 1>& cache, GroupedParams g, int max_items, int max_ks,
                          cudaStream_t stream) {
  const int ks = pick_ks(cache, kernel, max_ks, max_items, g.p.K / 128);
  g.p.ks = ks;
  const int resident = kernel_setup(cache, kernel, 0, ks * 32, 0, ks) * device_sm_count();
  if (resident <= 0) { set_error("grouped matmul: the kernel cannot be resident on this device"); return 2; }
  return launch_pdl(kernel, std::min(max_items, resident), ks * 32, 0, stream, pdl_enabled(), g);
}

template <typename T, int BITS, bool IL, bool SWIGLU>
int launch_grouped_nt(const GroupedParams& g, int rows, const int (&max_items)[3], cudaStream_t s) {
  return gemv_mma_instance(g.p, rows, [&](auto nt, auto zk, auto sc) {
    constexpr int NT = decltype(nt)::value;
    static KernelCache<MAX_KS + 1> cache;
    return launch_grouped_kernel(gemv_grouped_kernel<T, BITS, IL, NT, decltype(zk)::value, decltype(sc)::value, SWIGLU>, cache, g,
                                 max_items[NT == 1 ? 0 : (NT == 2 ? 1 : 2)], gemv_max_ks(NT), s);
  });
}

size_t elem_bytes(int dtype) { return dtype == BB_F32 ? 4 : 2; }

template <bool SWIGLU>
int launch_grouped_typed(const bb_matmul_desc& d, const GroupedParams& g, int rows, const int (&max_items)[3], cudaStream_t s) {
  return dispatch_t_bits_il(d, [&](auto t, auto bits, auto il) {
    return launch_grouped_nt<typename decltype(t)::type, decltype(bits)::value, decltype(il)::value, SWIGLU>(g, rows, max_items, s);
  });
}

}  // namespace

// the configurations the grouped kernel covers (those of gemv_mma, for any m); sets the error message otherwise
bool grouped_supported(const bb_matmul_desc& d) {
  if (d.a_dtype != BB_F16 && d.a_dtype != BB_BF16) { set_error("grouped matmul: activations must be float16 or bfloat16"); return false; }
  if ((d.w_fmt != BB_W_UINT && d.w_fmt != BB_W_INT) || (d.w_bits != 4 && d.w_bits != 2)) {
    set_error("grouped matmul: weights must be 4- or 2-bit uint / int (w_fmt=%d w_bits=%d)", d.w_fmt, d.w_bits);
    return false;
  }
  if (d.w_tile != BB_TILE_ROW_MAJOR) { set_error("grouped matmul: slab-tiled weights are not supported (row-major storage only)"); return false; }
  if (d.w_layout == BB_LAYOUT_INTERLEAVED_8) { set_error("grouped matmul: the int8-target interleave is not supported"); return false; }
  if (d.N % 16 || d.K % 128) { set_error("grouped matmul: needs N %% 16 == 0 and K %% 128 == 0 (N=%d K=%d)", d.N, d.K); return false; }
  const int g = d.group_size <= 0 ? d.K : d.group_size;
  if (g % 128) { set_error("grouped matmul: group_size must be a multiple of 128 or -1 (got %d)", d.group_size); return false; }
  if (!gemv_mma_supported(d, 1)) {
    set_error("grouped matmul: unsupported scale / zeros / out_dtype combination (zeros need scaling, int weights take no "
              "zeros, out_dtype float16 | bfloat16 | float32, quantized zeros need N*bits %% 8 == 0)");
    return false;
  }
  return true;
}

int launch_grouped(const GroupedArgs& a) {
  const bb_matmul_desc& d = a.d;
  GroupedParams g;
  g.p = make_params(d, a.A, a.W, a.scale, a.zeros, a.bias, make_outspec(a.C, a.swiglu ? d.N / 2 : d.N), 0);
  g.offsets = a.offsets; g.E = a.num_groups; g.T = a.total_rows;
  g.w_stride = a.w_stride; g.s_stride = a.s_stride; g.z_stride = a.z_stride; g.b_stride = a.b_stride;
  g.out_bytes = int(elem_bytes(d.out_dtype));
  // rows per pass: 8, 16 or 32 (gemv_nt), from the mean rows per active group (T rows over at most min(E, T) groups)
  const int total_rows = a.total_rows;
  const int active = std::min(a.num_groups, total_rows);
  const int mean_rows = (total_rows + active - 1) / active;
  // work items: sum_e ceil(m_e / R) row chunks per 16-row block <= T / R + (groups with rows)
  const long long nb = d.N / 16;
  int max_items[3];
  const int R[3] = {8, 16, 32};
  for (int i = 0; i < 3; ++i) {
    const long long items = nb * (total_rows / R[i] + active);
    if (items > INT_MAX) { set_error("grouped matmul: N/16 x (T/rows + groups) exceeds 2^31 work items"); return 1; }
    max_items[i] = int(items);
  }
  return a.swiglu ? launch_grouped_typed<true>(d, g, mean_rows, max_items, a.stream)
                  : launch_grouped_typed<false>(d, g, mean_rows, max_items, a.stream);
}

}  // namespace bb
