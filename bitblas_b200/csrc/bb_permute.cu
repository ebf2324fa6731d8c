// bb_permute.cu -- the activation column gather of GPTQ act-order layers (bb_permute_cols): out[r, j] = A[r, perm[e * K + j]],
// e the group of row r.
//
// An act-order checkpoint assigns input column k to quantization group g_idx[k]; the loader sorts the weight's K axis by g_idx
// (bitblas_b200/act_order.py), so the matmul kernels read the contiguous group layout, and the activations are gathered into the
// same order before the matmul.  The values are only moved, never converted, so fp16 and bf16 share one 16-bit instance.
//
// Schedule: a work item is a tile of up to R consecutive rows of one group (R from K: the tile's rows fill PERMUTE_TILE_BYTES of
// shared memory, at least one row).  The grid strides over the items; with offsets, every CTA computes the items from the clamped
// offsets itself (grouped_schedule, the grouped matmuls' rule), so the launch needs no host synchronisation.
//   * the tile's rows are copied into shared memory with 16-byte cp.async (the gather then reads shared memory, where 32 random
//     2-byte reads cost a few bank conflicts instead of up to 32 L1 line lookups);
//   * each thread takes 8 consecutive output columns, reads their 8 perm entries once (clamped to [0, K)) and, for every row of the
//     tile, gathers 8 values from shared memory and stores them as one 16-byte vector.
//   * PDL: griddepcontrol.wait before the first read of offsets or A (the preceding kernel's output); launch_dependents after the
//     last store, as the routing kernel does.  Triggering at the start measured no gain for the m = 1 decode GEMV and made the
//     grouped GEMV after it up to 1.4x slower (H100 80GB HBM3, 700 W: its persistent grid launched while this grid still held SMs).
#include <algorithm>

#include "bb_common.cuh"

namespace bb {

namespace {

constexpr int PERMUTE_THREADS = 256;
constexpr int PERMUTE_TILE_BYTES = 32 * 1024;   // shared memory of one tile, unless one row is larger
constexpr int PERMUTE_MAX_TILE_ROWS = 16;
constexpr int PERMUTE_MAX_SMEM = 2 * PERMUTE_MAX_K;   // the dynamic shared memory opted into: one row

struct PermuteParams {
  const uint16_t* A;          // [T, K]
  uint16_t* out;              // [T, K]
  const int32_t* perm;        // [E, K]
  const int32_t* offsets;     // [E + 1], or null: one group of all T rows
  int T, K, E, R;             // rows, columns, groups, rows per tile
};

__global__ void __launch_bounds__(PERMUTE_THREADS) permute_cols_kernel(const PermuteParams p) {
  extern __shared__ __align__(16) uint16_t tile_s[];   // [R, K]
  __shared__ int row0_s[BB_GROUPED_MAX_GROUPS], rows_s[BB_GROUPED_MAX_GROUPS], item0_s[BB_GROUPED_MAX_GROUPS + 1];
  pdl_wait();   // A and offsets are the preceding kernels' output
  const int tid = threadIdx.x, vecs = p.K / 8;
  int items;
  if (p.offsets) {
    if (tid < 32) grouped_schedule(p, p.R, 1, row0_s, rows_s, item0_s);
    __syncthreads();
    items = item0_s[p.E];
  } else {
    items = (p.T + p.R - 1) / p.R;
  }
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    int e = 0, r0, n;
    if (p.offsets) {
      e = grouped_find(item0_s, p.E, item);
      const int t = item - item0_s[e];
      r0 = row0_s[e] + t * p.R;
      n = min(p.R, rows_s[e] - t * p.R);
    } else {
      r0 = item * p.R;
      n = min(p.R, p.T - r0);
    }
    const uint4* src = reinterpret_cast<const uint4*>(p.A + size_t(r0) * p.K);
    uint4* tile4 = reinterpret_cast<uint4*>(tile_s);
    for (int v = tid; v < n * vecs; v += PERMUTE_THREADS) cp_async16(smem_u32(tile4 + v), src + v);
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    const int32_t* pe = p.perm + size_t(e) * p.K;
    for (int v = tid; v < vecs; v += PERMUTE_THREADS) {
      int col[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) col[i] = min(max(__ldg(pe + 8 * v + i), 0), p.K - 1);
      for (int r = 0; r < n; ++r) {
        const uint16_t* row = tile_s + size_t(r) * p.K;
        uint4 q;
        q.x = uint32_t(row[col[0]]) | (uint32_t(row[col[1]]) << 16);
        q.y = uint32_t(row[col[2]]) | (uint32_t(row[col[3]]) << 16);
        q.z = uint32_t(row[col[4]]) | (uint32_t(row[col[5]]) << 16);
        q.w = uint32_t(row[col[6]]) | (uint32_t(row[col[7]]) << 16);
        reinterpret_cast<uint4*>(p.out + size_t(r0 + r) * p.K)[v] = q;
      }
    }
    __syncthreads();   // the tile is read before the next item overwrites it
  }
  pdl_launch_dependents();
}

}  // namespace

int launch_permute_cols(const void* A, void* out, const int32_t* perm, int rows, int K, int num_groups, const int32_t* offsets,
                        cudaStream_t stream) {
  const size_t row_bytes = size_t(K) * 2;
  static KernelCache<> cache;
  if (kernel_setup(cache, permute_cols_kernel, PERMUTE_MAX_SMEM) <= 0) {
    set_error("permute cols: raising the kernel's shared-memory limit failed");
    return 2;
  }
  PermuteParams p;
  p.A = reinterpret_cast<const uint16_t*>(A); p.out = reinterpret_cast<uint16_t*>(out); p.perm = perm; p.offsets = offsets;
  p.T = rows; p.K = K; p.E = num_groups;
  p.R = int(std::max<size_t>(1, std::min<size_t>(PERMUTE_MAX_TILE_ROWS, PERMUTE_TILE_BYTES / row_bytes)));
  const size_t smem = size_t(p.R) * row_bytes;
  // an upper bound on the items when the offsets partition the rows; overlapping groups are covered by the grid-stride loop
  const long long items = (rows + p.R - 1) / p.R + (offsets ? num_groups : 0);
  const unsigned grid = unsigned(std::min<long long>(items, 1ll << 30));
  return launch_pdl(permute_cols_kernel, grid, PERMUTE_THREADS, smem, stream, pdl_enabled(), p);
}

}  // namespace bb
