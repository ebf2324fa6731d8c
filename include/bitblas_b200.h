/*
 * bitblas_b200.h -- C ABI of the H100-native (sm_90a) low-bit-weight matmul library.
 *
 * This is the drop-in boundary for the ONE hot path of microsoft/BitBLAS: the dequantize-matmul behind
 * bitblas.Matmul / bitblas.Linear.  In the reference every operator instance owns a generated .so that
 * exports
 *     extern "C" void init();
 *     extern "C" void call(<T>* A, int8_t* B, [half* LUT], [half* Scale], [int8_t* Qzeros | half* Zeros],
 *                          [half* Bias], <T>* C, [int m], cudaStream_t stream);
 * (reference: bitblas/builder/wrapper/base.py:5-19, bitblas/builder/wrapper/tl.py:90-166,278-300; called
 * from bitblas/ops/operator.py:458-463 and bitblas/module/__init__.py:287 via ctypes).
 *
 * Here ONE prebuilt library serves every MatmulConfig: the config travels in a POD descriptor and the
 * entry points below replace init()/call().  Plain pointers and sizes only -- no torch types.  All device
 * buffers are caller-owned; the library never allocates, frees or synchronises inside bb_matmul, so the call
 * is CUDA-graph capturable.  Every function returns 0 on success; on failure a non-zero code is returned and
 * bb_last_error() describes it (the reference returns void and swallows errors, operator.py:200-214).
 */
#ifndef BITBLAS_B200_H_
#define BITBLAS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BB_VERSION 100 /* 0.1.0 */

/* element types of A / accumulator / output (MatmulConfig.A_dtype, accum_dtype, out_dtype:
 * bitblas/ops/general_matmul/__init__.py:63-67) */
typedef enum bb_dtype {
  BB_F16 = 0,
  BB_BF16 = 1,
  BB_F32 = 2,
  BB_I8 = 3,
  BB_I32 = 4,
  BB_E4M3 = 5  /* float8 e4m3 (OCP "fn": no infinities, max 448): activations of bb_matmul_fp8 only */
} bb_dtype;

/* weight source formats (Matmul.BITBLAS_TRICK_DTYPE_MAP, general_matmul/__init__.py:324-345) */
typedef enum bb_wfmt {
  BB_W_UINT = 0,    /* "uint"    : u                               (quantization.py:200-208) */
  BB_W_INT = 1,     /* "int"     : u - 2^(bits-1); 1-bit: 2u-1     (quantization.py:185-194, lop3.py:723-727) */
  BB_W_NF = 2,      /* "nf"      : LUT[u]                          (matmul_dequantize_impl.py:424-430) */
  BB_W_FP4 = 3,     /* "fp"      : sign + 3-bit exponent 2^(e-7)   (quantization.py:141-156) */
  BB_W_FP8_E4M3 = 4,/* "fp_e4m3" : bit trick                       (quantization.py:169-176) */
  BB_W_FP8_E5M2 = 5 /* "fp_e5m2" : reinterpret<<8                  (quantization.py:179-182) */
} bb_wfmt;

/* MatmulConfig.zeros_mode (general_matmul/__init__.py:73-78) */
typedef enum bb_zeros_mode {
  BB_ZEROS_ORIGINAL = 0,  /* (w - Z[n,k/g]) * S[n,k/g]   ; Z is A_dtype [N, K/g]            */
  BB_ZEROS_RESCALE = 1,   /*  w * S[n,k/g] - Z[n,k/g]    ; Z is A_dtype [N, K/g]            */
  BB_ZEROS_QUANTIZED = 2  /* (u - QZ[k/g,n]) * S[n,k/g]  ; QZ is `bits`-packed int8 [K/g, N*bits/8] */
} bb_zeros_mode;

/* weight storage layout of W[N, K*bits/8] int8 (general_matmul/__init__.py:557-565) */
typedef enum bb_wlayout {
  BB_LAYOUT_COMPRESSED = 0,      /* general_compress only            (quantization/utils.py:54-69)   */
  BB_LAYOUT_INTERLEAVED_16 = 1,  /* + LOP3 interleave, 16-bit target (quantization/utils.py:73-110)  */
  BB_LAYOUT_INTERLEAVED_8 = 2    /* + LOP3 interleave,  8-bit target (A_dtype == int8)               */
} bb_wlayout;

/* Offline tiling of the packed weight matrix (MatmulConfig.propagate_b).  The reference's weight propagation re-tiles W offline
 * so that its mma.sync kernels can use ldmatrix-friendly, conflict-free tiles (bitblas/ops/ladder_permutate/
 * ladder_permutate_impl.py:12-116, bitblas/gpu/matmul_analysis.py:691-801, general_matmul/__init__.py:113-157).  Here the
 * tensor-core operand layout is produced in registers by the kernels themselves; what an offline layout can still buy is DRAM/TMA
 * locality.  BB_TILE_SLAB stores the packed rows as [N/32][row_bytes/512][32 rows][512 B] (row_bytes = K*bits/8): one 16 KB
 * work unit of the decode GEMV is ONE contiguous block, and the 128-row x k-block tile of the wgmma kernel is four 4-D TMA
 * box rows of it.  Same bytes, same size, same interleave inside each 32-bit word; only the order of 512-byte row segments
 * changes.  Needs N % 32 == 0 and row_bytes % 512 == 0. */
typedef enum bb_wtile {
  BB_TILE_ROW_MAJOR = 0,
  BB_TILE_SLAB = 1
} bb_wtile;
#define BB_TILE_ROWS 32
#define BB_TILE_ROW_BYTES 512

/* One matmul problem family: C[m, N] = A[m, K] x dequant(W[N, K])^T (+ bias).  Mirrors the fields of
 * MatmulConfig that reach the kernel (general_matmul/__init__.py:58-95); `layout` is always "nt"
 * (tirscript/matmul_dequantize_impl.py:912-915). */
typedef struct bb_matmul_desc {
  int32_t N;
  int32_t K;
  int32_t a_dtype;      /* bb_dtype: BB_F16 | BB_BF16 | BB_I8                         */
  int32_t w_fmt;        /* bb_wfmt                                                    */
  int32_t w_bits;       /* 1 | 2 | 4 | 8                                              */
  int32_t accum_dtype;  /* bb_dtype: float accumulate is done in fp32; BB_I32 is exact */
  int32_t out_dtype;    /* bb_dtype of C                                              */
  int32_t group_size;   /* -1 (== K) or a divisor of K                                */
  int32_t with_scaling; /* Scale[N, K/g] in A_dtype                                   */
  int32_t with_zeros;
  int32_t zeros_mode;   /* bb_zeros_mode                                              */
  int32_t with_bias;    /* Bias[N] in out_dtype-compatible A_dtype                    */
  int32_t w_layout;     /* bb_wlayout                                                 */
  int32_t w_tile;       /* enum bb_wtile, from MatmulConfig.propagate_b; 0 = the reference row-major storage */
  int32_t reserved[2];  /* must be 0                                                  */
} bb_matmul_desc;

/* kernel families the dispatcher can choose (introspection / tests) */
typedef enum bb_kernel_id {
  BB_KERNEL_AUTO = 0,
  BB_KERNEL_GENERIC = 1,   /* SIMT, every config (spec-order arithmetic)                     */
  BB_KERNEL_GEMV_MMA = 2,  /* m <= 32, fp16/bf16 A, 4/2-bit W: warp-level mma.sync streaming  */
  BB_KERNEL_GEMV_I8 = 3,   /* m <= 32, int8 A, 4/2-bit W: IMMA streaming, int32 exact         */
  BB_KERNEL_GEMM_TS = 4,   /* wgmma (W dequantised into registers as the MMA A operand) + TMA */
  BB_KERNEL_GEMM_TS_I8 = 5,/* wgmma int8 variant                                             */
  BB_KERNEL_GEMV_SLAB = 7,   /* m == 1, 4-bit W, fp16/bf16 A: per-CTA TMA slabs + CTA-level stream-K; the default
                              * decode kernel (needs the zero-initialised workspace of bb_workspace_bytes) */
  BB_KERNEL_GEMM_FP8 = 8     /* bb_matmul_fp8 only: block-scaled e4m3 x e4m3 wgmma, both operands from shared memory */
} bb_kernel_id;

/* replaces `init()` (builder/wrapper/base.py:5-13): one-time per-device setup (opt-in shared memory
 * sizes, driver entry points).  Idempotent and thread-safe. */
int bb_init(int device);

/* replaces `call(...)` (builder/wrapper/base.py:15-19).  Pointer order follows the reference's
 * A, B, [LUT], [Scale], [Zeros|Qzeros], [Bias], C, m, stream; absent operands are NULL.
 * `m` = product of A's leading dims (general_matmul/__init__.py:746-748); m == 0 returns immediately
 * (wrapper/tl.py:156-157).  `workspace` may be NULL unless bb_workspace_bytes() > 0.
 * Asynchronous on `stream` (a cudaStream_t). */
int bb_matmul(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
              const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes,
              void* stream);

/* Column-parallel variant (no reference counterpart: the reference is single-GPU, SURVEY.md §2a).  `desc->N` is THIS
 * rank's shard of the output features; the epilogue of the matmul kernel stores the [m, desc->N] result into columns
 * [col_offset, col_offset + desc->N) of EVERY buffer in `peer_C` (row stride `ldc` elements) -- the peers' copies are
 * peer-mapped device pointers (NVLink P2P / symmetric memory), so the all-gather of the sharded outputs happens inside the
 * kernel, tile by tile, instead of as a separate collective.  The caller must barrier across ranks before reading.
 * n_peers <= BB_MAX_PEERS. */
#define BB_MAX_PEERS 8
int bb_matmul_scatter(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                      const void* zeros, const void* bias, void* const* peer_C, int n_peers, int64_t ldc,
                      int64_t col_offset, int m, void* workspace, size_t workspace_bytes, void* stream);

/* The gate/up projection of a dense SwiGLU MLP in one call: the operands, workspace, kernel choice (bb_select_kernel, the kernel
 * override and the SM-count cap apply unchanged), launch count and stream semantics of bb_matmul, with desc->N = 2I fused gate/up
 * rows stored in the gate/up interleave of the grouped SwiGLU calls below (stored row 16b + i is gate row 8b + i for i < 8 and up
 * row 8b + i - 8 for i >= 8; scale, zeros and bias rows follow it, quantized zeros in whole bytes).  C is [m, I]:
 *     C[r, 8b + i] = round_out(silu(g) * u),   silu(g) = g / (1 + exp(-g)) in fp32, one rounding,
 * where g and u are exactly what bb_matmul stores for rows 16b + i and 16b + i + 8 (cast to out_dtype, bias added in out_dtype;
 * fp32 output stays fp32).  Covers every desc bb_matmul accepts with fp16 / bf16 activations and N % 16 == 0; int8 activations
 * and N % 16 != 0 are rejected.  m == 0 returns 0 and launches nothing. */
int bb_matmul_swiglu(const bb_matmul_desc* desc, const void* A, const void* W, const void* lut, const void* scale,
                     const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes,
                     void* stream);

/* BitNet b1.58 layers from 16-bit activations: bb_quantize_act_int8 quantizes each row of x to int8 with its own scale, and
 * bb_matmul_scaled runs the int8 matmul of those rows with an epilogue that undoes both quantization scales.  Every operation is
 * in fp32 and correctly rounded, so results are reproducible bit for bit.
 *
 * bb_quantize_act_int8: x [rows, K] of a_dtype (float16 | bfloat16) -> q int8 [rows, K] and scale fp32 [rows], per row r:
 *     amax     = max_k |float(x[r, k])|                                   (exact)
 *     scale[r] = 127.0f * (1.0f / max(amax, 1e-5f))                      (IEEE reciprocal, then IEEE product)
 *     q[r, k]  = int8(clamp(rint(float(x[r, k]) * scale[r]), -128, 127))  (IEEE product, then round half to even)
 * (BitNet's activation_quant exactly as torch evaluates it: `127.0 / t` is reciprocal(t) * 127 there; an all-zero row gives scale 1.27e7 and q = 0; a row holding Inf or NaN gives unspecified values.)
 * K % 8 == 0; x and q 16-byte aligned, scale 4-byte aligned (code 5 otherwise).  ONE launch, no workspace, no host
 * synchronisation (CUDA-graph capturable); programmatic stream serialization: x is read only after the preceding kernel has
 * completed, and the next kernel may launch once this one has stored its results.  rows == 0 validates and returns 0 without
 * touching the device.
 *
 * bb_matmul_scaled: the int8 matmul of bb_matmul (A int8 [m, K] x W, exact int32 accumulation acc) with a dequantizing epilogue
 *     C[r, n] = round_out((float(acc[r, n]) / a_scale[r]) / w_scale[n])   (+ bias[n], added in out_dtype after the rounding)
 * with float(acc) round-to-nearest and both divisions IEEE; an fp32 output is (...) + bias in fp32.  a_scale is fp32 [m] (the
 * scale of bb_quantize_act_int8), w_scale fp32 [N] (one quantization scale per output row of W; a per-tensor scale is N copies),
 * both 4-byte aligned; bias, when desc->with_bias, is [N] in out_dtype.  Covers every desc bb_matmul accepts with a_dtype ==
 * BB_I8, out_dtype float16 | bfloat16 | float32 and with_scaling == with_zeros == 0; everything else is rejected, each with its own
 * message, in bb_matmul's order (descriptor, then m, then pointers).  Kernel choice (bb_select_kernel, the kernel override, the
 * SM-count cap), bb_workspace_bytes, launch count and stream semantics are those of bb_matmul for the same desc; m == 0 returns 0
 * and launches nothing.  a_scale, like A, is read only after the preceding kernel has completed. */
int bb_quantize_act_int8(const void* x, int a_dtype, int rows, int K, int8_t* q, float* scale, void* stream);
int bb_matmul_scaled(const bb_matmul_desc* desc, const void* A, const void* W, const float* a_scale, const float* w_scale,
                     const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream);

/* GPTQ-style 4-bit weights with int8 activations (W4A8): A int8 [m, K] (from bb_quantize_act_int8) against 4-bit weights with one
 * fp32 scale per (row, group) and optional quantized zero points.  desc: a_dtype = BB_I8, accum_dtype = BB_I32, w_bits = 4, w_fmt
 * uint or int, with_scaling = 1, with_zeros only for uint weights and only in mode BB_ZEROS_QUANTIZED (zeros [K/g, N/2] packed as
 * bb_repack_gptq_qzeros_device writes them), out_dtype float16 | bfloat16 | float32, g = -1 or a divisor of K.  With w[n, k] the
 * integer bb_matmul decodes (u for uint, u - 8 for int, u - z[n, g] with zeros; always in [-15, 15]):
 *     acc[r, n, g] = sum_{k in group g} A[r, k] * w[n, k]                        exact int32
 *     S[r, n]      = sum_g float(acc[r, n, g]) * scale[n, g]                      fp32, each conversion, product and sum rounded
 *     C[r, n]      = round_out(S[r, n] / a_scale[r])   (+ bias[n], [N] in out_dtype, added after the rounding; IEEE division)
 * scale is fp32 [N, K/g] and a_scale fp32 [m], both 4-byte aligned.  The order of the fp32 sum over groups is fixed per kernel,
 * split factor and SM count, so a call is deterministic:
 *   - generic_simt and gemm_ts_wgmma_i8 without split-K: S = (((0 + p_0) + p_1) + ...) + p_{G-1}, p_g = float(acc) * scale, in
 *     group order;
 *   - gemm_ts_wgmma_i8 split s ways (s divides G; split j owns groups [jG/s, (j+1)G/s)): each split sums its groups as above, and
 *     S = ((0 + S_0) + S_1) + ... + S_{s-1};
 *   - gemv_i8: the CTA's warps own contiguous ranges of whole groups (as many warps as the launch picks, at most G); each sums
 *     its groups as above, and S = ((0 + S_warp0) + S_warp1) + ... in warp order.  So with few groups the K split is small: at
 *     g = -1 (G = 1) every 16-row block of W is streamed by one warp, which makes such a decode much slower than with g = 128.
 * Kernel choice: the family bb_select_kernel picks for the same desc with with_scaling = with_zeros = 0 (gemv_i8, gemm_ts_wgmma_i8
 * or generic_simt), except that g % 128 != 0 runs generic_simt instead of gemv_i8 / gemm_ts_wgmma_i8 (under a kernel override
 * forcing one of those two it is not supported).  The override and the SM-count cap apply; bb_select_kernel_w4a8 reports the
 * choice (-1 on an invalid desc).  The workspace is bb_workspace_bytes of that cleared desc, which always suffices (a split factor
 * is never above the plain call's); a smaller or null workspace runs without split-K.  Rejections come in bb_matmul_scaled's order,
 * each with its own message: 16-bit activations, an int out_dtype, with_scaling = 0, original / rescale zeros, other bit widths and
 * formats, int weights with zeros, then m, then null a_scale / scale (code 1) and misaligned ones (code 5).  m == 0 returns 0 and
 * launches nothing.  Launch count, stream semantics, PDL behaviour and graph capture are those of bb_matmul_scaled. */
int bb_matmul_w4a8(const bb_matmul_desc* desc, const void* A, const void* W, const float* a_scale, const float* scale,
                   const void* zeros, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream);
int bb_select_kernel_w4a8(const bb_matmul_desc* desc, int m);

/* 128 x 128 block-scaled FP8 checkpoints (DeepSeek-V3 / R1, Qwen3 -FP8: weight float8_e4m3fn [N, K], weight_scale_inv fp32
 * [ceil(N/128), K/128]) on the FP8 tensor cores, with activations quantized per (token, 128-column block) on the device.
 *
 * bb_quantize_act_fp8: x [rows, K] of a_dtype (float16 | bfloat16) -> q e4m3 bytes [rows, K] and one fp32 scale per (row r,
 * block b = k / 128), each step correctly rounded in fp32 (vLLM's per_token_group_quant_fp8 with IEEE division):
 *     amax[r, b] = max(max_{k in b} |float(x[r, k])|, 1e-10f)
 *     s[r, b]    = amax[r, b] / 448.0f                                     (IEEE division)
 *     q[r, k]    = e4m3_rn(clamp(float(x[r, k]) / s[r, b], -448, 448))     (IEEE division, round to nearest even)
 * An all-zero block gives q = 0; Inf or NaN inputs give unspecified values.  The scales are k-block-major: (r, b) is
 * scale[b * scale_ld + r], scale_ld >= rows and scale_ld % 4 == 0, so a GEMM tile's scales for one k-block are one contiguous,
 * 16-byte-aligned run.  K % 128 == 0; x, q and scale 16-byte aligned (code 5 otherwise).  ONE launch, no workspace, CUDA-graph
 * capturable; programmatic stream serialization as bb_quantize_act_int8.  rows == 0 validates and returns 0 without touching
 * the device.
 *
 * bb_matmul_fp8: A e4m3 [m, K] with a_scale (bb_quantize_act_fp8's layout, a_scale_ld >= m, a_scale_ld % 4 == 0) against W e4m3
 * [N, K] (the checkpoint's bytes, row-major) with w_scale fp32 [ceil(N/128), K/128] row-major.  desc: a_dtype = BB_E4M3, w_fmt =
 * BB_W_FP8_E4M3, w_bits = 8, accum_dtype = BB_F32, out_dtype float16 | bfloat16 | float32, group_size = 128, with_scaling = 1,
 * with_zeros = 0, compressed row-major storage; N % 16 == 0 (the last 128-row weight tile may be partial), K % 128 == 0.
 *     P[r, n, b] = sum_{k in block b} q_a[r, k] * q_w[n, k]          tensor-core e4m3 MMA, fp32 accumulator
 *     S[r, n]    = sum_b P[r, n, b] * (a_scale[r, b] * w_scale[n / 128, b])
 *     C[r, n]    = round_out(S[r, n])   (+ bias[n], [N] in out_dtype, added after the rounding; an fp32 output is one sum)
 * Each product of P is exact; how the tensor core accumulates the 128 products of a block is not specified.  S is fp32 with every
 * product and sum rounded (no fma): S = (((0 + t_0) + t_1) + ...) with t_b = P[r, n, b] * (a_scale * w_scale), blocks ascending.
 * Split s ways (split j owns blocks [j KB/s, (j+1) KB/s), KB = K/128), each split sums its own blocks from 0 as above, and
 * S = ((0 + S_0) + S_1) + ... + S_{s-1}.  The split factor is gemm_ts's rule on this kernel's tiles (m <= 128, a tile grid that
 * leaves SMs idle, at least 8 blocks per split) under bb_set_sm_count_cap; bb_workspace_bytes_fp8 is the fp32 [splits][m][N] it
 * needs (0 without a split), and a smaller or null workspace runs unsplit.  Kernel: BB_KERNEL_GEMM_FP8 under AUTO or that
 * override; any other override is refused (code 1), and bb_select_kernel_fp8 reports -1 then (and on an invalid desc or m < 1).
 * Rejections, each with its own message: the descriptor, then m, then a_scale_ld, then null pointers (code 1), then A, W and
 * a_scale not 16-byte aligned or w_scale not 4-byte aligned (code 5).  m == 0 returns 0 and launches nothing.  One launch, two
 * with split-K, counted by bb_launch_count; no host synchronisation (CUDA-graph capturable); A and a_scale are read only after
 * the preceding kernel has completed.  No other entry point but bb_matmul_grouped_fp8[_swiglu] accepts a_dtype = BB_E4M3. */
int bb_quantize_act_fp8(const void* x, int a_dtype, int rows, int K, void* q, float* scale, int scale_ld, void* stream);
int bb_matmul_fp8(const bb_matmul_desc* desc, const void* A, const float* a_scale, int a_scale_ld, const void* W,
                  const float* w_scale, const void* bias, void* C, int m, void* workspace, size_t workspace_bytes, void* stream);
int bb_select_kernel_fp8(const bb_matmul_desc* desc, int m);
size_t bb_workspace_bytes_fp8(const bb_matmul_desc* desc, int m);

/* Grouped matmul for mixture-of-experts layers (no reference counterpart; the contract of torch._grouped_mm with offsets).
 * `num_groups` problems share `desc` and run as ONE kernel launch.  A[total_rows, K] holds the rows of every group, sorted so
 * that group e owns rows [offsets[e], offsets[e+1]); `offsets` is a DEVICE int32 array of num_groups + 1 entries, read by the
 * kernel (no host synchronisation: the call is CUDA-graph capturable for every routing).  For every group e:
 *     C[offsets[e] : offsets[e+1]] = A[offsets[e] : offsets[e+1]] x dequant(W[e])^T (+ bias[e])
 * with the formula and rounding of bb_matmul for `desc`.  The per-group operands are stacked: W [E, N, K*bits/8] in the storage
 * of bb_matmul, scale [E, N, K/g], zeros [E, N, K/g] (A_dtype) or [E, K/g, N*bits/8] (quantized), bias [E, N].
 * Offsets are clamped to [0, total_rows] and a group whose end is below its start is empty, so a malformed table never reads or
 * writes outside A / C; rows no group claims are not written.  Covers fp16 / bf16 A, 4- and 2-bit uint / int W in row-major
 * compressed or interleaved-16 storage, K % 128 == 0, N % 16 == 0, group_size a multiple of 128 or -1; everything else is
 * rejected.  total_rows == 0 validates and returns 0 without touching the device.  num_groups <= BB_GROUPED_MAX_GROUPS.
 * Launched with programmatic stream serialization like the decode kernels, but offsets, A AND W are read only after the
 * preceding kernel has completed (which weights to read depends on the offsets). */
#define BB_GROUPED_MAX_GROUPS 256
int bb_matmul_grouped(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                      const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream);

/* Grouped matmul on the wgmma GEMM, for mixture-of-experts prefill: the signature, operand layout and offset contract of
 * bb_matmul_grouped, with the numerics of bb_matmul on the wgmma GEMM (gemm_ts, without split-K), in ONE CUDA-graph capturable
 * launch at any number of rows per group.  Covers what bb_matmul_grouped covers with N % 128 == 0 (the CTA tile is 128 weight
 * rows); everything else is rejected with a message.  Takes no workspace.  total_rows == 0 validates and returns 0 without
 * touching the device; A and W must be 16-byte aligned.  Launched with programmatic stream serialization; offsets, A and W
 * are read only after the preceding kernel has completed. */
int bb_matmul_grouped_gemm(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                           const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream);

/* SwiGLU forms of the two grouped calls, for the gate/up projection of a mixture-of-experts expert block: the operands, offset
 * contract, coverage and rejections of bb_matmul_grouped / bb_matmul_grouped_gemm, with desc->N = 2I fused gate/up rows stored in
 * the "gate/up interleave": stored row 16b + i is gate row 8b + i for i < 8 and up row 8b + i - 8 for i >= 8 (so I % 8 == 0; the
 * GEMM form also needs 2I % 128 == 0).  Scale, zeros and bias rows follow the same permutation (quantized zeros, packed along N,
 * move in whole bytes: 8 rows are 4 bytes at 4 bits, 2 at 2 bits).  C is [total_rows, I]:
 *     C[r, 8b + i] = round_out(silu(g) * u),   silu(g) = g / (1 + exp(-g)) in fp32, one rounding,
 * where g and u are exactly what the plain call stores for the two rows (cast to out_dtype, bias added in out_dtype; fp32 output
 * stays fp32).  The kernel instance is chosen from total_rows and num_groups exactly as in the plain calls. */
int bb_matmul_grouped_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                             const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream);
int bb_matmul_grouped_gemm_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const void* W,
                                  const void* scale, const void* zeros, const void* bias, void* C, int total_rows, void* stream);

/* bb_matmul_grouped_gemm_swiglu reading its rows through an index: sorted row r of group e is A[clamp(row_index[r], 0,
 * a_rows - 1)] of A [a_rows, K], so a mixture-of-experts block multiplies the token rows in place (row_index = the row_token of
 * bb_moe_route_index) instead of a routed copy.  row_index is a DEVICE int32 array of total_rows entries, 4-byte aligned, read
 * on the device; any value is clamped, so every read stays inside A.  Everything else -- coverage (N % 128 == 0), rejections,
 * offsets, the instance choice from total_rows and num_groups, the SwiGLU epilogue and C [total_rows, N / 2] -- is that of
 * bb_matmul_grouped_gemm_swiglu, and the result equals that call on the gathered rows bit for bit.  a_rows >= 1 when
 * total_rows > 0.  ONE launch, CUDA-graph capturable, programmatic stream serialization. */
int bb_matmul_grouped_gemm_swiglu_gather(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets,
                                         const int32_t* row_index, const void* A, int a_rows, const void* W,
                                         const void* scale, const void* zeros, const void* bias, void* C,
                                         int total_rows, void* stream);

/* Grouped block-scaled FP8 matmul for mixture-of-experts layers whose experts are 128 x 128 block-scaled e4m3 checkpoints
 * (DeepSeek-V3 / R1, Qwen3 -FP8): ONE launch over num_groups experts with the offset contract of bb_matmul_grouped, and for
 * every expert e the numerics of bb_matmul_fp8 without a split:
 *     C[r, n] = round_out(S[r, n]),  S[r, n] = sum_b P[r, n, b] * (a_scale[r, b] * w_scale[e, n / 128, b])   for offsets[e] <= r < offsets[e+1]
 * P the tensor core's e4m3 sum over block b (each product exact; its order within the block unspecified); S is fp32 with every
 * product and sum rounded (no fma), S = (((0 + t_0) + t_1) + ...), blocks ascending; round_out casts to out_dtype (fp32 stays).
 * So each expert's rows equal bb_matmul_fp8 on those rows and W[e] run unsplit (without a workspace), bit for bit.
 *   - A e4m3 [total_rows, K], sorted by expert; a_scale its bb_quantize_act_fp8 scales, k-block-major: (r, b) at
 *     a_scale[b * a_scale_ld + r], a_scale_ld >= total_rows, a_scale_ld % 4 == 0.
 *   - W e4m3 [E, N, K], the checkpoint's per-expert [N, K] bytes stacked; w_scale fp32 [E, N/128, K/128].
 *   - offsets: a DEVICE int32 array of num_groups + 1 entries, read by the kernel; clamped to [0, total_rows], a group whose end
 *     is below its start is empty, rows no group claims are not written.  1 <= num_groups <= BB_GROUPED_MAX_GROUPS.
 *   - desc: that of bb_matmul_fp8, with N % 128 == 0 (an expert's 128-row tile must not read the next expert's rows) and
 *     with_bias = 0.  No workspace.
 * bb_matmul_grouped_fp8_swiglu, the gate/up projection: desc->N = 2I rows of W[e] in the gate/up interleave (stored row 16b + i
 * is gate row 8b + i for i < 8 and up row 8b + i - 8 for i >= 8; 2I % 128 == 0), so stored 128-row tile t holds gate and up rows
 * 64t .. 64t + 63.  Its scales are interleaved by block: w_scale fp32 [E, 2 ceil(I/128), K/128], row 2c the gate block c and row
 * 2c + 1 the up block c, so tile t reads rows 2(t >> 1) and 2(t >> 1) + 1.  C is [total_rows, I]:
 *     C[r, c] = round_out(silu(g) * u),   silu(g) = g / (1 + exp(-g)) in fp32, one rounding,
 * with g and u exactly what the plain call would store for gate row c and up row c of the de-interleaved weights and scales.
 * Rejections, each with its own message: the descriptor (bb_matmul_fp8's checks), N % 128, with_bias, num_groups, total_rows < 0
 * (code 1); total_rows == 0 then validates and returns 0 without touching the device; then a_scale_ld, null pointers (code 1),
 * A, W and a_scale not 16-byte aligned or w_scale and offsets not 4-byte aligned (code 5), and a kernel override other than AUTO
 * or BB_KERNEL_GEMM_FP8 (code 1).  ONE launch counted by bb_launch_count, no host synchronisation (CUDA-graph capturable),
 * programmatic stream serialization; offsets, A, a_scale and W are read only after the preceding kernel has completed. */
int bb_matmul_grouped_fp8(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A, const float* a_scale,
                          int a_scale_ld, const void* W, const float* w_scale, void* C, int total_rows, void* stream);
int bb_matmul_grouped_fp8_swiglu(const bb_matmul_desc* desc, int num_groups, const int32_t* offsets, const void* A,
                                 const float* a_scale, int a_scale_ld, const void* W, const float* w_scale, void* C, int total_rows,
                                 void* stream);

/* Mixture-of-experts routing on the device: slot s = t * top_k + j of the DEVICE int32 table topk_ids [num_tokens, top_k] goes to
 * expert topk_ids[s].  Writes offsets [num_experts + 1] (the offsets of bb_matmul_grouped), slot_rows [T * top_k] (the sorted row
 * of each slot) and x_sorted [T * top_k, K] with x_sorted[slot_rows[s]] = x[s / top_k].  Rows are ordered by expert and, within
 * an expert, by slot: stable and deterministic.  Ids outside [0, num_experts) are dropped: slot_rows[s] = -1, and sorted rows
 * offsets[num_experts] .. T * top_k - 1 are not written (the grouped calls, given total_rows = T * top_k, leave them unwritten
 * too).  x is [num_tokens, K] of a_dtype (float16 | bfloat16), K % 8 == 0; 1 <= num_experts <= BB_GROUPED_MAX_GROUPS, top_k >= 1,
 * T * top_k < 2^31.  ONE launch, no workspace, no host synchronisation (CUDA-graph capturable); programmatic stream serialization,
 * nothing read before the preceding kernel has completed.  num_tokens == 0 validates and returns 0 without touching the device. */
int bb_moe_route(const int32_t* topk_ids, int num_tokens, int top_k, int num_experts, const void* x, int a_dtype, int K,
                 int32_t* offsets, int32_t* slot_rows, void* x_sorted, void* stream);

/* bb_moe_route without the copy: offsets and slot_rows bit-identical to bb_moe_route's for the same ids, and, for every kept
 * slot s, row_token[slot_rows[s]] = s / top_k (the token whose row sorted row slot_rows[s] would hold) -- the row_index of
 * bb_matmul_grouped_gemm_swiglu_gather.  Rows offsets[num_experts] .. T * top_k - 1 of row_token are not written.  The checks of
 * bb_moe_route without those on x, K and a_dtype; the int32 arrays 4-byte aligned.  ONE launch, no workspace, graph-capturable;
 * num_tokens == 0 validates and returns 0 without touching the device. */
int bb_moe_route_index(const int32_t* topk_ids, int num_tokens, int top_k, int num_experts, int32_t* offsets,
                       int32_t* slot_rows, int32_t* row_token, void* stream);

/* Weighted top-k combine: out[t, :] = sum_j topk_weights[t, j] * Y[slot_rows[t * top_k + j], :], accumulated in fp32 over
 * j = 0 .. top_k - 1 in that order and rounded once to out_dtype (float16 | bfloat16 | float32, also the type of Y [T * top_k, N]).
 * Slots whose row is -1 or outside [0, T * top_k) add nothing; a token with no valid slot gets zeros.  No atomics: two runs are
 * bit-identical.  N % 8 == 0; Y and out 16-byte aligned.  ONE launch with programmatic stream serialization, waiting for the
 * preceding kernel first.  num_tokens == 0 validates and returns 0 without touching the device. */
int bb_moe_combine(const int32_t* slot_rows, const float* topk_weights, const void* Y, int out_dtype, void* out, int num_tokens,
                   int top_k, int N, void* stream);

/* Mixture-of-experts top-k gating: router logits [num_tokens, num_experts] (DEVICE, logits_dtype float16 | bfloat16 | float32,
 * converted to fp32) -> topk_ids int32 [T, top_k] and topk_weights float32 [T, top_k], the router output bb_moe_route and
 * bb_moe_combine read.  Per token, with l[e] the logits (expf is the full-precision fp32 exponential):
 *   1. score: scoring 0 (softmax) s[e] = expf(l[e] - max) / sum_e' expf(l[e'] - max) over every expert (NaN logits are left
 *      out of the max and the sum, and their score is NaN); scoring 1 (sigmoid) s[e] = 1 / (1 + expf(-l[e])).
 *   2. selection value v[e] = s[e] + correction_bias[e] (fp32 [num_experts], DEVICE; NULL: no bias).  The bias steers the
 *      selection only.
 *   3. group limit, num_expert_group = n > 1: the experts form n contiguous groups of num_experts / n; a group's score is the
 *      max of its v (group_score 0) or the sum of its two largest v (group_score 1, "top2_sum"); only the topk_group groups
 *      with the highest scores can be chosen.  num_expert_group <= 1: no group limit (topk_group and group_score are ignored).
 *   4. the top_k experts with the largest v, in descending order of v: slot j holds the j-th choice.  Ties go to the lower expert
 *      (or group) index, and a NaN ranks below every number.
 *   5. weights w[j] = s[id[j]] (without the bias); renormalize != 0: w[j] /= sum_j' w[j'], summed in fp32 in j order (a zero
 *      sum gives zero weights); then w[j] *= routed_scaling_factor.
 * The order is part of the result: two runs, and a CUDA-graph replay, are bit-identical.  1 <= num_experts <=
 * BB_GROUPED_MAX_GROUPS; 1 <= top_k <= min(num_experts, 32); T * top_k < 2^31; scoring 0 | 1; with a group limit n <= 32 divides
 * num_experts, 1 <= topk_group <= n, group_score 0 | 1 (1 needs num_experts / n >= 2) and top_k <= topk_group * num_experts / n;
 * routed_scaling_factor finite (code 1 otherwise, each with its own message).  logits aligned to their element size, the other
 * arrays 4-byte aligned (code 5).  ONE launch, no workspace, no host synchronisation (CUDA-graph capturable); programmatic stream
 * serialization: the logits are read only after the preceding kernel has completed, and the next kernel may launch once this
 * one has stored its results.  num_tokens == 0 validates and returns 0 without touching the device; unlike the bb_moe_route /
 * bb_moe_combine calls it is still counted in bb_launch_count, so every accepted call adds exactly one step whatever T is. */
int bb_moe_topk(const void* logits, int logits_dtype, int num_tokens, int num_experts, int top_k, int scoring,
                const float* correction_bias, int num_expert_group, int topk_group, int group_score, int renormalize,
                float routed_scaling_factor, int32_t* topk_ids, float* topk_weights, void* stream);

/* Column gather of the activations of a GPTQ act-order layer: out[r, j] = A[r, perm[e * K + j]], e the group of row r.  An act-order
 * checkpoint puts input column k in quantization group g_idx[k]; with perm = stable_argsort(g_idx) the loader sorts the weight's
 * K axis into the contiguous group layout the matmuls read, and y = A[:, perm] x W_sorted^T.  A and out are [rows, K] of a_dtype
 * (float16 | bfloat16; the values are moved, not converted), both 16-byte aligned; K % 8 == 0 and K <= 112640.
 *   - num_groups == 1, offsets == NULL: perm [K] (DEVICE int32) applies to every row (a dense layer).
 *   - offsets (DEVICE int32 [num_groups + 1], the offset contract of bb_matmul_grouped): perm is [num_groups, K] and group e owns
 *     rows [offsets[e], offsets[e + 1]).  Offsets are clamped to [0, rows], a group whose end is below its start is empty, and rows
 *     no group claims are not written.
 * Perm values are clamped to [0, K - 1], so every read stays inside A's row.  perm and offsets 4-byte aligned (code 5 otherwise,
 * as for A and out).  1 <= num_groups <= BB_GROUPED_MAX_GROUPS.  ONE launch, no workspace, no host synchronisation
 * (CUDA-graph capturable); programmatic stream serialization: offsets and A are read only after the preceding kernel has
 * completed, and the next kernel may launch once this one has stored its rows.  rows == 0 validates and
 * returns 0 without touching the device.  Callers of bb_matmul on an act-order weight gather A with this call first. */
int bb_permute_cols(const void* A, void* out, const int32_t* perm, int rows, int K, int a_dtype, int num_groups,
                    const int32_t* offsets, void* stream);

/* Cross-rank barrier for the column-parallel path (no reference counterpart): rank `rank` of `n_peers` signals every peer and
 * waits for all of them, on `stream`, as ONE small kernel -- ordered after the preceding kernels' peer stores (it is launched as a
 * programmatic dependent and waits for them), so after it every rank may read what bb_matmul_scatter calls issued before it wrote.
 * peer_flags[i] = device pointer to rank i's flag block in peer-mapped (symmetric) memory, BB_PEER_FLAG_BYTES each, zeroed
 * once before first use; every rank must call it the same number of times.  CUDA-graph capturable (sequence numbers live in the
 * flag block, not in the launch parameters).  A peer that never arrives traps the kernel after ~10 s instead of hanging. */
#define BB_PEER_FLAG_BYTES 128
int bb_peer_barrier(void* const* peer_flags, int n_peers, int rank, void* stream);

/* scratch (the m = 1 slab kernel's tagged partial-sum slots; the wgmma kernel's fp32 split-K partials) the chosen kernel
 * needs for this (desc, m); 0 for most configs.
 * The buffer must be ZERO-INITIALISED once by the caller before its first use (cudaMemset / torch.zeros): the slab kernel
 * exchanges partial sums through tagged slots and leaves every slot zero-tagged again when it finishes, so the same
 * buffer can then be reused by later calls ON THE SAME STREAM without clearing (calls that may run concurrently need their
 * own buffers).  The wgmma kernel's split-K partials need no clearing; they start past the slab kernel's slot region (sized
 * at the device's full SM count), so one buffer can serve every m: a split-K call never dirties the slots an m = 1 call reads. */
size_t bb_workspace_bytes(const bb_matmul_desc* desc, int m);

/* which kernel family bb_matmul would run for (desc, m) -- bb_kernel_id; <0 on invalid desc. */
int bb_select_kernel(const bb_matmul_desc* desc, int m);
const char* bb_kernel_name(int kernel_id);
/* testing hook: force a kernel family (BB_KERNEL_AUTO restores dispatch). Returns previous value. */
int bb_set_kernel_override(int kernel_id);
/* testing hook: every kernel sizes its work decomposition (grids, split-K, stream-K ranges, bb_workspace_bytes) as if the device
 * had min(real SM count, cap) SMs, so one device runs the partitions of smaller parts (an H100 PCIe, a MIG slice).  Kernel choice
 * (bb_select_kernel) does not depend on it.  cap = 0 removes the cap.  A cap below 0 or above the current device's SM count is
 * refused (-1, bb_last_error set, cap unchanged): a capped grid must stay resident at once.  Returns the previous cap.  Global
 * to the process; set it while no call is in flight and size workspaces after setting it. */
int bb_set_sm_count_cap(int cap);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches counter). */
uint64_t bb_launch_count(void);

const char* bb_last_error(void);
int bb_version(void);

/* ---- weight pre-processing (replaces the TVM-LLVM CPU ops QuantCompress / LOP3Permutate,
 * bitblas/ops/quant_compress/quant_compress_impl.py:22-30, bitblas/ops/lop3_permutate/lop3_permutate_impl.py:27-34,
 * chained by OPExecutorCPU, bitblas/ops/operator.py:529-556) ---- */

/* host: in[rows, cols] one value per int8 -> out[rows, cols*bits/8] */
int bb_compress_host(const int8_t* in, int8_t* out, int64_t rows, int64_t cols, int bits);
/* host: per-int32-word LOP3 interleave; target_bits = 16 (f16/bf16 A) or 8 (int8 A) */
int bb_interleave_host(const int8_t* in, int8_t* out, int64_t nbytes, int bits, int target_bits);
/* device: fused compress (+ interleave if target_bits != 0) of w[rows, cols] int8 -> out[rows, cols*bits/8] */
int bb_transform_weight_device(const int8_t* w, int8_t* out, int64_t rows, int64_t cols, int bits,
                               int target_bits, void* stream);
/* device: GPTQ ingest (bitblas/module/__init__.py:24-74,315-363).  qweight_gptq is int32 [K*bits/32, N]
 * (GPTQ layout); writes BitBLAS layout out[N, K*bits/8] (compressed + optional interleave). */
int bb_repack_gptq_qweight_device(const int32_t* qweight_gptq, int8_t* out, int64_t K, int64_t N, int bits,
                                  int target_bits, void* stream);
/* device: GPTQ qzeros int32 [K/g, N*bits/32] -> unpacked (+1 unless v2, & mask) transposed int8 [N, K/g]
 * as A_dtype-typed `zeros_out` (mode original: value; rescale: value*scale) or re-packed [K/g, N*bits/8]
 * (mode quantized).  scales is [N, K/g] in a_dtype (already transposed). */
int bb_repack_gptq_qzeros_device(const int32_t* qzeros_gptq, const void* scales, void* zeros_out, int64_t groups,
                                 int64_t N, int bits, int zeros_mode, int a_dtype, int v2, void* stream);

/* device: BB_TILE_SLAB re-tiling of a stored weight matrix (either layout of bb_wlayout): in[rows, row_bytes] row-major ->
 * out as [rows/32][row_bytes/512][32][512] (inverse != 0: back to row-major).  in != out.  rows % 32 == 0, row_bytes % 512 == 0. */
int bb_retile_weight_device(const int8_t* in, int8_t* out, int64_t rows, int64_t row_bytes, int inverse, void* stream);

/* ---- test hook: run the library's own in-register decode over an array of packed words (device ptrs).
 * kind: 0 = to f16 (8 values / group), 1 = to bf16, 2 = to int8 (16 values / group).  Used by the GPU KATs
 * that compare against the reference's device decode functions (oracle/ref_shim.cu). ---- */
int bb_debug_decode(int kind, int bits, int is_signed, int w_layout, const void* in, void* out, int ngroups,
                    void* stream);

/* test hook: the tensor-core GEMM path's dequantise arithmetic -- decode, then ((w - zp) [- z]) * s in A_dtype with the
 * reference's rounding order (bitblas/gpu/intrin/lop3.py:172-175,256,269) -- over an array of packed 32-bit words.
 * kind: 0 = f16, 1 = bf16; mode: 0 none, 1 scale, 2 zeros "original", 3 zeros "rescale", 4 quantized zeros (qzeros: int32).
 * One (scale, zeros, qzeros) entry per group of 8 outputs, like the reference's decode_*_scale[_zeros_*] device functions
 * (testing/cpp/lop3_type_conversion/fast_decoding.hpp), which tests/test_gpu_decode_kat.py runs side by side. */
int bb_debug_dequant(int kind, int bits, int is_signed, int w_layout, int mode, const void* in, const void* scale,
                     const void* zeros, const void* qzeros, void* out, int nwords, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BITBLAS_B200_H_ */
