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
  BB_I32 = 4
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
  BB_KERNEL_GEMV_STREAMK = 6,/* m <= 2, 4-bit W: persistent stream-K + TMA rings; opt-in through
                              * bb_set_kernel_override only */
  BB_KERNEL_GEMV_SLAB = 7    /* m == 1, 4-bit W, fp16/bf16 A: per-CTA TMA slabs + CTA-level stream-K; the default
                              * decode kernel (needs the zero-initialised workspace of bb_workspace_bytes) */
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

/* Cross-rank barrier for the column-parallel path (no reference counterpart): rank `rank` of `n_peers` signals every peer and
 * waits for all of them, on `stream`, as ONE small kernel -- ordered after the preceding kernels' peer stores (it is launched as a
 * programmatic dependent and waits for them), so after it every rank may read what bb_matmul_scatter calls issued before it wrote.
 * peer_flags[i] = device pointer to rank i's flag block in peer-mapped (symmetric) memory, BB_PEER_FLAG_BYTES each, zeroed
 * once before first use; every rank must call it the same number of times.  CUDA-graph capturable (sequence numbers live in the
 * flag block, not in the launch parameters).  A peer that never arrives traps the kernel after ~10 s instead of hanging. */
#define BB_PEER_FLAG_BYTES 128
int bb_peer_barrier(void* const* peer_flags, int n_peers, int rank, void* stream);

/* scratch (fp32 split-K partials; stream-K slots + flags) the chosen kernel needs for this (desc, m); 0 for most configs.
 * The buffer must be ZERO-INITIALISED once by the caller before its first use (cudaMemset / torch.zeros): the stream-K
 * kernels exchange partial sums through tagged slots and leave every slot zero-tagged again when they finish, so the same
 * buffer can then be reused by later calls ON THE SAME STREAM without clearing (calls that may run concurrently need their
 * own buffers).  The split-K partials of the wgmma kernel carry no such requirement. */
size_t bb_workspace_bytes(const bb_matmul_desc* desc, int m);

/* which kernel family bb_matmul would run for (desc, m) -- bb_kernel_id; <0 on invalid desc. */
int bb_select_kernel(const bb_matmul_desc* desc, int m);
const char* bb_kernel_name(int kernel_id);
/* testing hook: force a kernel family (BB_KERNEL_AUTO restores dispatch). Returns previous value. */
int bb_set_kernel_override(int kernel_id);
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
