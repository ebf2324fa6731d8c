// oracle/ref_shim.cu -- TEST INFRASTRUCTURE ONLY.
//
// Thin extern "C" wrappers around the REFERENCE's own C++/CUDA decode test header, compiled from the
// source where it lies ($BITBLAS_REFERENCE_DIR/testing/cpp/lop3_type_conversion/fast_decoding.hpp) by
// oracle/build_ref.py into oracle/_ref/libbitblas_ref.so (git-ignored).
// No reference source is copied here: this file only #includes the header and calls into it.
//
//   host  : ref_general_compress / ref_general_interleave_fp16 / ref_general_interleave_int8
//           (fast_decoding.hpp:15-28, 30-95, 607-668) -> pin oracle/bitblas_oracle.py on CPU
//   device: ref_decode_f16(kind,...) / ref_decode_i8(kind,...) run the reference's LOP3 device decode
//           functions over an array of words -> pin bitblas_b200's own decode on the GPU box.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include "fast_decoding.hpp"

extern "C" {

void ref_general_compress(const int8_t* lowbit, int8_t* compressed, int nbit, int n, int is_signed) {
  general_compress(lowbit, compressed, nbit, n, is_signed != 0);
}
void ref_general_interleave_fp16(const int8_t* in, int8_t* out, int nbit, size_t size_in_bytes) {
  general_interleave_fp16(const_cast<int8_t*>(in), out, nbit, size_in_bytes, false);
}
void ref_general_interleave_int8(const int8_t* in, int8_t* out, int nbit, size_t size_in_bytes) {
  general_interleave_int8(const_cast<int8_t*>(in), out, nbit, size_in_bytes, false);
}

}  // extern "C"

// kind ids for ref_decode_f16 (8 outputs per input group)
enum {
  K_I4U = 0, K_I4S = 1, K_I2U = 2, K_I2S = 3, K_I1U = 4, K_I1S = 5,
  K_I4U_SCALE = 6, K_I4U_ZEROS_ORIGINAL = 7, K_I4U_ZEROS_RESCALE = 8, K_I4U_ZEROS_QUANTIZED = 9,
  K_I2U_SCALE = 10, K_I2U_ZEROS_ORIGINAL = 11, K_I2U_ZEROS_RESCALE = 12,
};

// in: packed+interleaved bytes; each group of 8 outputs consumes (nbit) bytes.
__global__ void ref_decode_f16_kernel(int kind, const int8_t* in, half* out, int ngroups, const half* scale,
                                      const half* zeros, const int* qzeros) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ngroups) return;
  half local[8];
  half s = scale ? scale[g] : __float2half(1.f);
  half z = zeros ? zeros[g] : __float2half(0.f);
  int qz = qzeros ? qzeros[g] : 0;
  switch (kind) {
    case K_I4U: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4u_to_f16(p, local); break; }
    case K_I4S: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4s_to_f16(p, local); break; }
    case K_I2U: { int8_t* p = const_cast<int8_t*>(in) + 2 * g; decode_i2u_to_f16(p, local); break; }
    case K_I2S: { int8_t* p = const_cast<int8_t*>(in) + 2 * g; decode_i2s_to_f16(p, local); break; }
    case K_I1U: { int8_t* p = const_cast<int8_t*>(in) + 1 * g; decode_i1u_to_f16(p, local); break; }
    case K_I1S: { int8_t* p = const_cast<int8_t*>(in) + 1 * g; decode_i1s_to_f16(p, local); break; }
    case K_I4U_SCALE: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4u_to_f16_scale(p, local, &s); break; }
    case K_I4U_ZEROS_ORIGINAL: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4u_to_f16_scale_zeros_original(p, local, &s, &z); break; }
    case K_I4U_ZEROS_RESCALE: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4u_to_f16_scale_zeros_rescale(p, local, &s, &z); break; }
    case K_I4U_ZEROS_QUANTIZED: { int8_t* p = const_cast<int8_t*>(in) + 4 * g; decode_i4u_to_f16_scale_zeros_quantized(p, local, &s, &qz); break; }
    case K_I2U_SCALE: { int8_t* p = const_cast<int8_t*>(in) + 2 * g; decode_i2u_to_f16_scale(p, local, &s); break; }
    case K_I2U_ZEROS_ORIGINAL: { int8_t* p = const_cast<int8_t*>(in) + 2 * g; decode_i2u_to_f16_scale_zeros_original(p, local, &s, &z); break; }
    case K_I2U_ZEROS_RESCALE: { int8_t* p = const_cast<int8_t*>(in) + 2 * g; decode_i2u_to_f16_scale_zeros_rescale(p, local, &s, &z); break; }
    default: return;
  }
  for (int i = 0; i < 8; ++i) out[8 * g + i] = local[i];
}

enum { K8_I4U = 0, K8_I4S = 1, K8_I2U = 2, K8_I2S = 3, K8_I1U = 4, K8_I1S = 5 };

// 16 int8 outputs per group; group consumes 2*nbit bytes.
__global__ void ref_decode_i8_kernel(int kind, const int8_t* in, int8_t* out, int ngroups) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ngroups) return;
  __align__(16) int8_t local[16];
  __align__(8) int8_t src[8];
  int nbytes = (kind <= K8_I4S) ? 8 : (kind <= K8_I2S ? 4 : 2);
  for (int i = 0; i < 8; ++i) src[i] = i < nbytes ? in[nbytes * g + i] : 0;
  switch (kind) {
    case K8_I4U: decode_i4u_to_i8s(src, local); break;
    case K8_I4S: decode_i4s_to_i8s(src, local); break;
    case K8_I2U: decode_i2u_to_i8s(src, local); break;
    case K8_I2S: decode_i2s_to_i8s(src, local); break;
    case K8_I1U: decode_i1u_to_i8s(src, local); break;
    case K8_I1S: decode_i1s_to_i8s(src, local); break;
    default: return;
  }
  for (int i = 0; i < 16; ++i) out[16 * g + i] = local[i];
}

extern "C" {

// All pointers are DEVICE pointers. Returns cudaError_t as int.
int ref_decode_f16(int kind, const void* in, void* out, int ngroups, const void* scale, const void* zeros,
                   const void* qzeros, void* stream) {
  int threads = 128, blocks = (ngroups + threads - 1) / threads;
  ref_decode_f16_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(
      kind, (const int8_t*)in, (half*)out, ngroups, (const half*)scale, (const half*)zeros, (const int*)qzeros);
  return (int)cudaGetLastError();
}
int ref_decode_i8(int kind, const void* in, void* out, int ngroups, void* stream) {
  int threads = 128, blocks = (ngroups + threads - 1) / threads;
  ref_decode_i8_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(kind, (const int8_t*)in, (int8_t*)out, ngroups);
  return (int)cudaGetLastError();
}

}  // extern "C"
