// tools/membench.cu -- load-pattern microbenchmark used to size the GEMV kernel's weight stream.
// Every variant reads the same N x (K/2)-byte packed-weight matrix exactly once and XOR-reduces it.
//   linear   : each warp reads 512 contiguous bytes per instruction (grid-stride)                       [upper bound]
//   rows16   : GEMV pattern: a warp owns 16 rows x a K range, lane (r,q) reads 16 B at row r/r+8, 64 B per row per
//              step, register prefetch depth D (plain ld.global.nc)
//   rows16cp : same addresses, cp.async ring of D stages into shared memory
//   rowsB    : like rows16cp but each step issues `B` consecutive 64 B pieces per row (B*64 contiguous bytes per row)
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint4 ldg_nc(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void cp16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void k_linear(const uint4* __restrict__ w, size_t n16, unsigned* out) {
  unsigned acc = 0;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
#pragma unroll 4
  for (; i < n16; i += stride) { uint4 v = ldg_nc(w + i); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
  if (acc == 0x12345678u) out[0] = acc;
}

// warp -> (row block rb, k split): 16 rows, steps [s0, s1); step = 64 B per row
template <int D>
__global__ void k_rows16(const uint8_t* __restrict__ w, int N, int row_bytes, int ks, unsigned* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
  const int steps = row_bytes / 64;
  const int per = steps / ks, s0 = warp * per, ns = per;
  const uint8_t* pa = w + (size_t)(rb * 16 + r) * row_bytes + q * 16 + (size_t)s0 * 64;
  const uint8_t* pb = pa + (size_t)8 * row_bytes;
  unsigned acc = 0;
  uint4 qa[D], qb[D];
#pragma unroll
  for (int i = 0; i < D; ++i) { qa[i] = ldg_nc(pa + (size_t)min(i, ns - 1) * 64); qb[i] = ldg_nc(pb + (size_t)min(i, ns - 1) * 64); }
  for (int s = 0; s < ns; s += D) {
#pragma unroll
    for (int i = 0; i < D; ++i) {
      uint4 a = qa[i], b = qb[i];
      const int nx = min(s + i + D, ns - 1);
      qa[i] = ldg_nc(pa + (size_t)nx * 64); qb[i] = ldg_nc(pb + (size_t)nx * 64);
      acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w;
    }
  }
  if (acc == 0x12345678u) out[0] = acc;
}

// cp.async version; B = consecutive 64-byte pieces per row issued per "macro step"; D = macro steps in the ring
template <int D, int B>
__global__ void k_rowscp(const uint8_t* __restrict__ w, int N, int row_bytes, int ks, unsigned* out) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
  const int msteps = row_bytes / (64 * B);
  const int per = msteps / ks, s0 = warp * per, ns = per;
  const uint8_t* pa = w + (size_t)(rb * 16 + r) * row_bytes + q * 16 + (size_t)s0 * 64 * B;
  const uint8_t* pb = pa + (size_t)8 * row_bytes;
  constexpr int STAGE = 1024 * B;
  const uint32_t slot = (uint32_t)__cvta_generic_to_shared(smem) + warp * (D * STAGE) + lane * 16;
  unsigned acc = 0;
  auto issue = [&](int ms, int st) {
    if (ms < ns) {
#pragma unroll
      for (int j = 0; j < B; ++j) {
        cp16(slot + st * STAGE + j * 1024, pa + (size_t)ms * 64 * B + j * 64);
        cp16(slot + st * STAGE + j * 1024 + 512, pb + (size_t)ms * 64 * B + j * 64);
      }
    }
    cp_commit();
  };
#pragma unroll
  for (int i = 0; i < D - 1; ++i) issue(i, i);
  int st = 0, stw = D - 1;
  for (int s = 0; s < ns; ++s) {
    issue(s + D - 1, stw);
    cp_wait<D - 1>();
#pragma unroll
    for (int j = 0; j < 2 * B; ++j) {
      uint4 v;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(slot + st * STAGE + j * 512));
      acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    st = st + 1 == D ? 0 : st + 1;
    stw = stw + 1 == D ? 0 : stw + 1;
  }
  if (acc == 0x12345678u) out[0] = acc;
}


// hypothesis test: the same register-queue weight stream (D=4) plus, per step, 64 B of "activations" per lane quad that
// are consumed immediately.  MODE 0: none, 1: ld.global (L1-hit) right when needed, 2: ld.shared from a slice staged once
// at kernel start, 3: cp.async staged one 4-step chunk ahead, read with ld.shared.
template <int MODE>
__global__ void k_rows16_act(const uint8_t* __restrict__ w, const uint8_t* __restrict__ act, int N, int row_bytes, int ks, unsigned* out) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int D = 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, q = lane & 3;
  const int rb = blockIdx.x;
  const int steps = row_bytes / 64;
  const int per = steps / ks, s0 = warp * per, ns = per;
  const uint8_t* pa = w + (size_t)(rb * 16 + r) * row_bytes + q * 16 + (size_t)s0 * 64;
  const uint8_t* pb = pa + (size_t)8 * row_bytes;
  const uint8_t* ap = act + (size_t)s0 * 256 + q * 64;  // 256 B of activations per step (128 fp16)
  unsigned acc = 0;
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  if (MODE == 2) {  // stage this warp's whole slice: ns * 256 B
    for (int i = lane; i < ns * 16; i += 32) cp16(sbase + warp * (per * 256) + i * 16, act + (size_t)s0 * 256 + i * 16);
    cp_commit(); cp_wait<0>(); __syncwarp();
  }
  const uint32_t cbase = sbase + warp * 2048;  // MODE 3: 2 chunks x 4 steps x 256 B
  auto stage_chunk = [&](int c) {              // chunk c = steps [4c, 4c+4): 1 KB = 64 pieces of 16 B, 2 per lane
    if (4 * c < ns) {
      cp16(cbase + (c & 1) * 1024 + lane * 16, act + (size_t)(s0 + 4 * c) * 256 + lane * 16);
      cp16(cbase + (c & 1) * 1024 + 512 + lane * 16, act + (size_t)(s0 + 4 * c) * 256 + 512 + lane * 16);
    }
    cp_commit();
  };
  if (MODE == 3) { stage_chunk(0); }
  // MODE 4: activations for chunk c+1 are loaded with plain ld.global into transit registers at the start of chunk c,
  // stored to shared memory at the start of chunk c+1 (a whole chunk later) and read with ld.shared when needed.
  uint4 tr0 = make_uint4(0, 0, 0, 0), tr1 = tr0;
  auto transit_load = [&](int c) {
    if (4 * c < ns) {
      tr0 = ldg_nc(act + (size_t)(s0 + 4 * c) * 256 + lane * 16);
      tr1 = ldg_nc(act + (size_t)(s0 + 4 * c) * 256 + 512 + lane * 16);
    }
  };
  auto transit_store = [&](int c) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(cbase + (c & 1) * 1024 + lane * 16), "r"(tr0.x), "r"(tr0.y), "r"(tr0.z), "r"(tr0.w));
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(cbase + (c & 1) * 1024 + 512 + lane * 16), "r"(tr1.x), "r"(tr1.y), "r"(tr1.z), "r"(tr1.w));
  };
  if (MODE == 4) { transit_load(0); transit_store(0); transit_load(1); __syncwarp(); }
  uint4 qa[D], qb[D];
#pragma unroll
  for (int i = 0; i < D; ++i) { qa[i] = ldg_nc(pa + (size_t)min(i, ns - 1) * 64); qb[i] = ldg_nc(pb + (size_t)min(i, ns - 1) * 64); }
  for (int s = 0; s < ns; s += D) {
    if (MODE == 3) { stage_chunk(s / 4 + 1); cp_wait<1>(); __syncwarp(); }
    if (MODE == 4 && s > 0) { __syncwarp(); transit_store(s / 4); transit_load(s / 4 + 1); __syncwarp(); }
#pragma unroll
    for (int i = 0; i < D; ++i) {
      uint4 a = qa[i], b = qb[i];
      uint4 x0, x1, x2, x3;
      if (MODE == 1) {
        const uint4* p = (const uint4*)(ap + (size_t)(s + i) * 256);
        x0 = __ldg(p); x1 = __ldg(p + 1); x2 = __ldg(p + 2); x3 = __ldg(p + 3);
      } else if (MODE == 2 || MODE == 3 || MODE == 4) {
        const uint32_t addr = MODE == 2 ? sbase + warp * (per * 256) + (s + i) * 256 + q * 64
                                        : cbase + ((s / 4) & 1) * 1024 + i * 256 + q * 64;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0.x), "=r"(x0.y), "=r"(x0.z), "=r"(x0.w) : "r"(addr));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x1.x), "=r"(x1.y), "=r"(x1.z), "=r"(x1.w) : "r"(addr + 16));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x2.x), "=r"(x2.y), "=r"(x2.z), "=r"(x2.w) : "r"(addr + 32));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x3.x), "=r"(x3.y), "=r"(x3.z), "=r"(x3.w) : "r"(addr + 48));
      } else { x0 = x1 = x2 = x3 = make_uint4(0, 0, 0, 0); }
      const int nx = min(s + i + D, ns - 1);
      qa[i] = ldg_nc(pa + (size_t)nx * 64); qb[i] = ldg_nc(pb + (size_t)nx * 64);
      // ~60 dependent-ish ALU ops to mimic the decode + MMA work of a step
      unsigned t = a.x ^ x0.x;
#pragma unroll
      for (int j = 0; j < 12; ++j) t = (t >> 3) ^ (t * 2654435761u) ^ ((j & 1) ? a.y : b.z);
      acc ^= t ^ a.z ^ a.w ^ b.x ^ b.y ^ b.w ^ x0.y ^ x1.x ^ x2.x ^ x3.x ^ x1.w ^ x2.z ^ x3.y;
    }
  }
  if (acc == 0x12345678u) out[0] = acc;
}

template <typename F>
float time_it(F f, int iters, std::vector<uint8_t*>& bufs) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) f(bufs[i % bufs.size()]);
  CK(cudaDeviceSynchronize());
  float best = 1e9f;
  for (int i = 0; i < iters; ++i) {
    cudaEventRecord(a); f(bufs[i % bufs.size()]); cudaEventRecord(b); CK(cudaEventSynchronize(b));
    float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
  }
  return best;
}

int main(int argc, char** argv) {
  const int N = argc > 1 ? atoi(argv[1]) : 12288, K = argc > 2 ? atoi(argv[2]) : 12288;
  const int row_bytes = K / 2;
  const size_t bytes = (size_t)N * row_bytes;
  std::vector<uint8_t*> bufs(5);
  for (auto& p : bufs) { CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 1, bytes)); }
  unsigned* out; CK(cudaMalloc(&out, 4));
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  auto rep = [&](const char* name, float ms) { printf("%-28s %8.2f us  %7.1f GB/s\n", name, ms * 1e3, bytes / (ms * 1e-3) / 1e9); };
  printf("N=%d K=%d bytes=%.1f MB\n", N, K, bytes / 1e6);
  for (int bpsm : {4, 8, 16}) {
    char nm[64]; snprintf(nm, 64, "linear %d x256thr/SM", bpsm);
    rep(nm, time_it([&](uint8_t* w) { k_linear<<<sms * bpsm, 256>>>((const uint4*)w, bytes / 16, out); }, 10, bufs));
  }
  for (int ks : {3}) {
    if ((row_bytes / 64) % ks) continue;
    char nm[64];
    snprintf(nm, 64, "rows16 regs D=4 ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16<4><<<N / 16, 32 * ks>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16 regs D=8 ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16<8><<<N / 16, 32 * ks>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows cp D=4 B=1 ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rowscp<4, 1><<<N / 16, 32 * ks, ks * 4 * 1024>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows cp D=8 B=1 ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rowscp<8, 1><<<N / 16, 32 * ks, ks * 8 * 1024>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    if ((row_bytes / 128) % ks == 0) {
      snprintf(nm, 64, "rows cp D=4 B=2 ks=%d", ks);
      rep(nm, time_it([&](uint8_t* w) { k_rowscp<4, 2><<<N / 16, 32 * ks, ks * 4 * 2048>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    }
    if ((row_bytes / 256) % ks == 0) {
      snprintf(nm, 64, "rows cp D=3 B=4 ks=%d", ks);
      rep(nm, time_it([&](uint8_t* w) { k_rowscp<3, 4><<<N / 16, 32 * ks, ks * 3 * 4096>>>(w, N, row_bytes, ks, out); }, 10, bufs));
    }
  }
  uint8_t* act; CK(cudaMalloc(&act, K * 2)); CK(cudaMemset(act, 3, K * 2));
  CK(cudaFuncSetAttribute(k_rows16_act<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  for (int ks : {3, 4}) {
    if ((row_bytes / 64) % ks || ((row_bytes / 64) / ks) % 4) continue;
    char nm[64];
    snprintf(nm, 64, "rows16+work act=none ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<0><<<N / 16, 32 * ks>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=LDG  ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<1><<<N / 16, 32 * ks>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=LDSall ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<2><<<N / 16, 32 * ks, K * 2>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=cpchunk ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<3><<<N / 16, 32 * ks, ks * 2048>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=transit ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<4><<<N / 16, 32 * ks, ks * 2048>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=none(2) ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<0><<<N / 16, 32 * ks>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
    snprintf(nm, 64, "rows16+work act=LDG(2) ks=%d", ks);
    rep(nm, time_it([&](uint8_t* w) { k_rows16_act<1><<<N / 16, 32 * ks>>>(w, act, N, row_bytes, ks, out); }, 10, bufs));
  }
  return 0;
}
