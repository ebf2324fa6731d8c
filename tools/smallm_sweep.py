import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bb
from bitblas_b200 import _lib
lib = _lib.load()
N = K = 12288
dev = "cuda"
cfg = bb.MatmulConfig(M=[1, 4096], N=N, K=K, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
op = bb.Matmul(cfg, enable_tuning=False)
Ws = [torch.randint(-128, 128, (N, K // 2), dtype=torch.int8, device=dev) for _ in range(4)]
sc = (torch.rand(N, K // 128, device=dev) * 0.02).half()
qz = torch.randint(-128, 128, (K // 128, N // 2), dtype=torch.int8, device=dev)
def t(m, override):
    A = (torch.rand(m, K, device=dev) - 0.5).half()
    out = torch.empty(m, N, dtype=torch.float16, device=dev)
    prev = lib.bb_set_kernel_override(override)
    try:
        for w in Ws: op.forward(A, w, scale=sc, zeros=qz, output=out)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(40): op.forward(A, Ws[i % 4], scale=sc, zeros=qz, output=out)
        e.record(); torch.cuda.synchronize()
        return s.elapsed_time(e) / 40 * 1000
    except Exception as ex:
        return str(ex)[:80]
    finally:
        lib.bb_set_kernel_override(prev)
for m in (1, 2, 4, 8, 9, 16, 24, 32, 48, 64, 96, 128, 256, 512, 1024):
    r = {"m": m}
    if m <= 32: r["gemv_mma_us"] = t(m, _lib.BB_KERNEL_GEMV_MMA)
    r["gemm_ts_us"] = t(m, _lib.BB_KERNEL_GEMM_TS)
    print(r, flush=True)
