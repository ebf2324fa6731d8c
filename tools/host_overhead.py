"""Host-side cost per call of Matmul.forward / forward_scatter / Linear.forward / GroupedLinear.forward (tiny problem: the GPU kernel
takes ~5 us, so the wall time of a long unsynchronised loop is the CPU launch path)."""
import os, sys, time, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bb
dev = "cuda"
N = K = 256
cfg = bb.MatmulConfig(M=1, N=N, K=K, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
op = bb.Matmul(cfg, enable_tuning=False)
W = torch.randint(-128, 128, (N, K // 2), dtype=torch.int8, device=dev)
sc = (torch.rand(N, K // 128, device=dev) * 0.02).half()
qz = torch.randint(-128, 128, (K // 128, N // 2), dtype=torch.int8, device=dev)
A = (torch.rand(1, K, device=dev) - 0.5).half()
out = torch.empty(1, N, dtype=torch.float16, device=dev)
def bench(f, n=2000):
    for _ in range(50): f()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n): f()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    return (t1 - t0) / n * 1e6
print("forward            us/call", round(bench(lambda: op.forward(A, W, scale=sc, zeros=qz, output=out)), 2))
ptrs = [out.data_ptr()]
print("forward_scatter    us/call", round(bench(lambda: op.forward_scatter(A, W, scale=sc, zeros=qz, peer_ptrs=ptrs, ldc=N, col_offset=0)), 2))
kw = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
lin = bb.Linear(K, N, opt_M=[1], **kw).cuda()
print("Linear.forward     us/call", round(bench(lambda: lin(A, output=out)), 2))
gl, xg, off = bb.GroupedLinear(8, K, N, **kw).cuda(), A.expand(8, K).contiguous(), torch.arange(9, dtype=torch.int32, device=dev)
print("GroupedLinear 8x1  us/call", round(bench(lambda: gl(xg, off)), 2))
hA = torch.empty((1, K), dtype=torch.float16).pin_memory()
hC = torch.empty((1, N), dtype=torch.float16).pin_memory()
print("h2d copy_          us/call", round(bench(lambda: A.copy_(hA, non_blocking=True)), 2))
print("d2h copy_          us/call", round(bench(lambda: hC.copy_(out, non_blocking=True)), 2))
print("current_stream     us/call", round(bench(lambda: torch.cuda.current_stream(device=A.device).cuda_stream), 2))
