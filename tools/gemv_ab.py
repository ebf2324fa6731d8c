"""Timing of the m<=8 streaming kernels over a few (N, K) (AB_SHAPES=NxK,..., AB_M=1,2,...): cold L2 by rotating over weight
copies that exceed L2; back-to-back launches."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bb
dev = "cuda"
shapes = [(12288, 12288), (9472, 12288), (14208, 12288), (8192, 8192), (28672, 8192), (8192, 28672), (10240, 8192)]
if os.environ.get("AB_SHAPES"):
    shapes = [tuple(int(v) for v in t.split("x")) for t in os.environ["AB_SHAPES"].split(",")]
reps_env = int(os.environ.get("AB_REPS", "60"))
ms = [int(x) for x in os.environ.get("AB_M", "1").split(",")]
for (N, K) in shapes:
    for m in ms:
        cfg = bb.MatmulConfig(M=1, N=N, K=K, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
                              with_zeros=True, zeros_mode="quantized")
        op = bb.Matmul(cfg, enable_tuning=False)
        ncopy = max(3, int(400e6 // (N * K // 2)) + 1)
        Ws = [torch.randint(-128, 128, (N, K // 2), dtype=torch.int8, device=dev) for _ in range(ncopy)]
        sc = (torch.rand(N, K // 128, device=dev) * 0.02).half()
        qz = torch.randint(-128, 128, (K // 128, N // 2), dtype=torch.int8, device=dev)
        A = (torch.rand(m, K, device=dev) - 0.5).half()
        out = torch.empty(m, N, dtype=torch.float16, device=dev)
        for w in Ws: op.forward(A, w, scale=sc, zeros=qz, output=out)
        torch.cuda.synchronize()
        reps = reps_env
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(reps): op.forward(A, Ws[i % ncopy], scale=sc, zeros=qz, output=out)
        e.record(); torch.cuda.synchronize()
        us = s.elapsed_time(e) / reps * 1000
        byt = N * K / 2 + N * (K // 128) * 2.5 + m * K * 2 + m * N * 2
        print(f"N={N} K={K} m={m} {us:.1f} us  {byt / us / 1e3:.0f} GB/s  kernel={op.kernel_for(m)}", flush=True)
        del Ws
