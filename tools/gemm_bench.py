"""Times dwm_b200_linear at the north-star GEMM shapes against torch.matmul (cuBLASLt)."""
import json
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from opendwm_b200 import ops, lib


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None
    shapes = [(86016, 12288, 1536, "geglu"), (86016, 1536, 6144, "resid"),
              (86016, 4608, 1536, "qknorm"), (86016, 1536, 1536, "resid"),
              (86016, 6144, 1536, "store"), (29568, 4608, 1536, "store"),
              (8192, 8192, 8192, "store")]
    res = []
    if only:
        shapes = [s for s in shapes if s[3] == only][:1]
    for M, N, K, epi in shapes:
        a = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.03).bfloat16()
        kw = {}
        if epi == "geglu":
            kw = dict(epilogue=lib.EPI_GEGLU)
        elif epi == "resid":
            r = torch.randn(M, N, device="cuda")
            kw = dict(epilogue=lib.EPI_RESID, resid=r, out=r)
        elif epi == "qknorm":
            qw = torch.ones(64, device="cuda")
            kw = dict(epilogue=lib.EPI_QKNORM, q_norm_weight=qw, k_norm_weight=qw, qk_region=N // 3)
        out = ops.linear(a, w, **kw)
        kw.setdefault("out", out)
        lib.set_option("gemm_2cta", 0)
        t = timeit(lambda: ops.linear(a, w, **kw))
        lib.set_option("gemm_2cta", 1)
        t2 = timeit(lambda: ops.linear(a, w, **kw))
        t_ref = timeit(lambda: torch.matmul(a, w.t()))
        fl = 2.0 * M * N * K
        res.append(dict(M=M, N=N, K=K, epi=epi, ms=t, tflops=fl / t / 1e9, tflops_2cta=fl / t2 / 1e9,
                        cublas_ms=t_ref, cublas_tflops=fl / t_ref / 1e9))
        print(res[-1], flush=True)
    os.makedirs("bench_out", exist_ok=True)
    with open("bench_out/gemm_bench.json", "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
