"""Isolated timings of the non-GEMM kernels at north-star shapes.

  python tools/kernel_bench.py                       all kernels
  python tools/kernel_bench.py --only groupnorm_stats [--baseline-lib OTHER.so]

--baseline-lib: a libdwm_b200.so built from another revision; its dwm_b200_groupnorm_stats is
timed alternately with this tree's at the same shapes, and the two results compared."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from opendwm_b200 import ops


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


# GroupNorm statistics shapes (nb, pixels, C): the four CTSD-2.1 UNet levels at 256 x 448 (12
# volumes: 2 CFG branches x 6 views), and the 2-D VAE decoder's largest frame (6 views,
# 256 x 448 pixels, 128 channels)
GN_SHAPES = [(12, 32 * 56, 320), (12, 16 * 28, 640), (12, 8 * 14, 1280), (12, 4 * 7, 2560),
             (6, 256 * 448, 128)]


def _device_info():
    """(card name, power limit) of GPU 0, read-only query."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def groupnorm_stats_bench(baseline_lib=None, rounds=5):
    """ms per call of dwm_b200_groupnorm_stats (this tree, and `baseline_lib` alternately) and the
    largest |difference| of the two results, per shape."""
    from opendwm_b200 import lib
    libs = {"this": lib.load()}
    if baseline_lib:
        other = ctypes.CDLL(baseline_lib)
        other.dwm_b200_groupnorm_stats.restype = ctypes.c_int
        other.dwm_b200_groupnorm_stats.argtypes = lib.SYMBOLS["dwm_b200_groupnorm_stats"][1]
        libs["baseline"] = other
    out = {"device": _device_info()}
    for nb, pixels, C in GN_SHAPES:
        x = torch.randn(nb, pixels, C, device="cuda") * 2 + 0.5
        sums = {k: torch.empty(nb, 32, 2, device="cuda", dtype=torch.float64) for k in libs}

        def call(h, s):
            return lambda: lib.check(h.dwm_b200_groupnorm_stats(
                x.data_ptr(), nb, pixels, C, 32, s.data_ptr(), torch.cuda.current_stream().cuda_stream),
                "dwm_b200_groupnorm_stats")

        fns = {k: call(libs[k], sums[k]) for k in libs}
        times = {k: [] for k in libs}
        for _ in range(rounds):                       # alternate the versions
            for k, f in fns.items():
                times[k].append(timeit(f, iters=50, warm=5))
        r = {"gbs_this": x.numel() * 4 / min(times["this"]) / 1e6}
        for k, t in times.items():
            r["ms_" + k] = sorted(t)[len(t) // 2]
            r["ms_%s_range" % k] = [min(t), max(t)]
        if "baseline" in sums:
            r["max_abs_diff"] = (sums["this"] - sums["baseline"]).abs().max().item()
        out["%dx%dx%d" % (nb, pixels, C)] = r
        print("groupnorm_stats", nb, pixels, C, r, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["groupnorm_stats"])
    ap.add_argument("--baseline-lib")
    a = ap.parse_args()
    if a.only == "groupnorm_stats":
        res = groupnorm_stats_bench(a.baseline_lib)
        os.makedirs("bench_out", exist_ok=True)
        json.dump(res, open("bench_out/kernel_bench_groupnorm_stats.json", "w"), indent=1)
        return
    res = {}
    D, heads, N, S, L = 1536, 24, 192, 448, 154
    dt = torch.bfloat16
    # joint attention
    qkv = torch.randn(N * (S + L), 3 * D, device="cuda").to(dt)
    o = torch.empty(N * S, D, device="cuda", dtype=dt)
    o2 = torch.empty(N * L, D, device="cuda", dtype=dt)
    f = lambda: ops.attention(qkv, o, D=D, heads=heads, group_dims=[N], group_strides=[S + L],
                              seq=S + L, out_group_strides=[S], out_stride_outer=0,
                              out_stride_inner=1, split=S, out2=o2)
    from opendwm_b200 import lib
    fl = 4.0 * (S + L) ** 2 * D * N
    qs = torch.randn(N * S, 3 * D, device="cuda").to(dt)
    f2 = lambda: ops.attention(qs, o, D=D, heads=heads, group_dims=[N], group_strides=[S], seq=S)
    t = timeit(f)
    res["joint_attention_tc2"] = dict(ms=t, tflops=fl / t / 1e9)
    t = timeit(f2)
    res["dual_attention_tc2"] = dict(ms=t, tflops=4.0 * S * S * D * N / t / 1e9)
    # cross-view row-wise (bt h) x (v w) = 512 x 168 with the ring view mask: gathered wgmma
    # kernel vs the mma.sync kernel; HBM floor = q|k|v read + out written
    Bc, Tc, Vc, Hp, Wp = 2, 16, 6, 16, 28
    ring = torch.zeros(Vc, Vc, dtype=torch.uint8)
    for i in range(Vc):
        for d in (-1, 0, 1):
            ring[i, (i + d) % Vc] = 1
    mask = ring.unsqueeze(0).repeat(Bc, 1, 1).cuda().contiguous()
    fcv = lambda: ops.attention(qs, o, D=D, heads=heads, group_dims=[Bc * Tc, Hp],
                                group_strides=[Vc * S, Wp], seq=Vc * Wp, inner=Wp,
                                stride_outer=S, stride_inner=1, mask=mask, mask_div=Tc)
    byts = qs.numel() * 2 + o.numel() * 2
    for variant, tag in ((0, "_mma"), (2, "_tc2")):
        lib.set_option("attn_tc", variant)
        t = timeit(fcv)
        res["crossview_attention" + tag] = dict(ms=t, gbs=byts / t / 1e6,
                                                tflops=4.0 * (Vc * Wp) ** 2 * 64 * heads * Bc * Tc * Hp / t / 1e9)
    lib.set_option("attn_tc", -1)
    # out-projection RESID GEMM (86016 x 1536 x 1536, gated, in place): TMA L2 prefetch of the residual
    # vs none
    xr = torch.randn(N * S, D, device="cuda")
    wo = (torch.randn(D, D, device="cuda") * 0.02).to(dt)
    bo = torch.zeros(D, device="cuda")
    gate = torch.randn(N, D, device="cuda")
    o16 = torch.randn(N * S, D, device="cuda").to(dt)
    fr = lambda: ops.linear(o16, wo, bo, epilogue=lib.EPI_RESID, resid=xr, out=xr, gate=gate,
                            rows_per_item=S)
    g16 = torch.randn(N * S, 4 * D, device="cuda").to(dt)
    w2 = (torch.randn(D, 4 * D, device="cuda") * 0.01).to(dt)
    fr2 = lambda: ops.linear(g16, w2, bo, epilogue=lib.EPI_RESID, resid=xr, out=xr, gate=gate,
                             rows_per_item=S)
    for variant, tag in ((0, "_regs"), (1, "_tma")):
        lib.set_option("resid_tma", variant)
        t = timeit(fr)
        res["resid_gemm_k1536" + tag] = dict(ms=t, tflops=2.0 * N * S * D * D / t / 1e9)
        t = timeit(fr2)
        res["resid_gemm_k6144" + tag] = dict(ms=t, tflops=2.0 * N * S * D * 4 * D / t / 1e9)
    lib.set_option("resid_tma", 1)
    del g16, w2, o16, xr
    # temporal pointwise (B'=2, T=16, V=6)
    B, T, V = 2, 16, 6
    f = lambda: ops.attention(qs, o, D=D, heads=heads, group_dims=[B, V * S],
                              group_strides=[T * V * S, 1], seq=T, inner=1, stride_outer=V * S,
                              stride_inner=0)
    t = timeit(f)
    res["temporal_attention"] = dict(ms=t, gbs=(qs.numel() * 2 + o.numel() * 2) / t / 1e6)
    # layernorm
    x = torch.randn(N * S, D, device="cuda")
    a16 = torch.empty(N * S, D, device="cuda", dtype=dt)
    mod = torch.randn(N, 6 * D, device="cuda")
    f = lambda: ops.layernorm(x, a16, eps=1e-6, rows_per_item=S, shift=mod[:, :D], scale=mod[:, D:2 * D])
    for staged, tag in ((1, ""), (0, "_resident")):
        lib.set_option("ln_staged", staged)
        t = timeit(f)
        res["layernorm_mod" + tag] = dict(ms=t, gbs=(x.numel() * 4 + a16.numel() * 2) / t / 1e6)
    lib.set_option("ln_staged", 1)
    w, b = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    y = torch.empty_like(x)
    emb = torch.randn(N, D, device="cuda")
    f = lambda: ops.layernorm(x, a16, weight=w, bias=b, add_item=emb, rows_per_item=S, sum_out=y)
    t = timeit(f)
    res["layernorm_affine_sum"] = dict(ms=t, gbs=(x.numel() * 8 + a16.numel() * 2) / t / 1e6)
    del x, y, a16, qkv, qs, o, o2
    res["groupnorm_stats"] = groupnorm_stats_bench(a.baseline_lib)
    for k, v in res.items():
        print(k, v, flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(res, open("bench_out/kernel_bench.json", "w"), indent=1)


if __name__ == "__main__":
    main()
