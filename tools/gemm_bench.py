"""Times dwm_b200_linear at the CTSD-3.5 step's GEMM shapes: the 256- and the 128-column tile,
each as the dispatcher runs it (a cluster of two CTAs for M >= 512) and forced to the 1-CTA
kernel, alternately in one process, with torch.matmul (cuBLAS) as a reference.

Every RESID / GEGLU shape is also run with the plain 16-bit STORE epilogue: the difference
bounds what the fused epilogue costs.  All variants must give the same bits; the script
checks that on every shape.  The card, its power limit and the median SM clock sampled
during the timed region are written next to the numbers (bench_out/gemm_bench.json).

    python tools/gemm_bench.py [--dtype fp16|bf16|both] [--only EPI] [--iters N] [--rounds R]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from opendwm_b200 import ops, lib  # noqa: E402
from bench import ClockSampler  # noqa: E402

# (M, N, K, epilogue): 86016 sample rows and 29568 context rows of the headline step
SHAPES = [
    (86016, 12288, 1536, "geglu"), (86016, 12288, 1536, "store"),
    (86016, 1536, 6144, "resid"), (86016, 1536, 6144, "store"),
    (86016, 1536, 1536, "resid"), (86016, 1536, 1536, "resid_blend"), (86016, 1536, 1536, "store"),
    (86016, 4608, 1536, "qknorm"), (86016, 6144, 1536, "store"),
    (29568, 4608, 1536, "qknorm"), (29568, 4608, 1536, "store"),
    # the same projections as the step runs them: into the joint q|k|v buffer, 448 sample rows
    # then 154 context rows per item, item pitch 602 rows (16-bit stores remapped per item)
    (86016, 4608, 1536, "qknorm_joint_sample"), (29568, 4608, 1536, "qknorm_joint_context"),
    (29568, 1536, 1536, "resid"), (29568, 1536, 1536, "store"),
    (29568, 6144, 1536, "store"), (29568, 1536, 6144, "resid"), (29568, 1536, 6144, "store"),
    (8192, 8192, 8192, "store"),
    # fewer tiles than SMs (either width) and a two-wave middle case, for the tile-width rule;
    # the pair threshold (M >= 512) from both sides
    (1000, 1536, 1536, "store"), (4096, 1536, 1536, "resid"),
    (256, 1536, 1536, "store"), (512, 1536, 1536, "store"), (2048, 1536, 1536, "store"),
    (8192, 1536, 1536, "store"), (16384, 1536, 1536, "store"),
    # narrow N, where the two widths differ in padding: the CTSD-2.1 UNet's level-1 and
    # level-2 transformer linears (config 2: 12 items of 32 x 56)
    (21504, 320, 320, "store"), (21504, 320, 1280, "store"), (5376, 640, 640, "store"),
]
# name -> (option gemm_bn, option gemm_2cta)
VARIANTS = {"bn256": (256, 1), "bn128": (128, 1), "bn256_1cta": (256, 0), "bn128_1cta": (128, 0)}


def select(bn, cta2):
    lib.set_option("gemm_bn", bn)
    lib.set_option("gemm_2cta", cta2)


def timeit(fn, iters, warm=2):
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, mx = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": plim, "max_sm_clock": mx}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "error": repr(e)[:200]}


def operands(M, N, K, epi, dtype):
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(dtype)
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    kw = dict(bias=b)
    if epi == "geglu":
        kw.update(epilogue=lib.EPI_GEGLU, out=torch.empty(M, N // 2, device="cuda", dtype=dtype))
    elif epi in ("resid", "resid_blend"):
        # the step's form: in place on the fp32 residual stream (blend: out = blend operand)
        r = torch.randn(M, N, device="cuda", generator=g)
        kw.update(epilogue=lib.EPI_RESID, resid=r, out=torch.empty_like(r))
        if epi == "resid_blend":
            kw.update(blend_x=kw["out"], alpha=torch.tensor([0.3, 0.9], device="cuda"),
                      rows_per_batch=M // 2)
    elif epi.startswith("qknorm"):
        qw = torch.ones(64, device="cuda")
        kw.update(epilogue=lib.EPI_QKNORM, q_norm_weight=qw, k_norm_weight=qw, qk_region=N // 3,
                  out=torch.empty(M, N, device="cuda", dtype=dtype))
        if epi.startswith("qknorm_joint"):
            S, L = 448, 154
            rpi = S if epi == "qknorm_joint_sample" else L
            kw.update(rows_per_item=rpi, out_item_stride=S + L, out_row_offset=0 if rpi == S else S,
                      out=torch.zeros(M // rpi * (S + L), N, device="cuda", dtype=dtype))
    else:
        kw.update(out=torch.empty(M, N, device="cuda", dtype=dtype))
    return a, w, kw


def run_shape(M, N, K, epi, dtype, iters, rounds):
    a, w, kw = operands(M, N, K, epi, dtype)
    out = kw["out"]
    blend = epi == "resid_blend"
    x0 = torch.randn(out.shape, device="cuda") if blend else None

    def call():
        ops.linear(a, w, **kw)

    # GEGLU always runs the 256-wide tile
    variants = {k: v for k, v in VARIANTS.items() if epi != "geglu" or v[0] == 256}
    # same bits from every variant (the blend output is reset: it is also an input)
    res = {}
    try:
        for name, (bn, cta2) in variants.items():
            select(bn, cta2)
            if blend:
                out.copy_(x0)
            call()
            res[name] = out.clone()
        identical = all(torch.equal(r, res["bn256"]) for r in res.values())
        del res
        ms = {k: [] for k in list(variants) + ["cublas"]}
        for _ in range(rounds):
            for name, (bn, cta2) in variants.items():
                select(bn, cta2)
                ms[name].append(timeit(call, iters))
            ms["cublas"].append(timeit(lambda: torch.matmul(a, w.t()), iters))
    finally:
        select(0, -1)   # the defaults: tile width by rule, pairs from DWM_GEMM_2CTA
    fl = 2.0 * M * N * K
    row = dict(M=M, N=N, K=K, epi=epi, dtype=str(dtype).split(".")[-1],
               identical_bits=identical)
    for k, v in ms.items():
        m = statistics.median(v)
        row[k + "_ms"] = m
        row[k + "_tflops"] = fl / m / 1e9
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="both", choices=["fp16", "bf16", "both"])
    ap.add_argument("--only", default=None, help="epilogue name: run only those shapes")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="bench_out/gemm_bench.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_bench needs a GPU"
    dtypes = {"fp16": [torch.float16], "bf16": [torch.bfloat16],
              "both": [torch.float16, torch.bfloat16]}[args.dtype]
    shapes = [s for s in SHAPES if args.only is None or s[3] == args.only]
    meta = card()
    print(json.dumps(meta), flush=True)
    clk = ClockSampler(torch.cuda.current_device())
    clk.start()
    rows = []
    try:
        for dtype in dtypes:
            for M, N, K, epi in shapes:
                rows.append(run_shape(M, N, K, epi, dtype, args.iters, args.rounds))
                print(json.dumps(rows[-1]), flush=True)
    finally:
        meta["clocks"] = clk.stop()
    print(json.dumps(meta["clocks"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({**meta, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
