"""FP8 vs 16-bit CTSD-2.1 UNet step, in one process.

Builds the BASELINE config-2 UNet (tools/unet_bench.py) twice with the same weights: 16-bit
GEMMs and convolutions, and gemm_dtype=torch.float8_e4m3fn.  For two workloads
- config 2: [2, 1, 6, 4, 32, 56] (CFG-doubled), T = 1, temporal blocks off;
- video:    [2, 8, 6, 4, 32, 56] (CFG-doubled), temporal blocks on
it alternates CUDA-graph replays of the DDIM step (denoise_step_graphed) of the two arms over
`--rounds` rounds, and compares the two noise predictions on the same seeded inputs.  It also
times the level-1 ResBlock conv (12 items, 32 x 56, 320 -> 320, 3 x 3, per-item residual) in
both precisions with CUDA events.  Prints one JSON line with the card name and power limit read
in the same run.

Usage: python tools/fp8_unet_bench.py [--steps 3] [--rounds 3] [--only config2|video] [--out F]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from fp8_bench import card  # noqa: E402
from unet_bench import MODEL  # noqa: E402

WORKLOADS = {"config2": (1, 1, 6, 32, 56, True), "video": (1, 8, 6, 32, 56, False)}


def conv_bench(iters=50):
    """Level-1 ResBlock conv1 (operand from GroupNorm+SiLU, + per-item temb row) in bf16 and
    FP8: ms per call and algorithmic TFLOP/s."""
    from opendwm_b200 import lib, ops
    n, h, w, c = 12, 32, 56, 320
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, 1, h, w, c, generator=g, device="cuda")
    wt = torch.randn(c, c, 3, 3, generator=g, device="cuda") * (9 * c) ** -0.5
    bias = torch.zeros(c, device="cuda")
    temb = torch.randn(n, c, generator=g, device="cuda")
    x16 = x.to(torch.bfloat16)
    w16 = ops.pack_conv_weight(wt, torch.bfloat16)
    q, s = ops.quantize_rows(x.view(n, -1))
    x8, sa = q.view(x.shape), s
    w8, sw = ops.pack_conv_weight_fp8(wt)
    out = torch.empty(n * h * w, c, device="cuda")
    kw = dict(kernel=(1, 3, 3), epilogue=lib.EPI_RESID, resid=temb, resid_rows_per_item=h * w,
              out=out)
    arms = {"bf16": lambda: ops.conv(x16, w16, bias, **kw),
            "fp8": lambda: ops.conv(x8, w8, bias, a_scale=sa, w_scale=sw, **kw)}
    flop = 2.0 * n * h * w * c * 9 * c
    res = {}
    for k, f in arms.items():
        for _ in range(5):
            f()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            f()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / iters
        res[k] = {"ms": round(ms, 4), "tflops": round(flop / (ms * 1e9), 1)}
    res["speedup"] = round(res["bf16"]["ms"] / res["fp8"]["ms"], 3)
    res["shape"] = "12 x 32 x 56, 320 -> 320, 3x3, RESID per item"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="timed steps per arm and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", choices=sorted(WORKLOADS))
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_unet_bench needs a GPU: there is nothing to measure on the CPU")

    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from dwm.pipelines.ctsd import CrossviewTemporalSD

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dtype = torch.bfloat16
    models = {}
    with torch.device(dev):
        models["16bit"] = U(**MODEL, compute_dtype=dtype)
        models["fp8"] = U(**MODEL, compute_dtype=dtype, gemm_dtype=torch.float8_e4m3fn)
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():     # the weights of tools/unet_bench.py
        for n, p in models["16bit"].named_parameters():
            if n.endswith("mix_factor"):
                continue
            if p.dim() == 1 and n.endswith(".weight"):
                p.fill_(1.0)
            elif n.endswith(".bias"):
                p.zero_()
            else:
                p.copy_(torch.randn(p.shape, generator=g, device="cuda") * 0.02)
    models["fp8"].load_state_dict(models["16bit"].state_dict())

    line = {"tool": "fp8_unet_bench", "card": card(), "dtype": "bf16", "cfg": True,
            "mode": "CUDA-graph replay of the DDIM step (denoise_step_graphed)", "workloads": {}}
    for name, (B, T, V, H, W, t_off) in WORKLOADS.items():
        if args.only and name != args.only:
            continue
        gen = torch.Generator().manual_seed(0)
        ring = torch.zeros(V, V, dtype=torch.bool)
        for i in range(V):
            for d in (-1, 0, 1):
                ring[i, (i + d) % V] = True
        cond = dict(
            encoder_hidden_states=(torch.randn(2 * B, T, V, 77, 1024, generator=gen) * 0.1)
            .to(dev, dtype),
            condition_image_tensor=None,
            disable_crossview=torch.zeros(2 * B, dtype=torch.bool, device=dev),
            disable_temporal=torch.full((2 * B,), t_off, dtype=torch.bool, device=dev),
            crossview_attention_mask=ring.unsqueeze(0).repeat(2 * B, 1, 1).to(dev),
            added_time_ids=torch.randn(2 * B, T, V, 11, generator=gen).to(dev))
        lat0 = torch.randn(B, T, V, 4, H, W, generator=gen).to(dev)
        pipes, lat = {}, {}
        for k, m in models.items():
            pipes[k] = CrossviewTemporalSD(
                None, {"generator_seed": 0}, dev, {"frame_prediction_style": "ctsd"}, {},
                {"guidance_scale": 3, "inference_steps": 50}, None, m, model_dtype=dtype)
            pipes[k].test_scheduler.set_timesteps(50, dev)
            lat[k] = lat0.clone()
        tsched = pipes["16bit"].test_scheduler.timesteps
        ts_list = [tsched[k].to(torch.int32).expand(B, T, V).contiguous() for k in range(50)]

        def step(k, i):
            pipes[k].denoise_step_graphed(lat[k], cond, None, ts_list[i % 50], None)

        for k in pipes:           # warm-up + capture
            for i in range(2):
                step(k, i)
        torch.cuda.synchronize()
        times = {k: [] for k in pipes}
        for r in range(args.rounds):
            for k in (("16bit", "fp8") if r % 2 == 0 else ("fp8", "16bit")):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    step(k, 2 + i)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / args.steps)
        # noise predictions of the two arms on the same CFG-doubled inputs
        sample = lat0.repeat(2, 1, 1, 1, 1, 1)
        t_in = ts_list[10].repeat(2, 1, 1)
        pred = {k: m(sample, t_in.float(), **cond)[0][0].float() for k, m in models.items()}
        diff = ((pred["fp8"] - pred["16bit"]).abs().max() / pred["16bit"].abs().max()).item()
        med = {k: statistics.median(v) for k, v in times.items()}
        line["workloads"][name] = {
            "latent_shape": [2 * B, T, V, 4, H, W], "temporal": not t_off,
            "step_ms_median": {k: round(v, 2) for k, v in med.items()},
            "step_ms_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()},
            "speedup": round(med["16bit"] / med["fp8"], 3),
            "noise_pred_max_rel_diff": diff,
            "finite": bool(all(torch.isfinite(v).all() for v in lat.values()))}
        del pipes, lat
        torch.cuda.empty_cache()
    line["level1_conv"] = conv_bench()
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
