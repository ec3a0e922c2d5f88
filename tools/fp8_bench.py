"""FP8 vs 16-bit GEMMs on the north-star denoise step (6 views x 16 frames, CFG), in one process.

Builds the north-star DiT twice with the same weights: 16-bit GEMMs, and
gemm_dtype=torch.float8_e4m3fn.  Alternates timed steps of the two (device events around each
step), profiles one step of each with ops.profile_begin for per-GEMM TFLOP/s, and compares the
two noise predictions (proj_out tokens) on the same seeded inputs.  Prints one JSON line with
the card name and power limit read in the same run.

Usage: python tools/fp8_bench.py [--steps 3] [--rounds 3] [--warmup 2] [--dtype fp16] [--small]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402  (north-star config, synthetic conditions, weight init)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    f = [x.strip() for x in out.split(",")] if out else []
    return {"name": torch.cuda.get_device_name(), "power_limit": f[1] if len(f) > 1 else None,
            "sm_max_clock": f[2] if len(f) > 2 else None}


def gemm_table(prof):
    """Per (M, N, K, epilogue): calls, ms, TFLOP/s of the profiled step's linears."""
    rows = {}
    for e in prof["linear"]:
        key = "{}x{}x{}/epi{}".format(*e["shape"], e["epilogue"])
        r = rows.setdefault(key, {"calls": 0, "ms": 0.0, "flop": 0.0})
        r["calls"] += 1
        r["ms"] += e["ms"]
        r["flop"] += e["flops"]
    for r in rows.values():
        r["tflops"] = round(r["flop"] / (r["ms"] * 1e9), 1) if r["ms"] > 0 else None
        r["ms"] = round(r["ms"], 3)
    total_ms = sum(e["ms"] for e in prof["linear"])
    total_flop = sum(e["flops"] for e in prof["linear"])
    return {"gemm_ms": round(total_ms, 2),
            "gemm_tflops": round(total_flop / (total_ms * 1e9), 1) if total_ms else None,
            "by_shape": dict(sorted(rows.items(), key=lambda kv: -kv[1]["ms"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="timed steps per arm and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dtype", default="fp16", choices=["bf16", "fp16"])
    ap.add_argument("--small", action="store_true", help="debug-size model/shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench needs a GPU: there is nothing to measure on the CPU")

    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    from opendwm_b200 import ops

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = bench.load_config(args.small)
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[args.dtype]
    B, T, V, C, H, W = cfg["latent_shape"]
    steps = cfg["inference_steps"]
    spi = steps // T

    models = {}
    torch.set_default_dtype(dtype)
    with torch.device(dev):
        models["16bit"] = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
        models["fp8"] = DiTCrossviewTemporalConditionModel(
            **cfg["model"], compute_dtype=dtype, gemm_dtype=torch.float8_e4m3fn)
    torch.set_default_dtype(torch.float32)
    bench.init_weights_(models["16bit"])
    models["fp8"].load_state_dict(models["16bit"].state_dict())

    cond = bench.synthetic_conditions(cfg, 2 * B, T, V, dev, dtype)
    latents0 = torch.randn(B, T, V, C, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    inf = {"guidance_scale": cfg["guidance_scale"], "inference_steps": steps,
           "sequence_length_per_iteration": T,
           "scheduler": "dwm.schedulers.temporal_independent.FlowMatchEulerDiscreteScheduler"}
    pipes, lat = {}, {}
    for k, m in models.items():
        pipes[k] = StreamingCrossviewTemporalSD(
            None, {"generator_seed": 0}, dev, {"frame_prediction_style": "diffusion_forcing"}, {},
            inf, None, m, model_dtype=dtype)
        pipes[k].reset_streaming((B, T, V, C, H, W), "pt")
        lat[k] = latents0.clone()
    idx_list = [pipes["16bit"]._df_step_tensors(i, T, spi, 0, B, V)
                for i in (steps - 3, steps - 2, steps - 1)]

    def step(k, i):
        idx, ts, in_range = idx_list[i % 3]
        pipes[k].denoise_step(lat[k], cond, idx, ts, in_range)

    for k in pipes:
        for i in range(args.warmup):
            step(k, i)
    torch.cuda.synchronize()

    times = {k: [] for k in pipes}
    for r in range(args.rounds):
        for k in (("16bit", "fp8") if r % 2 == 0 else ("fp8", "16bit")):
            for i in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(k, i)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1))

    gemms = {}
    for k in pipes:
        ops.profile_begin()
        step(k, 0)
        torch.cuda.synchronize()
        gemms[k] = gemm_table(ops.profile_end())

    # noise predictions of the two arms on the same inputs (CFG-doubled batch); after the
    # timed steps, which this call's condition-cache key would otherwise disturb
    _, ts, _ = idx_list[0]
    sample = latents0.repeat(2, 1, 1, 1, 1, 1)
    t_in = ts.repeat(2, 1, 1).to(dev)
    tok = {k: m.forward_tokens(sample, t_in, **cond)[0].clone() for k, m in models.items()}
    diff = ((tok["fp8"] - tok["16bit"]).abs().max() / tok["16bit"].abs().max()).item()

    med = {k: statistics.median(v) for k, v in times.items()}
    line = {
        "tool": "fp8_bench", "card": card(), "dtype": args.dtype, "small": args.small,
        "latent_shape": cfg["latent_shape"], "cfg": True,
        "step_ms_median": {k: round(v, 2) for k, v in med.items()},
        "step_ms_all": {k: [round(x, 2) for x in v] for k, v in times.items()},
        "speedup": round(med["16bit"] / med["fp8"], 3),
        "noise_pred_max_rel_diff": diff,
        "fp8_weight_bytes_saved": models["fp8"]._pk["fp8_bytes_saved"],
        "gemm": gemms,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
