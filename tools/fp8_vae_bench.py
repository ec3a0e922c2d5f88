"""FP8 vs 16-bit VAE decodes, in one process.

Builds each decoder twice with the same random-init weights (no checkpoint is read: the error
on real weights is not measured here): 16-bit, and gemm_dtype=torch.float8_e4m3fn (E4M3 decoder
ResNet convolutions).  Workloads
- cogvideox_window: the config-5 window decode of tools/vae_bench.py, [16, 5, 32, 56] latents ->
  17 frames 256x448, 2 views per call (reported per call and per 6-view window);
- cogvideox_df: the diffusion-forcing decode of one emitted frame of 6 views as the pipeline
  runs it (and as bench.py's frame_latency.cogvideox_decode_ms times it): the latent frame
  followed by a zero frame, [6, 16, 2, 32, 56], one chunk -> 8 frames 256x448;
- sd35_kl: the SD-3.5 AutoencoderKL decode of 6 views, [6, 16, 32, 56] -> 256x448
  (tools/vae2d_bench.py).
It alternates the two arms over `--rounds` rounds (CUDA events around at least `--iters`
calls and 250 ms of decodes per round), reports each round, the round-to-round spread and
whether the arms' round ranges overlap, and
compares the FP8 and 16-bit images on the same seeded latents: max|d| / max|16-bit| and the PSNR
with the 16-bit image's range (max - min) as the peak.  It also times the level-0 CogVideoX conv
(2 volumes of 8 + 2 frames, 256x448, 128 -> 128, 3x3x3, F32 epilogue) in both precisions.
Algorithmic TFLOP/s come from the decoder_flops of tools/vae_bench.py / tools/vae2d_bench.py.
The card's name and power limit and the median SM clock (nvidia-smi, sampled during the timed
rounds) are read in the same run.

Usage: python tools/fp8_vae_bench.py [--rounds 3] [--iters 3] [--only W] [--out F]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import threading

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from fp8_bench import card  # noqa: E402

F8 = torch.float8_e4m3fn
MIN_ROUND_MS = 250.0


class ClockSampler:
    """Samples the SM clock (MHz) with nvidia-smi every `period` seconds while active."""

    def __init__(self, period=0.5):
        self.period, self.samples, self._stop = period, [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        dev = str(torch.cuda.current_device())
        while not self._stop.wait(self.period):
            try:
                out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                      "-i", dev], capture_output=True, text=True, timeout=10).stdout
                self.samples.append(float(out.strip()))
            except (OSError, ValueError, subprocess.SubprocessError):
                pass

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        return statistics.median(self.samples) if self.samples else None


def compare(y8, y16):
    y8, y16 = y8.float(), y16.float()
    d = y8 - y16
    mse = d.pow(2).mean().item()
    peak = (y16.max() - y16.min()).item()
    return {"max_rel_diff": (d.abs().max() / y16.abs().max()).item(),
            "psnr_db": round(10 * math.log10(peak ** 2 / mse), 2) if mse > 0 else None,
            "finite": bool(torch.isfinite(y8).all() and torch.isfinite(y16).all())}


def workloads():
    """name -> (builder(gemm_dtype), latents, algorithmic FLOP per call, note)."""
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    from vae2d_bench import SD35_VAE
    from vae2d_bench import decoder_flops as kl_flops
    from vae_bench import decoder_flops as cv_flops
    g = torch.Generator().manual_seed(0)
    cv = lambda gd: AutoencoderKLCogVideoX(compute_dtype=torch.bfloat16, gemm_dtype=gd)  # noqa: E731
    kl = lambda gd: AutoencoderKL(**SD35_VAE, compute_dtype=torch.bfloat16, gemm_dtype=gd)  # noqa: E731
    ref = cv(None)
    cur = torch.randn(6, 16, 32, 56, generator=g)
    df = torch.cat([cur[:, :, None], cur[:, :, None] * 0], dim=2)   # ctsd.py: frame + zero frame
    return {
        "cogvideox_window": (cv, torch.randn(2, 16, 5, 32, 56, generator=g),
                             cv_flops(ref, 5, 32, 56) * 2, "config 5: 2 views per call"),
        "cogvideox_df": (cv, df, cv_flops(ref, 2, 32, 56) * 6,
                         "diffusion-forcing decode: latent frame + zero frame, 6 views"),
        "sd35_kl": (kl, torch.randn(6, 16, 32, 56, generator=g).bfloat16(),
                    kl_flops(SD35_VAE, 32, 56) * 6, "6 views, 256x448"),
    }


def time_calls(f, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def conv_bench(iters=20):
    """Level-0 CogVideoX ResNet conv1: 2 volumes of 8 + 2 frames, 256x448, 128 -> 128, 3x3x3,
    fp32 output + bias, in bf16 and FP8: ms per call and algorithmic TFLOP/s."""
    from opendwm_b200 import lib, ops
    n, tp, h, w, c = 2, 10, 256, 448, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, tp, h, w, c, generator=g, device="cuda")
    wt = torch.randn(c, c, 3, 3, 3, generator=g, device="cuda") * (27 * c) ** -0.5
    bias = torch.zeros(c, device="cuda")
    x16 = x.to(torch.bfloat16)
    w16 = ops.pack_conv_weight(wt, torch.bfloat16)
    q, sa = ops.quantize_rows(x.view(n, -1))
    x8 = q.view(x.shape)
    w8, sw = ops.pack_conv_weight_fp8(wt)
    del x
    out = torch.empty(n * (tp - 2) * h * w, c, device="cuda")
    kw = dict(kernel=(3, 3, 3), epilogue=lib.EPI_F32, out=out)
    arms = {"bf16": lambda: ops.conv(x16, w16, bias, **kw),
            "fp8": lambda: ops.conv(x8, w8, bias, a_scale=sa, w_scale=sw, **kw)}
    flop = 2.0 * n * (tp - 2) * h * w * c * 27 * c
    times = {k: [] for k in arms}
    for f in arms.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    for r in range(3):
        for k in (("bf16", "fp8") if r % 2 == 0 else ("fp8", "bf16")):
            times[k].append(time_calls(arms[k], iters))
    res = {k: {"ms": round(statistics.median(v), 4),
               "tflops": round(flop / (statistics.median(v) * 1e9), 1)} for k, v in times.items()}
    res["speedup"] = round(res["bf16"]["ms"] / res["fp8"]["ms"], 3)
    res["shape"] = "2 x (8 + 2) x 256 x 448, 128 -> 128, 3x3x3, F32 + bias"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3, help="timed calls per arm and round")
    ap.add_argument("--only", choices=["cogvideox_window", "cogvideox_df", "sd35_kl", "conv"])
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_vae_bench needs a GPU: there is nothing to measure on the CPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    line = {"tool": "fp8_vae_bench", "card": card(), "dtype": "bf16",
            "weights": "random init (no checkpoint): error on real weights not measured",
            "workloads": {}}
    with ClockSampler() as clocks:
        for name, (build, z, flop, note) in workloads().items():
            if args.only and name != args.only:
                continue
            torch.manual_seed(0)
            with torch.device(dev):
                models = {"16bit": build(None)}
                models["fp8"] = build(F8)
            models["fp8"].load_state_dict(models["16bit"].state_dict())
            z = z.to(dev)
            outs = {k: m.decode(z, return_dict=False)[0] for k, m in models.items()}   # warm-up
            torch.cuda.synchronize()
            # at least MIN_ROUND_MS of GPU time per arm and round, so that short decodes are not
            # timed over a window of a few tens of milliseconds
            once = time_calls(lambda: models["16bit"].decode(z, return_dict=False), 1)
            iters = max(args.iters, math.ceil(MIN_ROUND_MS / once))
            times = {k: [] for k in models}
            for r in range(args.rounds):
                for k in (("16bit", "fp8") if r % 2 == 0 else ("fp8", "16bit")):
                    times[k].append(time_calls(lambda: models[k].decode(z, return_dict=False), iters))
            med = {k: statistics.median(v) for k, v in times.items()}
            # the arms are told apart only if their round ranges do not overlap
            apart = max(times["fp8"]) < min(times["16bit"]) or max(times["16bit"]) < min(times["fp8"])
            line["workloads"][name] = {
                "note": note, "latent_shape": list(z.shape), "out_shape": list(outs["16bit"].shape),
                "ms_median": {k: round(v, 2) for k, v in med.items()},
                "calls_per_round": iters,
                "ms_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()},
                "ms_round_spread": {k: round(max(v) - min(v), 2) for k, v in times.items()},
                "arms_apart": apart,
                "tflops": {k: round(flop / (v * 1e9), 1) for k, v in med.items()},
                "speedup": round(med["16bit"] / med["fp8"], 3),
                "fp8_vs_16bit": compare(outs["fp8"], outs["16bit"])}
            if name == "cogvideox_window":
                line["workloads"][name]["ms_per_6view_window"] = {k: round(3 * v, 1) for k, v in med.items()}
            del models, outs
            torch.cuda.empty_cache()
        if not args.only or args.only == "conv":
            line["level0_conv"] = conv_bench()
    line["sm_clock_mhz_median"] = clocks.median()
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
