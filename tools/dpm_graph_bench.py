"""Eager against CUDA-graph replay of the CTSD-2.1 examples' scheduler (DPM-Solver++ 2M, CFG 3,
50 steps; examples/ctsd_21_6views_image_generation.json = BASELINE config 2):

* the step: `denoise_step` vs `denoise_step_graphed` of the UNet on [2, 1, 6, 4, 32, 56], in
  alternating rounds of one whole 50-step schedule each (the scheduler is reset between rounds,
  so every round replays the one captured graph); median and range of ms/step per round;
* the window: the whole 50-step `inference_pipeline` (conditions, steps; no VAE configured)
  with inference_config["cuda_graph"] off and on, alternating; the graphed window includes
  its warm-up step and capture.

The card's name and power limit are read in the same run.

    python tools/dpm_graph_bench.py [--rounds 5] [--windows 3] [--out PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

STEPS = 50


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": {"query": q, "value": out}}


def build(dev, dtype):
    from bench_extras import _init, _ring, _blocks
    from unet_bench import MODEL
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    blk = _blocks()["ctsd_21_6views_image_generation.json"]["pipeline"]
    common = {k: v for k, v in blk["common_config"].items()
              if k not in ("autocast", "text_encoder_load_args")}
    inf = {k: v for k, v in blk["inference_config"].items() if k != "preview_image_size"}
    assert inf["scheduler"] == "diffusers.DPMSolverMultistepScheduler"
    assert inf["inference_steps"] == STEPS and inf["guidance_scale"] == 3
    with torch.device(dev):
        m = U(**MODEL, compute_dtype=dtype)
    _init(m)
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, dev, common, {}, inf, None, m,
                               model_dtype=dtype)
    assert type(pipe.test_scheduler).__name__ == "DPMSolverMultistepScheduler"
    B, T, V = 1, 1, 6
    gen = torch.Generator().manual_seed(0)
    cond = dict(
        encoder_hidden_states=(torch.randn(2 * B, T, V, 77, 1024, generator=gen) * 0.1)
        .to(dev, dtype),
        condition_image_tensor=None,
        disable_crossview=torch.zeros(2 * B, dtype=torch.bool, device=dev),
        disable_temporal=torch.ones(2 * B, dtype=torch.bool, device=dev),
        crossview_attention_mask=_ring(V).unsqueeze(0).repeat(2 * B, 1, 1).to(dev),
        added_time_ids=torch.randn(2 * B, T, V, 11, generator=gen).to(dev))
    noise = torch.randn(B, T, V, 4, 32, 56, generator=gen).to(dev)
    return pipe, cond, noise


def step_rounds(pipe, cond, noise, rounds):
    """ms/step of whole 50-step schedules, eager and graphed rounds alternating."""
    from opendwm_b200 import ops
    sch = pipe.test_scheduler
    dev = noise.device
    lat = {False: noise.clone(), True: noise.clone()}      # the graph is keyed on its latents

    def schedule(graphed, count_launches=False):
        x = lat[graphed]
        x.copy_(noise)
        sch.set_timesteps(STEPS, dev)
        ts = [t.to(torch.int32).expand(1, 1, 6).contiguous() for t in sch.timesteps]
        fn = pipe.denoise_step_graphed if graphed else pipe.denoise_step
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if count_launches:
            ops.profile_begin()
        e0.record()
        for t in ts:
            fn(x, cond, None, t, None)
        e1.record()
        torch.cuda.synchronize()
        launches = ops.profile_end()["launches"] / STEPS if count_launches else None
        return e0.elapsed_time(e1) / STEPS, launches

    _, launches = schedule(False, count_launches=True)     # warm-up: packing, caches
    schedule(True)                                         # warm-up: capture
    ms = {False: [], True: []}
    for _ in range(rounds):
        for graphed in (False, True):
            ms[graphed].append(schedule(graphed)[0])
    diff = (lat[False] - lat[True]).abs().max().item()
    return ms, launches, diff, len(pipe._graphs), bool(torch.isfinite(lat[True]).all())


def window_rounds(pipe, windows):
    """Wall-clock seconds of the whole 50-step inference_pipeline, cuda_graph off / on."""
    from bench_extras import frame_batch
    batch = frame_batch(torch.Generator().manual_seed(1), 6, (256, 448), 77, 1024, 1024, 0)
    for k in ("3dbox_images", "hdmap_images"):     # the image example has no layout adapter
        batch.pop(k)
    shape = (1, 1, 6, 4, 32, 56)

    def window(graphed):
        pipe.inference_config["cuda_graph"] = graphed
        pipe.generator.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipe.inference_pipeline(shape, batch, "pt")
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out["latents"]

    window(False)
    window(True)
    s = {False: [], True: []}
    last = {}
    for _ in range(windows):
        for graphed in (False, True):
            dt, last[graphed] = window(graphed)
            s[graphed].append(dt)
    rel = ((last[False] - last[True]).abs().max() / last[False].abs().max()).item()
    return s, rel


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--dtype", default="float16", choices=["float16", "bfloat16"])
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "dpm_graph_bench.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpm_graph_bench needs a CUDA device")
    dev, dtype = torch.device("cuda", 0), getattr(torch, a.dtype)
    torch.cuda.set_device(dev)
    res = {"card": card(), "dtype": a.dtype,
           "workload": "config 2: ctsd_21 6-view image, UNet on [2,1,6,4,32,56], CFG 3, "
                       "DPM-Solver++ 2M (v_prediction), 50 steps"}
    with torch.no_grad():
        pipe, cond, noise = build(dev, dtype)
        ms, launches, diff, graphs, finite = step_rounds(pipe, cond, noise, a.rounds)
        res["step_ms"] = {"eager": summary(ms[False]), "graph": summary(ms[True]),
                          "rounds": a.rounds, "steps_per_round": STEPS,
                          "eager_launches_per_step": launches, "graphs_captured": graphs,
                          "eager_vs_graph_max_abs_diff": diff, "finite": finite}
        s, rel = window_rounds(pipe, a.windows)
        res["window_s"] = {"cuda_graph_off": summary(s[False]), "cuda_graph_on": summary(s[True]),
                           "windows": a.windows, "off_vs_on_max_rel_diff": rel}
    res["card_after"] = card()
    print(json.dumps(res))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
