"""Measurement only (not collected by pytest): the oracle restatement of the reference's
PyTorch path run EAGERLY ON THE GPU in bf16 (autocast + SDPA), one north-star
diffusion-forcing denoise step — SURVEY.md §8(d) "the real bar".  The reference itself
cannot be imported (diffusers is absent), so this is the closest stand-in for "stock
PyTorch on the same GPU".  Usage: python tests/eager_oracle_bench.py [steps]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src")):
    sys.path.insert(0, p)
import torch  # noqa: E402


def unet_main(n):
    """Config 2: the oracle UNet restatement, eager bf16 autocast, one CFG step."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from unet_bench import MODEL
    from oracle import unet as ounet
    from oracle.ctsd import DDIMSchedulerOracle
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    with torch.device(dev):
        o = ounet.UNetCrossviewTemporalConditionModel(**MODEL)
    o.to(dev).eval()
    B, T, V = 1, 1, 6
    g = torch.Generator().manual_seed(0)
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    cond = dict(
        encoder_hidden_states=(torch.randn(2 * B, T, V, 77, 1024, generator=g) * 0.1).to(dev),
        condition_image_tensor=None,
        disable_crossview=torch.zeros(2 * B, dtype=torch.bool, device=dev),
        disable_temporal=torch.ones(2 * B, dtype=torch.bool, device=dev),
        crossview_attention_mask=ring.unsqueeze(0).repeat(2 * B, 1, 1).to(dev),
        added_time_ids=torch.randn(2 * B, T, V, 11, generator=g).to(dev))
    lat = torch.randn(B, T, V, 4, 32, 56, generator=g).to(dev)
    sch = DDIMSchedulerOracle(beta_start=0.00085, beta_end=0.012)
    sch.set_timesteps(50)

    def step(x, t):
        tt = torch.full((2 * B, T, V), t, device=dev)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = o(torch.cat([x, x]), tt.float(), **cond)[0].float()
        u, c = out.chunk(2)
        return sch.step(u + 3.0 * (c - u), tt[:B], x)

    ts = sch.timesteps.tolist()
    x = step(lat, ts[0])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(n):
        x = step(x, ts[1 + k])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    res = {"impl": "oracle UNet restatement, eager PyTorch bf16 autocast + SDPA on the GPU",
           "workload": "ctsd_21 6-view image step [2,1,6,4,32,56]", "ms_per_step": ms,
           "steps_per_s": 1000.0 / ms, "steps": n}
    print(json.dumps(res))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "eager_oracle_unet_bench.json"), "w") as f:
        json.dump(res, f)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "unet":
        return unet_main(int(sys.argv[2]) if len(sys.argv) > 2 else 10)
    import bench
    from oracle import ctsd as octsd
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    cfg = bench.load_config()
    B, T, V, C, H, W = cfg["latent_shape"]
    steps = cfg["inference_steps"]
    spi = steps // T
    dev = torch.device("cuda", 0)
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        oracle = octsd.DiTCrossviewTemporalConditionModel(**cfg["model"])
    torch.set_default_dtype(torch.float32)
    bench.init_weights_(oracle)
    oracle.to(dev).eval()
    cond = bench.synthetic_conditions(cfg, 2 * B, T, V, dev, torch.bfloat16)
    lat = torch.randn(B, T, V, C, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(steps)
    sched.timesteps = sched.timesteps.to(dev)
    sched.sigmas = sched.sigmas.to(dev)

    def step(i, x):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return octsd.df_denoise_step(oracle, sched, x, cond, i=i, steps_per_inference=spi,
                                         guidance_scale=cfg["guidance_scale"],
                                         model_dtype=torch.bfloat16)[0].float()

    x = step(steps - 3, lat)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(n):
        x = step(steps - 3 + k % 3, x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    res = {"impl": "oracle restatement, eager PyTorch bf16 autocast + SDPA on the GPU",
           "ms_per_step": ms, "steps_per_s": 1000.0 / ms, "steps": n,
           "executed_tflop_per_step": 447.4, "algorithmic_tflop_per_step": bench.F_STEP_TFLOP,
           "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
    print(json.dumps(res))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "eager_oracle_bench.json"), "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main()
