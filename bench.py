#!/usr/bin/env python
"""Benchmark of the CTSD-3.5 diffusion-forcing denoise step (BASELINE.json metric:
denoise-steps/sec, 6 views x 16 frames, CFG on).

  python bench.py --gpus N --steps K --warmup W            # this repo (sm_90a kernels)
  python bench.py --impl reference --steps K --warmup W    # reference semantics on host CPU

One "step" = one iteration of StreamingCrossviewTemporalSD.inference_pipeline's loop
(reference ctsd.py:2046-2090): CFG-doubled noise-predict forward on latents
[2,16,6,16,32,56], CFG combine, per-frame Euler update, masked latent update, at the
steady-state diffusion-forcing indices i in {45,46,47} of a 48-step schedule.
Synthetic inputs (seed 0) and random-init weights N(0, 0.02) of the north-star
architecture (no checkpoints / datasets offline).

Multi-GPU (torchrun, one rank per GPU): the 6xT view-frame grid x CFG branch is
sharded: first over the two CFG branches, then over frames; strong scaling.
Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "src")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

METRIC = "CTSD-3.5 6view x 16f denoise-steps/sec"
F_STEP_TFLOP = 396.2   # algorithmic FLOPs per step, SURVEY.md §8(d) / tools/flops.py


def load_config(small=False):
    with open(os.path.join(ROOT, "configs", "ctsd_35_df16_northstar.json")) as f:
        cfg = json.load(f)
    if small:
        m = cfg["model"]
        m.update(num_layers=4, dual_attention_layers=[0, 1],
                 crossview_block_layers=[1], temporal_block_layers=[2, 3],
                 pos_embed_max_size=96)
        cfg["latent_shape"] = [1, 4, 6, 16, 16, 24]
        cfg["text_tokens"] = 20
        cfg["inference_steps"] = 12
    return cfg


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            d = json.load(f)
        _PEAKS.update(d)
        return d.get("bf16_tflops_sustained", 989.0), d.get("hbm_gbs"), "measured"
    # NVIDIA H100 SXM data sheet (700 W): dense BF16 / FP16 and HBM3 bandwidth
    return 989.0, 3350.0, "datasheet"


_PEAKS = {}


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.lines, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                 "-i", str(self.index), "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:  # noqa: BLE001
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:  # noqa: BLE001
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown",
                                "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx,
                "reasons": sorted(reasons), "samples": len(sm)}


# ----------------------------------------------------------------------------- synthetic data
def synthetic_conditions(cfg, B_cfg, T, V, device, dtype, seed=0):
    """SURVEY.md §8(d) synthetic inputs; B_cfg = CFG-doubled batch (uncond first)."""
    m = cfg["model"]
    g = torch.Generator().manual_seed(seed)
    L = cfg["text_tokens"]
    H, W = cfg["latent_shape"][-2:]
    ehs = (torch.randn(B_cfg, T, V, L, m["joint_attention_dim"], generator=g) * 0.1)
    pooled = torch.randn(B_cfg, T, V, m["pooled_projection_dim"], generator=g)
    img = torch.rand(B_cfg, T, V, 6, H * 8, W * 8, generator=g)
    ids = torch.randn(B_cfg, T, V, 13, generator=g)
    ids[..., 0] = 10.0                                   # fps
    ids[..., 11] = torch.rand(B_cfg, T, V, generator=g) * 60   # speed km/h
    ids[..., 12] = torch.randn(B_cfg, T, V, generator=g) * 30  # steering
    half = B_cfg // 2
    if half:
        img[:half] = 0.1255                               # uncondition_image_color
        ids[:half, ..., 11:] = -1000.0
        ids[half:, ..., :11] = ids[:half, ..., :11]
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    return dict(
        encoder_hidden_states=ehs.to(device=device, dtype=dtype),
        pooled_projections=pooled.to(device=device, dtype=dtype),
        condition_image_tensor=img.to(device=device, dtype=dtype),
        disable_crossview=torch.zeros(B_cfg, dtype=torch.bool, device=device),
        disable_temporal=torch.zeros(B_cfg, dtype=torch.bool, device=device),
        crossview_attention_mask=ring.unsqueeze(0).repeat(B_cfg, 1, 1).to(device),
        added_time_ids=ids.to(device))


def init_weights_(model, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("mix_factor"):
                continue
            if p.dim() == 1 and name.endswith(".weight"):
                p.fill_(1.0)
            elif name.endswith(".bias"):
                p.zero_()
            else:
                p.copy_(torch.randn(p.shape, generator=g, device="cuda",
                                    dtype=torch.float32).mul_(0.02).to(p.dtype))


# ----------------------------------------------------------------------------- native arm
def run_native(args):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    from opendwm_b200 import ops

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run for --gpus > 1")
    if args.dump_outputs and world > 1:
        # each rank holds only its CFG branch / frame shard of the latents
        raise SystemExit("--dump-outputs records the unsharded step: run it with --gpus 1")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)

    cfg = load_config(args.small)
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[args.dtype]
    B, T, V, C, H, W = cfg["latent_shape"]
    steps = cfg["inference_steps"]
    spi = steps // T

    from opendwm_b200.sharding import ShardPlan
    plan = ShardPlan(world, rank, T, cfg=True) if world > 1 else None
    cfg_ways = plan.cfg_ways if plan else 1
    t_ways = plan.t_ways if plan else 1

    torch.set_default_dtype(dtype)
    with torch.device(dev):
        model = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
    torch.set_default_dtype(torch.float32)
    init_weights_(model)
    pipe_cfg = {"generator_seed": 0}
    common = {"frame_prediction_style": "diffusion_forcing"}
    inf = {"guidance_scale": cfg["guidance_scale"], "inference_steps": steps,
           "sequence_length_per_iteration": T,
           "scheduler": "dwm.schedulers.temporal_independent."
                        "FlowMatchEulerDiscreteScheduler"}
    pipe = StreamingCrossviewTemporalSD(
        None, pipe_cfg, dev, common, {}, inf, None, model, model_dtype=dtype)
    pipe.reset_streaming((B, T, V, C, H, W), "pt")

    pipe.sharding = plan
    cond_full = synthetic_conditions(cfg, 2 * B, T, V, dev, dtype)
    gen = torch.Generator().manual_seed(0)
    latents_full = torch.randn(B, T, V, C, H, W, generator=gen)
    if plan is not None:     # this rank's CFG branch / frames, sliced ONCE
        cond = plan.local_conditions(cond_full, cfg_doubled=True)
        latents_host = plan.local_latents(latents_full).pin_memory()
        fs = plan.frame_slice()
    else:
        cond, latents_host, fs = cond_full, latents_full.pin_memory(), slice(0, T)
    del cond_full
    latents = latents_host.to(dev)

    def step_tensors(i):
        idx, ts, in_range = pipe._df_step_tensors(i, T, spi, 0, B, V)
        return (idx[:, fs].contiguous(), ts[:, fs].contiguous(), in_range[fs].contiguous())

    idx_list = [step_tensors(i) for i in (steps - 3, steps - 2, steps - 1)]

    def one_step(k, lat):
        idx, ts, in_range = idx_list[k % 3]
        pipe.denoise_step(lat, cond, idx, ts, in_range)

    lat_dev = torch.empty_like(latents)
    idx_dev = torch.empty_like(idx_list[0][0])

    # the end-to-end loop replays the step from a CUDA graph (`denoise_step_graphed`, the
    # pipeline's `cuda_graph` inference option) unless --graph 0; sharded steps are captured
    # only with DWM_CUDA_GRAPH_SHARDED=1
    os.environ.setdefault("DWM_CUDA_GRAPH_SHARDED", "1")   # measured on 8 GPUs (r02): captures
    use_graph = bool(args.graph) and (world == 1 or
                                      os.environ["DWM_CUDA_GRAPH_SHARDED"] == "1")
    e2e_step = pipe.denoise_step_graphed if use_graph else pipe.denoise_step

    def step_host(src_host, dst_host, idx_host, k):
        """End-to-end step: pinned host latents + indices in, updated latents out."""
        lat_dev.copy_(src_host, non_blocking=True)
        idx_dev.copy_(idx_host, non_blocking=True)
        _, ts, in_range = idx_list[k % 3]
        e2e_step(lat_dev, cond, idx_dev, ts, in_range)
        dst_host.copy_(lat_dev, non_blocking=True)

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize()

    for k in range(args.warmup):
        one_step(k, latents)
    sync()

    # ---- timed region: device-resident inputs -----------------------------------------
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ops.profile_begin()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync()
    e0.record()
    for k in range(args.steps):
        one_step(k, latents)
    e1.record()
    sync()
    prof = ops.profile_end()
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, latents)
    ms = e0.elapsed_time(e1) / args.steps
    if world > 1:
        t = torch.tensor([ms], device=dev)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms = t.item()

    # ---- end-to-end: host latents in, host latents out, every step --------------------
    out_host = torch.empty_like(latents_host).pin_memory()
    idx_host = [t[0].cpu().pin_memory() for t in idx_list]
    for k in range(2):
        step_host(latents_host, out_host, idx_host[k % 3], k)
    sync()
    e0.record()
    for k in range(args.steps):
        step_host(latents_host, out_host, idx_host[k % 3], k)
    e1.record()
    sync()
    ms_e2e = e0.elapsed_time(e1) / args.steps
    if world > 1:
        t = torch.tensor([ms_e2e], device=dev)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms_e2e = t.item()

    if rank != 0:
        _leave(world)
        return
    frame_latency = None
    if world == 1 and not args.small:
        frame_latency = decode_latency(dev, dtype, V, C, H, W, ms)
    peak_tf, peak_hbm, peak_src = peaks()
    gemm_ms = sum(p["ms"] for p in prof["linear"])
    gemm_fl = sum(p["flops"] for p in prof["linear"])
    n_gemm = len(prof["linear"])
    all_gemm = gemm_fl / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else None
    # dominant kernel = the (shape, epilogue) GEMM with the largest share of the timed region
    by_shape = {}
    for p_ in prof["linear"]:
        k = (tuple(p_["shape"]), p_["epilogue"])
        a = by_shape.setdefault(k, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += p_["ms"]
        a[2] += p_["flops"]
    dom_key, dom = max(by_shape.items(), key=lambda kv: kv[1][1])
    achieved = dom[2] / (dom[1] * 1e-3) / 1e12
    # DRAM bytes per launch of that kernel are not measurable inside this run (no counters)
    traffic, traffic_src = None, None
    scale = 1.0 if not args.small else None
    line = {
        "metric": METRIC, "value": 1000.0 / ms, "unit": "steps/s",
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": args.dtype, "data": "synthetic",
        "config": {
            "workload": "ctsd_35 DFoT 6-view x 16-frame with layout "
                        "(examples/ctsd_35_df16_6views_video_generation_with_layout.json)"
                        + (" [--small debug shape]" if args.small else ""),
            "latent_shape": [2 * B, T, V, C, H, W], "cfg": True,
            "df_indices": [steps - 3, steps - 2, steps - 1], "inference_steps": steps,
            "weights": "random N(0,0.02)", "parallelism":
                "cfg%dxframes%d" % (cfg_ways, t_ways),
            "l2": "inputs larger than L2 (7.4 GB weights + >5 GB activations per step)",
            "step_flops_tflop": F_STEP_TFLOP if scale else None},
        "roofline": {
            "bound": "tensor", "achieved": achieved, "peak": peak_tf, "unit": "TFLOP/s",
            "frac": (achieved / peak_tf) if achieved else None, "traffic": traffic,
            "traffic_source": traffic_src,
            "kernel": "gemm_wgmma_kernel M=%d N=%d K=%d epilogue=%d (CUDA events around "
                      "each of its %d launches in the timed steps)" % (dom_key[0] + (dom_key[1], dom[0])),
            "algorithmic_flops_per_launch": dom[2] / dom[0],
            "kernel_share_of_step": dom[1] / (ms * args.steps),
            "all_gemm_achieved": all_gemm, "all_gemm_launches": n_gemm,
            "gemm_share_of_step": gemm_ms / (ms * args.steps),
            "peak_source": peak_src + " bf16_tflops_sustained (cuBLAS inside a long step; "
                           "the kernel may exceed it, see frac_of_burst_peak)",
            "frac_of_burst_peak": (achieved / _PEAKS["bf16_tflops"])
            if achieved and _PEAKS.get("bf16_tflops") else None,
            "step_frac_of_peak": (F_STEP_TFLOP / world / (ms * 1e-3) / peak_tf)
            if scale else None},
        "e2e": {"value": 1000.0 / ms_e2e, "unit": "steps/s",
                "h2d_bytes_per_step": latents_host.numel() * 4 + idx_host[0].numel() * 4,
                "d2h_bytes_per_step": out_host.numel() * 4,
                "cuda_graph": use_graph,
                "api": "StreamingCrossviewTemporalSD.denoise_step%s with pinned host "
                       "latents + index tensors copied in and latents copied out; a separate "
                       "timed loop (the device-resident loop above also records one CUDA-event "
                       "pair around each of its GEMM launches for the roofline, this one does "
                       "not, which is why it can come out marginally faster)" %
                       ("_graphed (CUDA-graph replay of the step)" if use_graph else "")},
        "gpu_launches": prof["launches"],
        "clocks": clocks,
    }
    if frame_latency is not None:
        line["frame_latency"] = frame_latency
    if args.profile_dump:
        agg = {}
        for p_ in prof["linear"]:
            k = (tuple(p_["shape"]), p_["epilogue"])
            a = agg.setdefault(k, [0, 0.0, 0.0])
            a[0] += 1
            a[1] += p_["ms"]
            a[2] += p_["flops"]
        rows = [{"M": k[0][0], "N": k[0][1], "K": k[0][2], "epilogue": k[1],
                 "launches_per_step": v[0] / args.steps, "ms_per_step": v[1] / args.steps,
                 "tflops": v[2] / v[1] / 1e9} for k, v in agg.items()]
        rows.sort(key=lambda r: -r["ms_per_step"])
        with open(args.profile_dump, "w") as f:
            json.dump({"ms_per_step": ms, "gemm_ms_per_step": gemm_ms / args.steps,
                       "rows": rows}, f, indent=1)
    if world == 1 and not args.small and not args.no_extras:
        # what a user of the reference API sees + the other BASELINE configs + the eager bar;
        # every piece is wrapped so that a failure never loses the headline
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import bench_extras as bx
        try:
            line["streaming_e2e"] = bx.streaming_e2e(model, cfg, dev, dtype)
        except Exception as e:  # noqa: BLE001
            line["streaming_e2e"] = {"error": repr(e)[:300]}
        del pipe, model, cond, latents
        bx._free()
        line["workloads"] = bx.workloads(dev, dtype)
        try:
            line["eager_gpu_baseline"] = bx.eager_gpu_baseline(cfg, dev, dtype)
            line["eager_gpu_baseline"]["native_speedup"] = \
                line["eager_gpu_baseline"]["ms_per_step"] / ms
        except Exception as e:  # noqa: BLE001
            line["eager_gpu_baseline"] = {"error": repr(e)[:300]}
        other = "bf16" if args.dtype == "fp16" else "fp16"
        try:    # same step at the other 16-bit operand type, fresh process (own memory)
            out = subprocess.run(
                [sys.executable, os.path.abspath(__file__), "--dtype", other, "--no-extras",
                 "--no-cpu-baseline", "--steps", str(args.steps), "--warmup",
                 str(args.warmup)], capture_output=True, text=True, timeout=600)
            o = json.loads(out.stdout.strip().splitlines()[-1])
            line["other_dtype"] = {"dtype": other, "value": o["value"], "unit": o["unit"],
                                   "ms_per_step": o["ms_per_step"],
                                   "e2e_value": o["e2e"]["value"],
                                   "roofline_frac": o["roofline"]["frac"],
                                   "clocks": o.get("clocks")}
        except Exception as e:  # noqa: BLE001
            line["other_dtype"] = {"dtype": other, "error": repr(e)[:300]}
    if world == 1 and not args.no_cpu_baseline:
        line["cpu_baseline"] = cpu_baseline(budget_s=args.cpu_budget, small=args.small)
    print(json.dumps(line), flush=True)
    _leave(world)


def dump_outputs(out_dir, latents):
    """What the timed loop computed: the latents its last step left behind, the array a caller
    of `denoise_step` receives (11 MB in float32 at the north-star shape; single GPU only).
    Inputs and weights are seeded, so two builds run with the same arguments can be compared
    output for output."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "latents.npy"), latents.float().cpu().numpy())


def _leave(world):
    """Multi-rank exit.  `destroy_process_group` was observed to hang on this pool after runs
    that used symmetric-memory handles / captured NCCL work (8 GPUs, r02: every rank sat in it
    until the watchdog fired, AFTER the result line had been printed), which would turn a good
    measurement into a timed-out run.  The result is out and nothing needs flushing, so the
    ranks synchronise and leave without tearing NCCL down."""
    if world <= 1:
        return
    try:
        torch.cuda.synchronize()
        torch.distributed.barrier()
        torch.cuda.synchronize()
    except Exception:  # noqa: BLE001
        pass
    sys.stdout.flush()
    sys.stderr.flush()
    os._exit(0)


def decode_latency(dev, dtype, V, C, H, W, ms_step):
    """Per-emitted-frame latency of the streaming loop (SURVEY.md §8(d)): 3 denoise steps
    + the 6-view decode of the exiting frame as StreamingCrossviewTemporalSD.receive_frame
    issues it — with the SD-3.5 2-D AutoencoderKL the north-star config uses (reference
    ctsd.py:2095-2098), and for comparison with the CogVideoX temporal VAE (frame + zero
    frame, :1609-1621).  Untimed by the headline; reported beside it."""
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX

    def timed(fn, n=3):
        fn()                                             # warm-up: packs weights
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            y = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, list(y.shape)
    try:
        torch.manual_seed(0)
        with torch.device(dev):
            vae2d = AutoencoderKL(
                block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                latent_channels=C, norm_num_groups=32, scaling_factor=1.5305,
                shift_factor=0.0609, use_quant_conv=False, use_post_quant_conv=False,
                compute_dtype=dtype)
            vae3d = AutoencoderKLCogVideoX(compute_dtype=dtype)
        cur = torch.randn(V, C, H, W, device=dev).to(dtype)
        dec2, shp2 = timed(lambda: vae2d.decode(cur, return_dict=False)[0])
        z = torch.cat([cur[:, :, None], cur[:, :, None] * 0], dim=2).float()
        dec3, shp3 = timed(lambda: vae3d.decode(z, return_dict=False)[0])
        return {"ms": 3 * ms_step + dec2, "decode_ms": dec2, "denoise_ms": 3 * ms_step,
                "decode_out_shape": shp2,
                "definition": "3 denoise steps (spi) + SD-3.5 AutoencoderKL decode of the "
                              "6 views of the exiting frame at 256x448",
                "cogvideox_decode_ms": dec3, "cogvideox_decode_out_shape": shp3}
    except Exception as e:                               # never lose the headline line
        return {"error": repr(e)[:200]}


# ----------------------------------------------------------------------------- CPU arms
def _host_cores():
    """Cores this process may actually run on (cpuset / affinity aware), capped at 64:
    oversubscribing a cgroup-limited container makes the CPU arm slower, not faster."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:   # cgroup v2 CPU quota
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except Exception:  # noqa: BLE001
        pass
    return max(1, min(n, 64))


def _cpu_reference_sample(small, n_timed, warm, budget_s):
    """The ONE definition of the CPU arm, used by `--impl reference` and by the native arm's
    `cpu_baseline`: the oracle restatement of the reference's PyTorch modules (the reference
    itself needs diffusers==0.31.0, not installable offline), fp32 on the host cores,
    full-depth north-star model, a bounded sample of the step per timed forward: 1 frame x
    6 views without CFG (6 of the 192 view-frame items; every cost of the step is per item
    or per frame-group), scaled by 192/6.  Returns (ms per full step, #timed, dict)."""
    from oracle import ctsd as octsd
    cores = _host_cores()
    torch.set_num_threads(cores)
    cfg = load_config(small)
    B, T, V, C, H, W = cfg["latent_shape"]
    mcfg = dict(cfg["model"])
    t0 = time.perf_counter()
    # Build cost only (not timed work): the sin/cos position table is zeroed below anyway, so
    # its 38 s float64 numpy evaluation is skipped; the large weights are views into ONE
    # 128 MB N(0, 0.02) buffer instead of 15 GB of first-touch pages (this can only favour
    # the CPU arm: its weights stay cache-resident).
    import numpy as np
    from oracle import d31
    real_sincos = d31.get_2d_sincos_pos_embed
    d31.get_2d_sincos_pos_embed = lambda dim, grid, **kw: np.zeros((grid * grid, dim), np.float32)
    try:
        with torch.device("meta"):
            model = octsd.DiTCrossviewTemporalConditionModel(**mcfg)
    finally:
        d31.get_2d_sincos_pos_embed = real_sincos
    pattern = torch.randn(1 << 25, generator=torch.Generator().manual_seed(0)) * 0.02
    with torch.no_grad():
        for mod in model.modules():
            for name, p in list(mod._parameters.items()):
                if p is None:
                    continue
                if p.dim() == 1 and name == "weight":
                    new = torch.ones(p.shape)
                elif name in ("bias", "mix_factor") or p.numel() > pattern.numel():
                    new = torch.zeros(p.shape)
                else:
                    new = pattern[:p.numel()].view(p.shape)
                mod._parameters[name] = torch.nn.Parameter(new, requires_grad=False)
            for name, b in list(mod._buffers.items()):
                if b is not None and b.is_meta:
                    mod._buffers[name] = torch.zeros(b.shape, dtype=b.dtype)
    model.eval()
    t_build = time.perf_counter() - t0
    Ts, items = 1, V
    cond = synthetic_conditions(cfg, 1, Ts, V, "cpu", torch.float32)
    sample = torch.randn(1, Ts, V, C, H, W)
    timestep = torch.full((1, Ts, V), 500.0)
    times = []
    t_loop = time.perf_counter()
    with torch.no_grad():
        for k in range(warm + n_timed):
            t0 = time.perf_counter()
            model(sample, timestep, **cond)
            dt = time.perf_counter() - t0
            if k >= warm:
                times.append(dt)
            if times and time.perf_counter() - t_loop + dt > budget_s:
                break
    full_items = 2 * B * T * V
    ms = statistics.mean(times) * 1000.0 * full_items / items
    info = {"value": 1000.0 / ms, "unit": "steps/s", "cores": cores, "kind": "port",
            "sample": "oracle fp32 full-depth DiT forward incl. ImageAdapter on 1 frame x "
                      "%d views (no CFG) = %d of %d view-frame items per timed forward, "
                      "scaled x%d; %d warm-up + %d timed forwards (budget %d s); model build "
                      "%.0f s" % (V, items, full_items, full_items // items, warm, len(times),
                                  int(budget_s), t_build)}
    return ms, len(times), info


def cpu_baseline(budget_s=30.0, small=False):
    """`cpu_baseline` of the native arm: the same sample definition as `--impl reference`,
    one warm-up and at most two timed forwards inside `budget_s`."""
    return _cpu_reference_sample(small, 2, 1, budget_s)[2]


def run_reference(args):
    """Reference arm (rank 0 only): see `_cpu_reference_sample`."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cfg = load_config(args.small)
    B, T, V, C, H, W = cfg["latent_shape"]
    warm = min(args.warmup, 1)
    ms, n_timed, info = _cpu_reference_sample(args.small, args.steps, warm, 150.0)
    line = {
        "impl": "reference", "metric": METRIC, "value": 1000.0 / ms, "unit": "steps/s",
        "n_gpus": args.gpus, "steps": n_timed, "warmup": warm,
        "steps_requested": args.steps, "warmup_requested": args.warmup,
        "ms_per_step": ms, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "ctsd_35 DFoT 6-view x 16-frame with layout",
                   "latent_shape": [2 * B, T, V, C, H, W]},
        "cpu_baseline": info,
        "e2e": {"value": 1000.0 / ms, "unit": "steps/s", "h2d_bytes_per_step": 0,
                "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def main():
    if os.environ.get("DWM_BENCH_WATCHDOG"):      # debugging aid: dump all stacks and exit
        import faulthandler
        faulthandler.dump_traceback_later(float(os.environ["DWM_BENCH_WATCHDOG"]), exit=True)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--dtype", default="fp16", choices=["bf16", "fp16"],
                    help="compute dtype of the GEMM / attention operands; fp16 is the "
                         "reference's own (model_dtype torch.float16 + cuda autocast in "
                         "examples/ctsd_35_df16_*.json) and the headline; bf16 is reported "
                         "beside it (`other_dtype`)")
    ap.add_argument("--small", action="store_true", help="debug-size model/shape")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--graph", type=int, default=1,
                    help="1: the end-to-end loop replays the step from a CUDA graph")
    ap.add_argument("--cpu-budget", type=float, default=30.0)
    ap.add_argument("--no-extras", action="store_true",
                    help="skip streaming_e2e / workloads / eager_gpu_baseline / other dtype")
    ap.add_argument("--profile-dump", default=None,
                    help="write per-shape GEMM timing of the timed steps to this JSON")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write the latents of the last step to "
                         "DIR/latents.npy (float32)")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "native":
        ap.error("--dump-outputs records the native step; it has no meaning with --impl reference")
    if args.impl == "reference":
        run_reference(args)
    else:
        if args.warmup < 3 and not args.small:
            args.warmup = 3
        run_native(args)


if __name__ == "__main__":
    main()
