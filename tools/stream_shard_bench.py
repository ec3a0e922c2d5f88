"""Per-frame latency of the north-star streaming loop under a ShardPlan (one rank per GPU):

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \\
      --master-port 29533 tools/stream_shard_bench.py [--frames 8] [--check]

Every rank builds the same random-init north-star DiT and SD-3.5-shaped AutoencoderKL, attaches
`ShardPlan(N, rank, 16, cfg=True)` (also at N = 1, so the plan's code path is what is timed)
and drives `StreamingCrossviewTemporalSD.send_frame_condition` / `receive_frame` with host frame
data: the 16-frame fill (the last gathering call runs the 48-step warm-up), then `--frames`
emitted frames after one untimed warm-up frame.  A frame's time is the host clock around the
call pair plus the copy of the decoded views to the host, synchronised on both sides: 3
denoise steps, the condition-cache ring update, the FIFO all-gather and the item-parallel VAE
decode.

`--views` attaches `ShardPlan(N, rank, 16, cfg=True, views=6)` instead (the split of the view
and frame axes the plan picks, or `--view-ways K`).

`--check`: the FIFO latents after every call are also kept on rank 0, which then streams the
same frames without a plan and compares them bit for bit.

Prints one JSON line on rank 0: ms per frame (rank 0's mean, and the slowest rank's), the plan,
the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def _power_limit(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _stream(pipe, cfg, n_fill, n_frames, keep_fifo, timed):
    """Fill, then n_frames + 1 emitted frames; returns (seconds per timed frame, FIFO list)."""
    from bench_extras import frame_batch
    B, T, V, C, H, W = cfg["latent_shape"]
    m = cfg["model"]
    g = torch.Generator().manual_seed(3)
    pipe.generator.manual_seed(0)
    pipe.reset_streaming((B, T, V, C, H, W), "pt")
    secs, fifo = [], []
    for t in range(n_fill + n_frames + 1):
        fb = frame_batch(g, V, (H * 8, W * 8), cfg["text_tokens"], m["joint_attention_dim"],
                         m["pooled_projection_dim"], t)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe.send_frame_condition(fb)
        img = pipe.receive_frame()
        host = None if img is None else img.cpu()
        dt = time.perf_counter() - t0
        if timed and t > n_fill:                 # the first emitted frame warms the ring path
            secs.append(dt)
        assert (host is None) == (t < n_fill - 1), t
        if keep_fifo and pipe.latents is not None:
            fifo.append(pipe.latents.cpu())
    return secs, fifo


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=8, help="timed emitted frames after the fill")
    ap.add_argument("--check", action="store_true",
                    help="compare the FIFO after every call with an unsharded stream on rank 0")
    ap.add_argument("--dtype", choices=["bf16", "fp16"], default="fp16")
    ap.add_argument("--small", action="store_true", help="4-layer model, 4 frames (smoke)")
    ap.add_argument("--views", action="store_true",
                    help="plan with the view axis (CFG x views x frames)")
    ap.add_argument("--view-ways", type=int, default=None, help="force the view split")
    args = ap.parse_args()

    import bench
    from bench_extras import _blocks
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    from opendwm_b200.sharding import ShardPlan

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("stream_shard_bench needs a GPU")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    cfg = bench.load_config(args.small)
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[args.dtype]
    B, T, V, C, H, W = cfg["latent_shape"]
    torch.set_default_dtype(dtype)
    with torch.device(dev):
        model = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
    torch.set_default_dtype(torch.float32)
    bench.init_weights_(model)
    torch.manual_seed(0)
    with torch.device(dev):
        vae = AutoencoderKL(
            block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=C,
            norm_num_groups=32, scaling_factor=1.5305, shift_factor=0.0609,
            use_quant_conv=False, use_post_quant_conv=False, compute_dtype=dtype)
    blk = _blocks()["ctsd_35_df16_6views_video_generation_with_layout.json"]["pipeline"]
    common = {k: v for k, v in blk["common_config"].items()
              if k not in ("autocast", "text_encoder_load_args")}
    common["vae_instance"] = vae
    inf = dict(blk["inference_config"])
    inf.update(guidance_scale=cfg["guidance_scale"], inference_steps=cfg["inference_steps"],
               sequence_length_per_iteration=T)

    def pipeline(plan):
        pipe = StreamingCrossviewTemporalSD(None, {"generator_seed": 0}, dev, common, {}, inf,
                                            None, model, model_dtype=dtype)
        pipe.sharding = plan
        return pipe

    plan = ShardPlan(world, rank, T, cfg=True, views=V if args.views else None,
                     view_ways=args.view_ways)
    secs, fifo = _stream(pipeline(plan), cfg, T, args.frames, args.check, timed=True)
    mean = sum(secs) / len(secs)
    slowest = mean
    if world > 1:
        t = torch.tensor([mean], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        slowest = t.item()
    res = {"tool": "stream_shard_bench", "world": world, "parallelism": plan.parallelism,
           "frame_shards": plan.counts, "peer_scatter": plan.use_peer_scatter and plan.t_ways > 1,
           "latent_shape": [B, T, V, C, H, W], "dtype": args.dtype,
           "ms_per_frame": mean * 1e3, "ms_per_frame_slowest_rank": slowest * 1e3,
           "ms_per_frame_min": min(secs) * 1e3, "ms_per_frame_max": max(secs) * 1e3,
           "frames": len(secs), "denoise_steps_per_frame": cfg["inference_steps"] // T,
           "gpu": torch.cuda.get_device_name(dev), "power_limit": _power_limit(local_rank)}
    if args.check:
        if world > 1:
            dist.barrier()
        if rank == 0:
            _, want = _stream(pipeline(None), cfg, T, args.frames, True, timed=False)
            same = len(want) == len(fifo) and all(torch.equal(a, b) for a, b in zip(fifo, want))
            err = max(((a - b).abs().max() / b.abs().max()).item() for a, b in zip(fifo, want))
            res["check"] = {"fifo_states": len(want), "bit_identical": same,
                            "max_rel_err": err}
        if world > 1:
            dist.barrier()
    if rank == 0:
        print(json.dumps(res), flush=True)
    if world > 1:
        dist.destroy_process_group()
    if args.check and rank == 0 and not res["check"]["bit_identical"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
