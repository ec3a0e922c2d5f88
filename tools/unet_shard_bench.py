"""Times the CTSD-2.1 UNet denoise step (eager, CFG 3, DDIM) unsharded and through a ShardPlan.

  python tools/unet_shard_bench.py [steps]                      # one GPU: world 1
  python -m torch.distributed.run --nproc-per-node N tools/unet_shard_bench.py [steps]
  ... tools/unet_shard_bench.py [steps] --views       # plans with the view axis (views=6)

Workloads: BASELINE config 2, the 6-view image step [2,1,6,4,32,56] (temporal blocks off), and a
16-frame video step [2,16,6,4,32,56] with temporal ResBlocks and row-wise temporal attention.
On one GPU the unsharded step and the step through a world-1 plan alternate over several rounds
(the plan's overhead is judged against the rounds' spread).  Under torchrun every rank times the
sharded step; rank 0 prints it.  Each line also gives the exchanges per step and rank: count
and bytes of the GroupNorm statistics / amax all-reduces and halo frames of every temporal conv,
the K,V of every temporal attention block, and the CFG prediction exchange, counted from the
shapes; with --views also the K,V of every cross-view block over the view group.  The GPU name
and power limit are printed with the numbers."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "src"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from unet_bench import MODEL  # noqa: E402

WORKLOADS = [("config2_image", 1, True), ("video_16f", 16, False)]


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                               "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def exchanges(plan, B, T, V, H, W, image, elem=2):
    """(count, bytes) this rank sends per step, from the UNet's shapes."""
    boc, n = MODEL["block_out_channels"], len(MODEL["block_out_channels"])
    B_loc = B // plan.cfg_ways
    V = V if plan.V is None else plan.V_loc       # the views this rank holds
    nb = B_loc * V
    count = nbytes = 0
    if plan.cfg_ways == 2:      # the branch prediction [B_loc, T_loc, V, 4, H, W] fp32
        count, nbytes = 1, B_loc * plan.T_loc * V * 4 * H * W * 4
    temporal = plan.t_ways > 1 and not image
    nbr = (plan.t_rank > 0) + (plan.t_rank + 1 < plan.t_ways)
    # temporal ResBlocks per level: down (layers_per_block), mid 2, up (layers_per_block + 1);
    # temporal / cross-view attention blocks per level: one per CrossAttn ResBlock (levels
    # 0..2) + mid 1
    lpb = MODEL["layers_per_block"]
    res = [lpb + (lpb + 1) for _ in range(n)]
    res[n - 1] += 2
    attn = [2 * lpb + 1 if i < n - 1 else 0 for i in range(n)]
    attn[n - 1] += 1
    h, w = H, W
    for i, c in enumerate(boc):
        kv = B_loc * plan.T_loc * V * h * w * 2 * c * elem
        if temporal:
            frame = nb * h * w * c * elem
            convs = 2 * res[i]
            count += convs * (1 + nbr)                 # sums all-reduce + halo frames
            nbytes += convs * (nb * 32 * 2 * 8 + nbr * frame)
            count += attn[i]
            nbytes += attn[i] * kv * (plan.t_ways - 1)
        if plan.v_ways > 1:                            # cross-view K,V over the view group
            count += attn[i]
            nbytes += attn[i] * kv * (plan.v_ways - 1)
        h, w = (h + 1) // 2, (w + 1) // 2
    return count, nbytes


def main():
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from opendwm_b200.sharding import ShardPlan
    steps = next((int(a) for a in sys.argv[1:] if a.isdigit()), 5)
    views = 6 if "--views" in sys.argv else None
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dev = torch.device("cuda")
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    dtype = torch.bfloat16
    torch.manual_seed(0)
    with torch.device(dev):
        m = U(**MODEL, compute_dtype=dtype)
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("mix_factor"):
                continue
            if p.dim() == 1 and n.endswith(".weight"):
                p.fill_(1.0)
            elif n.endswith(".bias"):
                p.zero_()
            else:
                p.copy_(torch.randn(p.shape, generator=g, device="cuda") * 0.02)
    pipe = CrossviewTemporalSD(
        None, {"generator_seed": 0}, dev, {"frame_prediction_style": "ctsd"}, {},
        {"guidance_scale": 3, "inference_steps": 50}, None, m, model_dtype=dtype)
    pipe.test_scheduler.set_timesteps(50, dev)
    gpu = _gpu()
    for name, T, image in WORKLOADS:
        B, V, H, W = 1, 6, 32, 56
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
            disable_temporal=torch.full((2 * B,), image, dtype=torch.bool, device=dev),
            crossview_attention_mask=ring.unsqueeze(0).repeat(2 * B, 1, 1).to(dev),
            added_time_ids=torch.randn(2 * B, T, V, 11, generator=gen).to(dev))
        lat0 = torch.randn(B, T, V, 4, H, W, generator=gen).to(dev)
        ts = [pipe.test_scheduler.timesteps[k].to(torch.int32).expand(B, T, V).contiguous()
              for k in range(50)]

        def timed(plan):
            pipe.sharding = plan
            m._cond_key = None
            c = cond if plan is None else plan.local_conditions(cond, cfg_doubled=True)
            lat = lat0.clone() if plan is None else plan.local_latents(lat0)
            fs = slice(0, T) if plan is None else plan.frame_slice()
            vs = slice(None) if plan is None else plan.view_slice()
            pipe.denoise_step(lat, c, None, ts[0][:, fs, vs].contiguous(), None)     # warm-up
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(steps):
                pipe.denoise_step(lat, c, None, ts[1 + k][:, fs, vs].contiguous(), None)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / steps
        res = dict(workload=name, shape=[2 * B, T, V, 4, H, W], gpu=gpu, world=world,
                   steps=steps)
        if world == 1:
            plan = ShardPlan(1, 0, T, make_groups=False, views=views)
            rounds = [(timed(None), timed(plan)) for _ in range(3)]
            base = [a for a, _ in rounds]
            res.update(ms_unsharded=base, ms_plan_world1=[b for _, b in rounds],
                       spread_unsharded_ms=max(base) - min(base),
                       multi_gpu="not measured (one GPU)")
        else:
            plan = ShardPlan(world, rank, T, views=views)
            ms = timed(plan)
            cnt, nbytes = exchanges(plan, 2 * B, T, V, H, W, image)
            res.update(plan=plan.parallelism, shards=plan.counts, view_shards=plan.v_counts,
                       ms_sharded=ms,
                       peer_scatter=plan.use_peer_scatter, exchanges_per_step_rank0=cnt,
                       exchange_bytes_per_step_rank0=nbytes)
        if world == 1:
            for w in (2, 4, 8):
                if T >= w // 2 or views is not None:
                    p = ShardPlan(w, 0, T, make_groups=False, views=views)
                    cnt, nbytes = exchanges(p, 2 * B, T, V, H, W, image)
                    res["exchanges_rank0_world%d" % w] = dict(plan=p.parallelism, count=cnt,
                                                              bytes=nbytes)
        if rank == 0:
            print(json.dumps(res), flush=True)
    pipe.sharding = None
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
