"""Multi-GPU parity check (run under torchrun, one rank per GPU):

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      --master-port 29533 tools/shard_check.py

Every rank builds the same seeded small DiT, runs diffusion-forcing denoise steps with the
CFG x frame sharding plan, and the gathered latents are compared with an unsharded run of
the same steps on rank 0.  Exit code 0 = match.  `--unet` checks the CTSD-2.1 UNet instead
(`unet_main`).

`--views` adds the view axis to the plan (CFG x views x frames, the split `ShardPlan` picks, or
`--view-ways K`): cross-view blocks then gather their K,V over the view group.

`--count [--world N] [--frames T] [--views V]` runs no GPU work: it prints, for the DiT plans of
N GPUs, the K,V exchanges per denoise step and the bytes each rank sends in them (CTSD-3.5 DiT:
6 cross-view and 12 temporal blocks, D = 1536, 16 x 28 patches per view, 16-bit K,V), for
config 2's image window (T = 1) and config 5's 5 latent frames by default."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def _arg(name, default):
    return int(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def count_main():
    """--count: K,V exchanges per step and bytes sent per rank, from shapes (no GPU)."""
    from opendwm_b200.sharding import ShardPlan
    D, S, n_cv, n_tp, eb = 1536, 16 * 28, 6, 12, 2
    worlds = [_arg("--world", 0)] if "--world" in sys.argv else [2, 4, 8]
    windows = [(_arg("--frames", 5), _arg("--views", 6))] if "--frames" in sys.argv else \
        [(1, 6), (5, 6)]
    for T, V in windows:
        for world in worlds:
            for views in (None, V):
                try:
                    p = ShardPlan(world, 0, T, make_groups=False, views=views)
                except ValueError as e:
                    print("count T=%d V=%d world=%d views=%s: %s" % (T, V, world, views, e))
                    continue
                V_loc = V if views is None else max(p.v_counts)
                T_loc = max(p.counts)
                rows = T_loc * V_loc * S                     # largest shard, one CFG branch
                kv = rows * 2 * D * eb
                cv = n_cv if p.v_ways > 1 else 0
                tp = n_tp if p.t_ways > 1 else 0
                sent = cv * kv * (p.v_ways - 1) + tp * kv * (p.t_ways - 1)
                print("count T=%d V=%d world=%d plan=%s largest_shard_items=%d "
                      "crossview_exchanges=%d temporal_exchanges=%d cfg_exchanges=%d "
                      "MB_sent_per_rank_per_step=%.1f" % (
                          T, V, world, p.parallelism, T_loc * V_loc, cv, tp,
                          1 if p.cfg_ways > 1 else 0, sent / 1e6))


def main():
    from common import TINY, synthetic_inputs
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    from opendwm_b200.sharding import ShardPlan
    from opendwm_b200 import lib
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda")
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    V = 3
    use_cfg = os.environ.get("SHARD_CFG", "1") != "0"
    views = V if "--views" in sys.argv else None
    view_ways = _arg("--view-ways", None)
    t_ways = ShardPlan(world, 0, 64, cfg=use_cfg, make_groups=False, views=views,
                       view_ways=view_ways).t_ways
    # (frames, temporal attention type): 8 = even shards; 5 / 11 / 19 = the uneven shards of
    # BASELINE configs 5 and 3 (19 with row-wise temporal attention as in config 3); full
    # temporal attention on even and uneven shards
    cases = [(8, "pointwise"), (5, "pointwise"), (11, "pointwise"), (19, "pointwise"),
             (19, "rowwise"), (5, "rowwise"), (8, "full"), (5, "full")]
    cases = [c for c in cases if c[0] >= t_ways]
    # row-wise / full sequences longer than 64 take the wgmma kernel when unsharded and the
    # separate-K,V mma.sync kernel when sharded; with attn_tc = 0 both runs use the same kernel
    # and the comparison is bit for bit
    lib.set_option("attn_tc", 0)
    worst, all_equal = 0.0, True
    for T, kind in cases:
        cfg = dict(TINY, temporal_attention_type=kind)
        torch.manual_seed(0)
        model = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.float16)
        g = torch.Generator().manual_seed(1)
        with torch.no_grad():
            for name, p in model.named_parameters():
                if name.endswith("mix_factor"):
                    p.fill_(0.3)
                elif p.dim() == 1 and name.endswith(".weight"):
                    p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
                else:
                    p.copy_(0.05 * torch.randn(p.shape, generator=g))
        steps = 2 * T
        inf = {"guidance_scale": 2.0, "inference_steps": steps,
               "sequence_length_per_iteration": T}
        pipe = StreamingCrossviewTemporalSD(
            None, {"generator_seed": 0}, dev, {"frame_prediction_style": "diffusion_forcing"},
            {}, inf, None, model, model_dtype=torch.float16)
        pipe.reset_streaming((1, T, V, 16, 8, 12), "pt")
        sample, _, cond = synthetic_inputs(cfg, B=2, T=T, V=V, device="cuda")
        cond = {k: (v.half() if v.is_floating_point() and k != "added_time_ids" else v)
                for k, v in cond.items()}
        latents0 = sample[:1].float().contiguous()
        spi = steps // T

        def run(plan):
            pipe.sharding = plan
            pipe.model._cond_key = None
            lat = latents0.clone() if plan is None else plan.local_latents(latents0)
            c = cond if plan is None else plan.local_conditions(cond, cfg_doubled=True)
            fs = slice(0, T) if plan is None else plan.frame_slice()
            vs = slice(None) if plan is None else plan.view_slice()
            for i in (steps - 3, steps - 2, steps - 1):
                idx, ts, in_range = pipe._df_step_tensors(i, T, spi, 0, 1, V)
                pipe.denoise_step(lat, c, idx[:, fs, vs].contiguous(),
                                  ts[:, fs, vs].contiguous(), in_range[fs].contiguous())
            return lat if plan is None else plan.gather_latents(lat)

        plan = ShardPlan(world, rank, T, cfg=use_cfg, views=views, view_ways=view_ways)
        sharded = run(plan)
        ref = run(None)
        err = ((sharded - ref).abs().max() / ref.abs().max()).item()
        moved = ((ref - latents0).abs().max()).item()
        t = torch.tensor([err, 0.0 if torch.equal(sharded, ref) else 1.0,
                          0.0 if moved > 1e-3 else 1.0], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        worst = max(worst, t[0].item())
        all_equal = all_equal and t[1].item() == 0.0 and t[2].item() == 0.0
        if rank == 0:
            print("shard_check world=%d plan=%s T=%d shards=%s view_shards=%s temporal=%s "
                  "peer_scatter=%s bit_identical=%s max_rel_err=%.3e (latents moved %.3f)" % (
                      world, plan.parallelism, T, plan.counts, plan.v_counts, kind,
                      plan.use_peer_scatter and (plan.t_ways > 1 or plan.v_ways > 1),
                      t[1].item() == 0.0, t[0].item(), moved), flush=True)
        del pipe, model
        torch.cuda.empty_cache()
    dist.destroy_process_group()
    sys.exit(0 if all_equal and worst == 0.0 else 1)


def unet_main():
    """--unet: every rank's sharded noise prediction of the CTSD-2.1 UNet (its CFG branch and
    frames) against its own unsharded forward, relative to the output's range (GroupNorm
    statistics are atomics, so within 2e-3 in 16 bit and 8e-2 in E4M3 rather than bit for bit).  Run it with and
    without DWM_PEER_SCATTER=0 to check the symmetric-memory halo and K,V stores across GPUs."""
    from test_unet_sharded_gpu import _forward, _forward_inputs, _model
    from opendwm_b200.sharding import ShardPlan
    from opendwm_b200 import lib
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda")
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    lib.set_option("attn_tc", 0)
    t_ways = world // (2 if world >= 2 else 1)
    cases = [(v, T, fp8) for v, T, fp8 in [("video", 8, False), ("video", 5, False),
                                           ("pointwise", 11, False), ("video", 8, True)]
             if T >= t_ways]
    ok = True
    for variant, T, fp8 in cases:
        m = _model(variant, fp8)
        x, t, c = _forward_inputs(T)
        ref = _forward(m, x, t, c)
        plan = ShardPlan(world, rank, T)
        fs = plan.frame_slice()
        half = slice(None) if plan.cfg_ways == 1 else slice(plan.cfg_rank, plan.cfg_rank + 1)
        m.shard = plan
        got = _forward(m, x[half, fs].contiguous(), t[half, fs].contiguous(),
                       plan.local_conditions(c, cfg_doubled=True))
        m.shard = None
        err = torch.tensor([((got - ref[half, fs]).abs().max() / ref.abs().max()).item()],
                           device=dev)
        dist.all_reduce(err, op=dist.ReduceOp.MAX)
        tol = 8e-2 if fp8 else 2e-3
        ok = ok and err.item() <= tol
        if rank == 0:
            print("shard_check unet world=%d plan=%s T=%d shards=%s temporal=%s e4m3=%s "
                  "peer_scatter=%s max_rel_err=%.3e (tolerance %.0e)" % (
                      world, plan.parallelism, T, plan.counts, variant, fp8,
                      plan.use_peer_scatter and plan.t_ways > 1, err.item(), tol), flush=True)
        del m
        torch.cuda.empty_cache()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    if "--count" in sys.argv:
        count_main()
    elif "--unet" in sys.argv:
        unet_main()
    else:
        main()
