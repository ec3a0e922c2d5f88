"""The CTSD-2.1 UNet under a ShardPlan with a view axis, with gloo process groups sharing one GPU
(DWM_PEER_SCATTER=0: the cross-view K,V all-gather over the view group, and for a video window
the frame group's statistics / amax all-reduces, halo exchange and temporal K,V all-gather).

Every rank's noise prediction (its CFG branch, frames and views) and every rank's
`inference_pipeline` latents are compared with the unsharded run, within twice the unsharded
run's own run-to-run spread (GroupNorm statistics are summed with atomics) and at least the
spread DESIGN §7 documents, as tests/test_unet_sharded_gpu.py does.  Cases: the image window
of config 2's shape (T = 1, 6 views) at cfg2 x views2 and cfg2 x views3, and a video window at
cfg2 x views2 x frames2."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_unet_sharded_gpu import _forward, _model

pytestmark = pytest.mark.gpu
V, STEPS = 6, 2


def _forward_inputs(T):
    from test_unet import _inputs
    x, t, c = _inputs(2, T, V)
    return x.cuda(), t.cuda(), {k: None if v is None else v.cuda() for k, v in c.items()}


def _pipeline(m, T, plan=None):
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from test_pipeline_gpu import COMMON, _batch
    common = dict(COMMON, frame_prediction_style="ctsd")
    inf = {"guidance_scale": 3.0, "inference_steps": STEPS}
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {}, inf, None, m,
                               model_dtype=torch.float32)
    batch = _batch(T, V, dict(joint_attention_dim=96, pooled_projection_dim=8), hw=(128, 192))
    pipe.sharding = plan
    return pipe.inference_pipeline((1, T, V, 4, 16, 24), batch, "pt")["latents"]


def _worker(rank, world, port, T, view_ways, want_pred, want_lat, tol_pred, tol_lat):
    from opendwm_b200 import lib
    from opendwm_b200.sharding import ShardPlan
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DWM_PEER_SCATTER="0")
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lib.set_option("attn_tc", 0)
        m = _model("video", False)
        plan = ShardPlan(world, rank, T, cfg=True, views=V, view_ways=view_ways)
        assert plan.v_ways == view_ways
        x, t, c = _forward_inputs(T)
        fs, vs = plan.frame_slice(), plan.view_slice()
        half = slice(plan.cfg_rank, plan.cfg_rank + 1)
        c = plan.local_conditions(c, cfg_doubled=True)
        assert c["crossview_attention_mask"].shape[-2:] == (V, V)
        m.shard = plan
        got = _forward(m, x[half, fs, vs].contiguous(), t[half, fs, vs].contiguous(), c).cpu()
        err = (got - want_pred[half, fs, vs]).abs().max().item()
        assert err <= tol_pred, ("prediction", rank, err, tol_pred)
        m.shard = None
        lat = _pipeline(m, T, plan).cpu()
        err = (lat - want_lat).abs().max().item()
        assert err <= tol_lat, ("pipeline", rank, err, tol_lat)
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,T,view_ways", [(4, 1, 2), (6, 1, 3), (8, 4, 2)],
                         ids=["image_cfg2xviews2", "image_cfg2xviews3",
                              "video_cfg2xviews2xframes2"])
def test_view_sharded_unet_matches_unsharded(world, T, view_ways):
    from opendwm_b200 import lib
    lib.set_option("attn_tc", 0)
    try:
        m = _model("video", False)
        x, t, c = _forward_inputs(T)
        preds = [_forward(m, x, t, c) for _ in range(2)]
        lats = [_pipeline(m, T) for _ in range(2)]
    finally:
        lib.set_option("attn_tc", -1)

    def tol(a, b):
        return 2 * max((a - b).abs().max().item(), 2e-3 * a.abs().max().item())
    port = 29100 + (os.getpid() % 400)
    mp.spawn(_worker, args=(world, port, T, view_ways, preds[0].cpu(), lats[0].cpu(),
                            tol(*preds), tol(*lats)), nprocs=world, join=True)
