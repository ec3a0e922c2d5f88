"""The CTSD-2.1 UNet under a ShardPlan, with world-2 and world-4 process groups sharing one GPU
(gloo, DWM_PEER_SCATTER=0: the statistics / amax all-reduces, the halo point-to-point
exchange and the K,V all-gather replace the symmetric-memory stores).

Every rank's noise prediction (its CFG branch and frames) and every rank's `inference_pipeline`
latents (CFG + DDIM, gathered window) are compared with the unsharded run.  The UNet's GroupNorm
statistics are summed with atomics and the shards sum theirs in another order, so the runs are
not bit-identical: the tolerance is twice the unsharded run's own run-to-run spread, measured
here, and at least the spread DESIGN §7 documents (2e-3 of the output's range in 16 bit, 8e-2 in
E4M3).  Cases: the video configuration of tests/test_unet.py (row-wise temporal attention) and
its point-wise temporal attention variant, even and uneven shards, the CFG split on and off,
16-bit and E4M3; T = 1 on two ranks shards the CFG branches only."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
V, STEPS = 2, 2


def _model(variant, fp8):
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from test_unet import UCFG, _oracle
    cfg = dict(UCFG)
    if variant == "pointwise":
        # point-wise temporal attention; cross-view stays row-wise (rank-local either way) so
        # that the pipeline's view mask applies
        cfg.update(enable_rowwise_temporal=False)
    m = U(**cfg, compute_dtype=torch.float16,
          gemm_dtype=torch.float8_e4m3fn if fp8 else None)
    m.load_state_dict(_oracle(cfg).state_dict())
    return m.cuda()


def _forward_inputs(T):
    """CFG-doubled (B = 2: [uncond ; cond]) model inputs of a T-frame window."""
    from test_unet import _inputs
    x, t, c = _inputs(2, T, V)
    return x.cuda(), t.cuda(), {k: None if v is None else v.cuda() for k, v in c.items()}


def _forward(m, x, t, c):
    return m(x, t, **c)[0][0].float()


def _pipe(m, T):
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from test_pipeline_gpu import COMMON, _batch
    common = dict(COMMON, frame_prediction_style="ctsd")
    inf = {"guidance_scale": 3.0, "inference_steps": STEPS}
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {}, inf, None, m,
                               model_dtype=torch.float32)
    batch = _batch(T, V, dict(joint_attention_dim=96, pooled_projection_dim=8), hw=(128, 192))
    return pipe, batch


def _pipeline(m, T):
    pipe, batch = _pipe(m, T)
    return pipe.inference_pipeline((1, T, V, 4, 16, 24), batch, "pt")["latents"]


def _worker(rank, world, port, variant, T, cfg, fp8, want_pred, want_lat, tol_pred, tol_lat):
    from opendwm_b200 import lib
    from opendwm_b200.sharding import ShardPlan
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DWM_PEER_SCATTER="0")
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lib.set_option("attn_tc", 0)
        m = _model(variant, fp8)
        plan = ShardPlan(world, rank, T, cfg=cfg)
        if T == 1:
            assert (plan.cfg_ways, plan.t_ways) == (2, 1)
        # noise prediction of this rank's CFG branch and frames
        x, t, c = _forward_inputs(T)
        fs = plan.frame_slice()
        half = slice(None) if plan.cfg_ways == 1 else \
            slice(plan.cfg_rank, plan.cfg_rank + 1)
        c = plan.local_conditions(c, cfg_doubled=True)
        m.shard = plan
        got = _forward(m, x[half, fs].contiguous(), t[half, fs].contiguous(), c).cpu()
        err = (got - want_pred[half, fs]).abs().max().item()
        assert err <= tol_pred, ("prediction", rank, err, tol_pred)
        # the whole window through the pipeline: every rank holds the gathered latents
        m.shard = None
        pipe, batch = _pipe(m, T)
        pipe.sharding = plan
        lat = pipe.inference_pipeline((1, T, V, 4, 16, 24), batch, "pt")["latents"].cpu()
        err = (lat - want_lat).abs().max().item()
        assert err <= tol_lat, ("pipeline", rank, err, tol_lat)
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


CASES = [
    ("video", 2, 4, False, False),      # frames 2 + 2, row-wise temporal attention
    ("video", 4, 5, True, False),       # CFG 2 x frames 3 + 2
    ("pointwise", 4, 5, False, False),  # frames 2 + 1 + 1 + 1
    ("pointwise", 2, 3, False, True),   # E4M3, frames 2 + 1
    ("video", 4, 4, True, True),        # E4M3, CFG 2 x frames 2 + 2
    ("video", 2, 1, True, False),       # image (T = 1): CFG branches only
]
IDS = ["video_w2_frames2+2", "video_cfg2xframes3+2", "pointwise_frames2+1+1+1",
       "pointwise_e4m3_frames2+1", "video_e4m3_cfg2xframes2+2", "image_cfg_only"]


@pytest.mark.parametrize("variant,world,T,cfg,fp8", CASES, ids=IDS)
def test_sharded_unet_matches_unsharded(variant, world, T, cfg, fp8):
    from opendwm_b200 import lib
    lib.set_option("attn_tc", 0)      # the sharded temporal attention is the mma.sync kernel
    try:
        m = _model(variant, fp8)
        x, t, c = _forward_inputs(T)
        preds = [_forward(m, x, t, c) for _ in range(2)]
        lats = [_pipeline(m, T) for _ in range(2)]
    finally:
        lib.set_option("attn_tc", -1)
    floor = 8e-2 if fp8 else 2e-3

    def tol(a, b):
        return 2 * max((a - b).abs().max().item(), floor * a.abs().max().item())
    tol_pred, tol_lat = tol(*preds), tol(*lats)
    port = 29100 + (os.getpid() % 400)
    mp.spawn(_worker, args=(world, port, variant, T, cfg, fp8, preds[0].cpu(), lats[0].cpu(),
                            tol_pred, tol_lat), nprocs=world, join=True)
