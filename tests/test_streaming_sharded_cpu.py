"""The streaming FIFO (`StreamingCrossviewTemporalSD`) under a ShardPlan, on CPU processes over
gloo: gathering phase, streaming frames and the flush emit, on every rank, the frames and FIFO
latents of the unsharded pipeline bit for bit.

The denoise step is a stand-in whose update depends only on a frame's own conditions, its
sigma index and the CFG branch, and which exchanges the branch predictions through the plan the
way the real step does; so a wrong frame slice, a stale condition slice, a missed gather or a
mis-ordered decode changes the result."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from common import CONDITION_COMMON, condition_batch  # noqa: E402

V = 3


def _run(fn, world, *args):
    port = 28500 + (os.getpid() % 500)
    mp.spawn(_entry, args=(fn, world, port, args), nprocs=world, join=True)


def _entry(rank, fn, world, port, args):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fn(rank, world, *args)
    finally:
        dist.destroy_process_group()


class _FakeVae:
    class config:
        scaling_factor, shift_factor = 0.5, 0.25
        down_block_types = ("D",) * 4          # 8x down-sampling: 16 x 24 images, 2 x 3 latents
        latent_channels = 4
    dtype = torch.float32

    def decode(self, x, return_dict=False):
        return (x[:, :3] * 2 + 1,)


def _stream_pipe(plan, T, model=None):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm import _compat
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    pipe = object.__new__(StreamingCrossviewTemporalSD)
    pipe.config = {"generator_seed": 0}
    pipe.common_config = dict(CONDITION_COMMON, added_time_ids="fps_camera_transforms_action",
                              camera_ego_sensor_indices=[1, 2, 3])
    pipe.inference_config = {
        "guidance_scale": 2.0, "inference_steps": 3 * T, "sequence_length_per_iteration": T,
        "autoregression_data_exception_for_take_sequence": ["crossview_mask"],
        "autoregression_condition_exception_for_take_sequence": [
            "disable_crossview", "disable_temporal", "crossview_attention_mask",
            "camera_intrinsics_norm", "camera2referego"]}
    pipe.device, pipe.model_dtype = torch.device("cpu"), torch.float32
    pipe.generator = torch.Generator().manual_seed(0)
    pipe.model = model if model is not None else \
        object.__new__(DiTCrossviewTemporalConditionModel)
    pipe.is_dit = isinstance(pipe.model, _compat.SD3Transformer2DModelMarker)
    pipe.text_encoders = pipe.tokenizers = None
    pipe.is_temporal_vae, pipe.vae = False, _FakeVae()
    pipe.should_save = not dist.is_initialized() or dist.get_rank() == 0
    pipe.sharding, pipe._step_cache = plan, {}
    pipe.test_scheduler = type("S", (), {
        "timesteps": torch.linspace(1000, 50, 3 * T), "num_inference_steps": 3 * T,
        "init_noise_sigma": 1.0, "set_timesteps": lambda self, n, device=None: None})()

    def fake_step(latents, conditions, idx, timesteps, in_range=None):
        B, T_loc = latents.shape[:2]
        ids = conditions["added_time_ids"].float()     # [branches * B, T_loc, V, 13]
        assert ids.shape[1] == T_loc == idx.shape[1] == timesteps.shape[1]
        n = ids.shape[0] // B
        # per-branch prediction: the unconditional branch carries -1000 action ids
        pred = 1e-4 * ids.sum(-1) + timesteps.float().repeat(n, 1, 1) / 1000 + \
            1e-2 * idx.float().repeat(n, 1, 1)
        plan = pipe.sharding
        if plan is not None and plan.cfg_ways == 2:     # the partner holds the other branch
            both = torch.empty(2 * pred.numel())
            plan.gather_cfg_tokens(pred.contiguous().flatten(), both)
            pred = both.view(2 * B, T_loc, V)
        u, c = pred.chunk(2)
        new = latents * 0.9 + 0.1 * (u + 2.0 * (c - u))[..., None, None, None]
        if in_range is not None:
            new = torch.where(in_range.bool().view(1, -1, 1, 1, 1, 1), new, latents)
        latents.copy_(new)
        return latents
    pipe.denoise_step = fake_step
    return pipe


def _frames(T, n):
    batch = condition_batch(T=n, V=V)
    batch["vae_images"] = torch.rand(1, n, V, 3, 16, 24, generator=torch.Generator().manual_seed(3))
    from dwm.functional import take_sequence_clip
    skip = ["crossview_mask"]
    return batch, [{k: v if k in skip else take_sequence_clip(v, i, i + 1)
                    for k, v in batch.items()} for i in range(n)]


def _drive(pipe, T, frames):
    """Feeds the frames one by one, then flushes; returns (FIFO after every call, frames)."""
    pipe.reset_streaming((1, T, V, 4, 2, 3), "pt")
    fifo, out = [], []
    for f in frames + [None]:
        pipe.send_frame_condition(f)
        fifo.append(None if pipe.latents is None else pipe.latents.clone())
        while True:
            img = pipe.receive_frame()
            if img is None:
                break
            out.append(img)
    return fifo, out


def _sharded_stream(rank, world, T, tmp):
    from opendwm_b200.sharding import ShardPlan
    n = T + 3                                     # gathering + 3 streaming frames, then the flush
    batch, frames = _frames(T, n)
    want_fifo, want = _drive(_stream_pipe(None, T), T, frames)
    assert len(want) == n
    plan = ShardPlan(world, rank, T, cfg=True)
    pipe = _stream_pipe(plan, T)
    got_fifo, got = _drive(pipe, T, frames)
    assert len(got_fifo) == len(want_fifo)
    for k, (g, w) in enumerate(zip(got_fifo, want_fifo)):
        assert (g is None) == (w is None), k
        assert g is None or torch.equal(g, w), (rank, k)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), (rank, k)
    # the whole-clip entry points on the same plan, from the same seed
    pipe.generator.manual_seed(0)
    out = pipe.fifo_inference_pipeline((1, T, V, 4, 2, 3), batch, "pt")
    assert torch.equal(out["images"], torch.cat(want)), rank
    pipe.generator.manual_seed(0)
    out = pipe.preview_pipeline(batch, tmp, 0)
    assert torch.equal(out["images"], torch.cat(want)), rank


@pytest.mark.parametrize("world,T", [(2, 4), (4, 4), (4, 5), (8, 5)],
                         ids=["cfg2xframes1", "cfg2xframes2", "cfg2xframes2_T5_3+2",
                              "cfg2xframes4_T5_2+1+1+1"])
def test_sharded_stream_matches_unsharded(world, T, tmp_path):
    _run(_sharded_stream, world, T, str(tmp_path))
    assert os.listdir(os.path.join(tmp_path, "preview"))       # rank 0 dumped the clip


def test_unet_stream_with_a_plan_is_refused():
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel
    from opendwm_b200.sharding import ShardPlan
    T = 4
    unet = object.__new__(UNetCrossviewTemporalConditionModel)
    plan = ShardPlan(2, 0, T, cfg=True, make_groups=False)
    pipe = _stream_pipe(plan, T, model=unet)
    with pytest.raises(NotImplementedError, match="DiT"):
        pipe.reset_streaming((1, T, V, 4, 2, 3), "pt")
    # a plan attached after the reset is refused at the first denoising call
    pipe.sharding = None
    pipe.reset_streaming((1, T, V, 4, 2, 3), "pt")
    pipe.sharding = plan
    _, frames = _frames(T, T)
    with pytest.raises(NotImplementedError, match="DiT"):
        for f in frames:
            pipe.send_frame_condition(f)
