"""The streaming FIFO under a ShardPlan on one GPU.

1. The ring update of the step-invariant condition cache on a frame shard (any t_offset, the
   shard's own frame count, the window's T as T_total) equals a fresh build of that shard's cache
   bit for bit, over successive one-frame moves of the window, with and without the CFG split.
2. End to end at a tiny size: world-2 and world-4 process groups (gloo, the NCCL-free K,V
   all-gather) share the GPU and stream gathering, streaming and flush frames.  The FIFO latents
   after every call equal a single-process unsharded stream bit for bit on every rank; decoded
   frames agree within the run-to-run spread of two unsharded decodes (VAE GroupNorm statistics
   are summed with atomics)."""
import functools
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from common import CONDITION_COMMON, TINY, condition_batch, seeded_oracle, synthetic_inputs

pytestmark = pytest.mark.gpu
V = 3


@functools.lru_cache(maxsize=None)
def _state_dict():
    return seeded_oracle(TINY).state_dict()


def _model():
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    m = DiTCrossviewTemporalConditionModel(**TINY, compute_dtype=torch.float16)
    m.load_state_dict(_state_dict())
    return m.cuda()


def _assert_same(a, b, path="cd"):
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.shape == b.shape and torch.equal(a, b), path
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for k, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, "{}[{}]".format(path, k))
    elif isinstance(a, dict):
        assert a.keys() == b.keys(), (path, sorted(a.keys() ^ b.keys()))
        for k in a:
            _assert_same(a[k], b[k], "{}[{}]".format(path, k))
    else:
        assert a == b, path


@pytest.mark.parametrize("cfg", [False, True], ids=["frames_only", "cfg_split"])
@pytest.mark.parametrize("T", [16, 5])
@pytest.mark.parametrize("t_ways", [2, 4])
def test_sharded_ring_cache_equals_fresh_build(t_ways, T, cfg):
    from opendwm_b200.sharding import FRAME_KEYS, ShardPlan
    H, W = 8, 12
    _, _, stream = synthetic_inputs(TINY, B=2, T=T + 3, V=V, H=H, W=W, device="cuda")
    windows = [{k: v[:, s:s + T].contiguous() if k in FRAME_KEYS else v
                for k, v in stream.items()} for s in range(4)]
    ring, fresh = _model(), _model()
    ring._pack()
    fresh._pack()
    shifted = []
    inner = ring._conditions_shifted
    ring._conditions_shifted = lambda *a: shifted.append(a[1]) or inner(*a)
    world = t_ways * (2 if cfg else 1)
    for rank in range(world):
        plan = ShardPlan(world, rank, T, cfg=cfg, make_groups=False)
        shifted.clear()
        for s, window in enumerate(windows):
            c = plan.local_conditions(window, cfg_doubled=True)
            args = (c["encoder_hidden_states"].shape[0], plan.T_loc, V, H // 2, W // 2,
                    plan.t_offset, T, c["encoder_hidden_states"], c["pooled_projections"],
                    c["condition_image_tensor"], c["added_time_ids"], c["disable_crossview"],
                    c["disable_temporal"], c["crossview_attention_mask"])
            if s > 0:
                ring._ring_shift = True
            got = ring._conditions(*args)
            assert "_ring_shift" not in ring.__dict__
            fresh._cond_key = None
            _assert_same(got, fresh._conditions(*args))
        # shards of one frame are rebuilt whole (nothing to shift); every other shard shifts
        assert shifted == ([plan.T_loc] * 3 if plan.T_loc > 1 else []), (rank, shifted)


# -- end to end: processes sharing the GPU ---------------------------------------------------

VAE = dict(in_channels=3, out_channels=3, block_out_channels=(32, 64, 128, 128),
           layers_per_block=2, latent_channels=16, norm_num_groups=8, scaling_factor=1.5305,
           shift_factor=0.0609, use_quant_conv=False, use_post_quant_conv=False)


def _pipe(T):
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    torch.manual_seed(0)
    vae = AutoencoderKL(**VAE, compute_dtype=torch.float16).cuda()
    common = dict(CONDITION_COMMON, added_time_ids="fps_camera_transforms_action",
                  camera_ego_sensor_indices=[1, 2, 3], vae_instance=vae)
    inf = {"guidance_scale": 2.0, "inference_steps": 3 * T, "sequence_length_per_iteration": T,
           "autoregression_data_exception_for_take_sequence": ["crossview_mask"],
           "autoregression_condition_exception_for_take_sequence": [
               "disable_crossview", "disable_temporal", "crossview_attention_mask",
               "camera_intrinsics_norm", "camera2referego"]}
    return StreamingCrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {}, inf,
                                        None, _model(), model_dtype=torch.float16)


def _stream(pipe, T, n):
    """n frames of conditions, then the flush: (FIFO after every call, emitted frames)."""
    from dwm.functional import take_sequence_clip
    batch = condition_batch(T=n, V=V, hw=(64, 96), text_dim=TINY["joint_attention_dim"],
                            pooled_dim=TINY["pooled_projection_dim"])
    frames = [{k: v if k == "crossview_mask" else take_sequence_clip(v, i, i + 1)
               for k, v in batch.items()} for i in range(n)]
    pipe.reset_streaming((1, T, V, 16, 8, 12), "pt")
    fifo, out = [], []
    for f in frames + [None]:
        pipe.send_frame_condition(f)
        fifo.append(None if pipe.latents is None else pipe.latents.cpu())
        while True:
            img = pipe.receive_frame()
            if img is None:
                break
            out.append(img.float().cpu())
    return fifo, out


def _worker(rank, world, port, T, n, want_fifo, want_frames, tol):
    from opendwm_b200 import lib
    from opendwm_b200.sharding import ShardPlan
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DWM_PEER_SCATTER="0")
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lib.set_option("attn_tc", 0)
        pipe = _pipe(T)
        pipe.sharding = ShardPlan(world, rank, T, cfg=True)
        fifo, frames = _stream(pipe, T, n)
        assert len(fifo) == len(want_fifo)
        for k, (g, w) in enumerate(zip(fifo, want_fifo)):
            assert (g is None) == (w is None), (rank, k)
            assert g is None or torch.equal(g, w), \
                (rank, k, (g - w).abs().max().item())
        assert len(frames) == len(want_frames) == n
        for k, (g, w) in enumerate(zip(frames, want_frames)):
            err = (g - w).abs().max().item()
            assert err <= tol, (rank, k, err, tol)
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,T", [(2, 4), (4, 5)], ids=["cfg2xframes1", "cfg2xframes2_3+2"])
def test_sharded_stream_on_one_gpu(world, T):
    from opendwm_b200 import lib
    n = T + 3
    lib.set_option("attn_tc", 0)      # the sharded temporal attention is the mma.sync kernel
    try:
        want_fifo, want = _stream(_pipe(T), T, n)
        _, again = _stream(_pipe(T), T, n)
    finally:
        lib.set_option("attn_tc", -1)
    assert sum(f is not None for f in want_fifo) == n - T + 1 + 1
    # run-to-run spread of the unsharded decode (floored at one fp16 ulp at 1.0, the VAE's
    # output dtype).  The sharded decode is a third sample of the same variation and two
    # samples only estimate its range, so the sharded frames get twice the measured spread
    spread = max((a - b).abs().max().item() for a, b in zip(want, again))
    tol = 2 * max(spread, 2.0 ** -10)
    port = 29000 + (os.getpid() % 500)
    mp.spawn(_worker, args=(world, port, T, n, want_fifo, want, tol), nprocs=world, join=True)
