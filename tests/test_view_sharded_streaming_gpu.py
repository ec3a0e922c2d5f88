"""The streaming FIFO under a ShardPlan with a view axis, on one GPU.

1. The ring update of the step-invariant condition cache on a view (and frame) shard equals a
   fresh build of that shard's cache bit for bit over successive one-frame moves of the window.
2. End to end at a tiny size: gloo process groups (the NCCL-free K,V all-gathers over the view
   and frame groups) share the GPU and stream gathering, streaming and flush frames.  The FIFO
   latents after every call equal a single-process unsharded stream bit for bit on every rank;
   decoded frames (still item-parallel over all ranks) agree within the run-to-run spread of
   two unsharded decodes."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from common import TINY, synthetic_inputs
from test_streaming_sharded_gpu import V, _assert_same, _model, _pipe, _stream

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world,T,view_ways", [(4, 16, 2), (6, 5, 3), (8, 5, 2)],
                         ids=["cfg2xviews2", "cfg2xviews3", "cfg2xviews2xframes2"])
def test_view_sharded_ring_cache_equals_fresh_build(world, T, view_ways):
    from opendwm_b200.sharding import FRAME_KEYS, ShardPlan
    H, W = 8, 12
    _, _, stream = synthetic_inputs(TINY, B=2, T=T + 3, V=V, H=H, W=W, device="cuda")
    windows = [{k: v[:, s:s + T].contiguous() if k in FRAME_KEYS else v
                for k, v in stream.items()} for s in range(4)]
    ring, fresh = _model(), _model()
    ring._pack()
    fresh._pack()
    for rank in range(world):
        plan = ShardPlan(world, rank, T, make_groups=False, views=V, view_ways=view_ways)
        for s, window in enumerate(windows):
            c = plan.local_conditions(window, cfg_doubled=True)
            args = (c["encoder_hidden_states"].shape[0], plan.T_loc, plan.V_loc, H // 2, W // 2,
                    plan.t_offset, T, c["encoder_hidden_states"], c["pooled_projections"],
                    c["condition_image_tensor"], c["added_time_ids"], c["disable_crossview"],
                    c["disable_temporal"], c["crossview_attention_mask"], plan.v_offset, V)
            if s > 0:
                ring._ring_shift = True
            got = ring._conditions(*args)
            fresh._cond_key = None
            _assert_same(got, fresh._conditions(*args))


def _worker(rank, world, port, T, n, view_ways, cfg, want_fifo, want_frames, tol):
    from opendwm_b200 import lib
    from opendwm_b200.sharding import ShardPlan
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DWM_PEER_SCATTER="0")
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lib.set_option("attn_tc", 0)
        pipe = _pipe(T)
        pipe.sharding = ShardPlan(world, rank, T, cfg=cfg, views=V, view_ways=view_ways)
        assert pipe.sharding.v_ways == view_ways
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


@pytest.mark.parametrize("world,T,view_ways,cfg", [(4, 4, 2, True), (4, 5, 2, False)],
                         ids=["cfg2xviews2", "views2xframes2_3+2"])
def test_view_sharded_stream_on_one_gpu(world, T, view_ways, cfg):
    from opendwm_b200 import lib
    n = T + 3
    lib.set_option("attn_tc", 0)      # the frame-sharded temporal attention is the mma.sync kernel
    try:
        want_fifo, want = _stream(_pipe(T), T, n)
        _, again = _stream(_pipe(T), T, n)
    finally:
        lib.set_option("attn_tc", -1)
    spread = max((a - b).abs().max().item() for a, b in zip(want, again))
    tol = 2 * max(spread, 2.0 ** -10)
    port = 29000 + (os.getpid() % 500)
    mp.spawn(_worker, args=(world, port, T, n, view_ways, cfg, want_fifo, want, tol),
             nprocs=world, join=True)
