"""Exchange helpers of the frame-sharded CTSD-2.1 UNet over gloo (CPU processes).

A temporal ResBlock couples frames twice: GroupNorm statistics span the window's T frames, and
the (3,1,1) convolution reads each frame's two neighbours (zero padding at the window's ends).
Worlds of 2, 4 and 8 ranks with even and uneven frame shards check that
`ShardPlan.reduce_group_sums`, `reduce_amax` and `exchange_halo` give the unsharded statistics,
amax and neighbour frames, and that a torch restatement of one temporal ResBlock
(GroupNorm -> SiLU -> conv3d (3,1,1), twice) run per shard with them equals the unsharded one."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

G = 4


def _inputs(T, nb=2, S=3, C=8):
    g = torch.Generator().manual_seed(T)
    x = torch.randn(nb, T, S, C, generator=g, dtype=torch.float64)
    w = [torch.randn(3, C, C, generator=g, dtype=torch.float64) / C for _ in range(2)]
    return x, w


def _sums(x):
    """[nb, T, S, C] -> [nb, G, 2] (sum, sum of squares) over (C/G, T, S)."""
    nb, C = x.shape[0], x.shape[-1]
    xg = x.reshape(nb, -1, G, C // G).transpose(1, 2).reshape(nb, G, -1)
    return torch.stack([xg.sum(-1), (xg * xg).sum(-1)], -1)


def _norm_silu(x, sums, frames, eps=1e-5):
    nb, T, S, C = x.shape
    cnt = frames * S * C // G
    mean = sums[..., 0] / cnt
    rstd = (sums[..., 1] / cnt - mean * mean + eps).rsqrt()
    mean = mean.repeat_interleave(C // G, 1).view(nb, 1, 1, C)
    rstd = rstd.repeat_interleave(C // G, 1).view(nb, 1, 1, C)
    return torch.nn.functional.silu((x - mean) * rstd)


def _conv_t(buf, w):
    """conv3d (3,1,1) over a zero- or halo-padded operand [nb, T + 2, S, C]."""
    T = buf.shape[1] - 2
    return sum(buf[:, k:k + T] @ w[k] for k in range(3))


def _padded(y):
    buf = y.new_zeros(y.shape[0], y.shape[1] + 2, *y.shape[2:])
    buf[:, 1:-1] = y
    return buf


def _temporal_res(x, w, plan=None):
    """GroupNorm -> SiLU -> conv (3,1,1), twice; plan: x is the plan's frame shard."""
    T = x.shape[1] if plan is None else plan.T
    h = x
    for wk in w:
        sums = _sums(h)
        if plan is not None:
            plan.reduce_group_sums(sums)
        buf = _padded(_norm_silu(h, sums, T))
        if plan is not None:
            plan.exchange_halo(buf)
        h = _conv_t(buf, wk)
    return h + x


def _worker(rank, world, port, T, cfg):
    from opendwm_b200.sharding import ShardPlan
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        plan = ShardPlan(world, rank, T, cfg=cfg)
        fs = plan.frame_slice()
        x, w = _inputs(T)
        # a different window per CFG branch: the exchanges stay inside the frame group
        x = x + plan.cfg_rank
        xl = x[:, fs].contiguous()
        # statistics
        sums = plan.reduce_group_sums(_sums(xl))
        torch.testing.assert_close(sums, _sums(x), rtol=1e-12, atol=1e-12)
        # amax: exact
        amax = xl.abs().amax(dim=(1, 2, 3)).float()
        assert torch.equal(plan.reduce_amax(amax), x.abs().amax(dim=(1, 2, 3)).float())
        # halo frames, 16-bit and one-byte (E4M3 operand) buffers
        for dt in (torch.float16, torch.float8_e4m3fn):
            full = _padded(x.to(dt).float()).to(dt)
            buf = _padded(xl.to(dt).float()).to(dt)
            plan.exchange_halo(buf)
            want = full[:, plan.t_offset:plan.t_offset + plan.T_loc + 2]
            assert torch.equal(buf.view(torch.uint8), want.contiguous().view(torch.uint8)), \
                (rank, dt)
        # one temporal ResBlock
        got = _temporal_res(xl, w, plan)
        torch.testing.assert_close(got, _temporal_res(x, w)[:, fs], rtol=1e-10, atol=1e-10)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,T,cfg", [
    (2, 8, False), (2, 5, False), (4, 5, False), (4, 8, False), (4, 11, True), (8, 11, False),
    (8, 8, True)],
    ids=["w2_8", "w2_5_3+2", "w4_5_2+1+1+1", "w4_8", "cfg2xframes2_11", "w8_11", "cfg2xframes4_8"])
def test_unet_exchange_helpers(world, T, cfg):
    port = 29600 + (os.getpid() + world * 7 + T) % 300
    mp.spawn(_worker, args=(world, port, T, cfg), nprocs=world, join=True)
