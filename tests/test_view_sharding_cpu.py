"""CPU tests (plain arithmetic and gloo ranks) of the view axis of the shard plan: the
cfg x views x frames split rule, rank layout, groups, uneven view shards, condition and
latent slicing, and the cross-view K,V exchange of a view shard (local query views against
the gathered views, emulated with plain torch)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _run(fn, world, *args):
    port = 29000 + (os.getpid() % 500)
    mp.spawn(_entry, args=(fn, world, port, args), nprocs=world, join=True)


def _entry(rank, fn, world, port, args):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fn(rank, world, *args)
    finally:
        dist.destroy_process_group()


def _plans(world, T, V=None, **kw):
    from opendwm_b200.sharding import ShardPlan
    return [ShardPlan(world, r, T, make_groups=False, views=V, **kw) for r in range(world)]


def _ceil(a, b):
    return -(-a // b)


# ---- plan arithmetic ---------------------------------------------------------------------------

@pytest.mark.parametrize("world,T,V,want", [
    (8, 5, 6, "cfg2xviews2xframes2"),       # config 5 on 8 GPUs: largest shard 9 of 30 items
    (4, 1, 6, "cfg2xviews2xframes1"),       # config 2 (image window) on 4 GPUs
    (12, 1, 6, "cfg2xviews6xframes1"),
    (8, 16, 6, "cfg2xviews1xframes4"),      # the north star keeps its frame shards (tie)
])
def test_split_rule_results(world, T, V, want):
    assert _plans(world, T, V)[0].parallelism == want


@pytest.mark.parametrize("world", [1, 2, 4, 6, 8, 12, 16])
@pytest.mark.parametrize("T", [1, 2, 3, 5, 16, 19])
@pytest.mark.parametrize("V", [1, 3, 6])
def test_plan_grid(world, T, V):
    """Every rank of every feasible plan: the rank layout, counts / offsets of both axes, the
    three groups, and that the split minimises the largest shard (ties: more frame shards)."""
    from opendwm_b200.sharding import view_frame_ways
    cfg_ways = 2 if world >= 2 else 1
    rest = world // cfg_ways
    feasible = [(rest // v, v) for v in range(1, rest + 1)
                if rest % v == 0 and v <= V and rest // v <= T]
    if not feasible:
        with pytest.raises(ValueError):
            _plans(world, T, V)
        return
    best = min(_ceil(T, t) * _ceil(V, v) for t, v in feasible)
    t_best = max(t for t, v in feasible if _ceil(T, t) * _ceil(V, v) == best)
    plans = _plans(world, T, V)
    p0 = plans[0]
    assert (p0.t_ways, p0.v_ways) == (t_best, rest // t_best)
    assert view_frame_ways(rest, T, V) == (p0.t_ways, p0.v_ways)
    cells = set()
    for r, p in enumerate(plans):
        assert (p.cfg_ways, p.t_ways, p.v_ways) == (cfg_ways, p0.t_ways, p0.v_ways)
        assert r == (p.cfg_rank * p.v_ways + p.v_rank) * p.t_ways + p.t_rank == \
            p.rank_of(p.cfg_rank, p.v_rank, p.t_rank)
        cells.add((p.cfg_rank, p.v_rank, p.t_rank))
        for n, ways, counts, offsets, loc, off, idx in (
                (T, p.t_ways, p.counts, p.offsets, p.T_loc, p.t_offset, p.t_rank),
                (V, p.v_ways, p.v_counts, p.v_offsets, p.V_loc, p.v_offset, p.v_rank)):
            assert sum(counts) == n and len(counts) == ways
            assert max(counts) - min(counts) <= 1 and counts == sorted(counts, reverse=True)
            assert offsets == [sum(counts[:i]) for i in range(ways)]
            assert (loc, off) == (counts[idx], offsets[idx])
        assert p.view_slice() == slice(p.v_offset, p.v_offset + p.V_loc)
        assert p.frame_slice() == slice(p.t_offset, p.t_offset + p.T_loc)
        # each group: the ranks sharing the other two coordinates, this rank among them
        for axis, i, j, ways in (("t", p.cfg_rank, p.v_rank, p.t_ways),
                                 ("v", p.cfg_rank, p.t_rank, p.v_ways),
                                 ("cfg", p.v_rank, p.t_rank, p.cfg_ways)):
            members = p.group_ranks(axis, i, j)
            assert len(members) == ways and r in members
            for q in members:
                o = plans[q]
                same = {"t": (o.cfg_rank, o.v_rank) == (p.cfg_rank, p.v_rank),
                        "v": (o.cfg_rank, o.t_rank) == (p.cfg_rank, p.t_rank),
                        "cfg": (o.v_rank, o.t_rank) == (p.v_rank, p.t_rank)}[axis]
                assert same, (axis, r, q)
    assert len(cells) == world


@pytest.mark.parametrize("world,T", [(1, 16), (2, 4), (8, 16), (8, 5), (8, 19), (8, 11),
                                     (8, 6), (4, 5), (4, 11), (4, 19), (4, 4)])
@pytest.mark.parametrize("cfg", [True, False])
def test_views_none_is_the_frame_plan(world, T, cfg):
    """Without a view count the plan is the CFG x frames plan: rank layout, counts, names."""
    if (world // (2 if cfg and world >= 2 else 1)) > T:
        pytest.skip("infeasible frame split")
    from opendwm_b200.sharding import ShardPlan
    for r in range(world):
        p = ShardPlan(world, r, T, cfg=cfg, make_groups=False)
        cfg_ways = 2 if cfg and world >= 2 else 1
        t_ways = world // cfg_ways
        assert (p.cfg_ways, p.t_ways, p.v_ways) == (cfg_ways, t_ways, 1)
        assert (p.cfg_rank, p.t_rank, p.v_rank) == (r // t_ways, r % t_ways, 0)
        assert p.parallelism == "cfg{}xframes{}".format(cfg_ways, t_ways)
        assert (p.V_loc, p.v_offset, p.view_slice()) == (None, 0, slice(None))
        assert p.group_ranks("t", p.cfg_rank, 0) == [p.cfg_rank * t_ways + t
                                                     for t in range(t_ways)]
        assert p.group_ranks("cfg", 0, p.t_rank) == [c * t_ways + p.t_rank
                                                     for c in range(cfg_ways)]


def test_uneven_view_shards_and_forced_splits():
    plans = _plans(8, 1, 6, view_ways=4)
    assert plans[0].v_counts == [2, 2, 1, 1] and plans[0].v_offsets == [0, 2, 4, 5]
    assert [(p.v_offset, p.V_loc) for p in plans if p.cfg_rank == 0] == \
        [(0, 2), (2, 2), (4, 1), (5, 1)]
    p = _plans(8, 5, 6, view_ways=1)[0]
    assert p.parallelism == "cfg2xviews1xframes4" and p.counts == [2, 1, 1, 1]
    p = _plans(4, 16, 6, view_ways=2, cfg=False)[0]
    assert p.parallelism == "cfg1xviews2xframes2" and p.v_counts == [3, 3]


def test_view_plan_refusals():
    from opendwm_b200.sharding import ShardPlan
    with pytest.raises(ValueError, match="6 views cannot feed 12 view shards"):
        ShardPlan(24, 0, 1, make_groups=False, views=6, view_ways=12)
    with pytest.raises(ValueError, match="not divisible by 3 view shards"):
        ShardPlan(8, 0, 4, make_groups=False, views=6, view_ways=3)
    with pytest.raises(ValueError, match="cannot feed 8 shards"):
        ShardPlan(16, 0, 1, make_groups=False, views=6)          # 8 ranks per branch, 6 views
    with pytest.raises(ValueError, match="frames cannot feed"):
        ShardPlan(8, 0, 1, make_groups=False, views=6, view_ways=2)   # 2 frame shards of T = 1
    with pytest.raises(ValueError, match="view_ways needs"):
        ShardPlan(4, 0, 4, make_groups=False, view_ways=2)


def test_conditions_and_latents_are_sliced_on_both_axes():
    B, T, V = 1, 5, 6
    cond = {"encoder_hidden_states": torch.randn(2 * B, T, V, 3, 4),
            "condition_image_tensor": torch.randn(2 * B, 1, V, 2, 2, 2),   # first frame only
            "added_time_ids": torch.randn(2 * B, T, V, 7),
            "crossview_attention_mask": torch.ones(2 * B, V, V, dtype=torch.bool),
            "disable_temporal": torch.tensor([False, True])}
    lat = torch.randn(B, T, V, 4, 3, 5)
    for p in _plans(8, T, V):
        loc = p.local_conditions(cond, cfg_doubled=True)
        c, fs, vs = slice(p.cfg_rank, p.cfg_rank + 1), p.frame_slice(), p.view_slice()
        assert torch.equal(loc["encoder_hidden_states"], cond["encoder_hidden_states"][c, fs, vs])
        assert torch.equal(loc["added_time_ids"], cond["added_time_ids"][c, fs, vs])
        assert torch.equal(loc["condition_image_tensor"],
                           cond["condition_image_tensor"][c, :, vs])
        assert torch.equal(loc["crossview_attention_mask"], cond["crossview_attention_mask"][c])
        assert loc["disable_temporal"].tolist() == [bool(p.cfg_rank)]
        mine = p.local_latents(lat)
        assert mine.is_contiguous() and torch.equal(mine, lat[:, fs, vs])


# ---- gloo ranks ----------------------------------------------------------------------------------

def _view_exchange(rank, world, T, V, view_ways, cfg):
    """The cross-view K,V all-gather of a view shard into the unsharded (b, t, v, s) layout, the
    index arithmetic of local query views against it (query unit u reads mask row
    v_offset + u), the groups, and the latents round trip over both axes."""
    from opendwm_b200.sharding import ShardPlan
    B, Hp, Wp, C = 2, 2, 3, 8
    S = Hp * Wp
    plan = ShardPlan(world, rank, T, cfg=cfg, views=V, view_ways=view_ways)
    assert plan.v_ways == view_ways
    # group membership seen through collectives
    for group, axis, i, j in ((plan.t_group, "t", plan.cfg_rank, plan.v_rank),
                              (plan.v_group, "v", plan.cfg_rank, plan.t_rank),
                              (plan.cfg_group, "cfg", plan.v_rank, plan.t_rank)):
        members = plan.group_ranks(axis, i, j)
        if group is None:
            assert members == [rank]
            continue
        got = torch.zeros(len(members), dtype=torch.long)
        dist.all_gather_into_tensor(got, torch.tensor([rank]), group=group)
        assert got.tolist() == members, axis
    g = torch.Generator().manual_seed(0)
    q = torch.randn(B, T, V, S, C, generator=g)
    kv = torch.randn(B, T, V, S, 2 * C, generator=g)
    mask = torch.rand(B, V, V, generator=g) > 0.4
    mask |= torch.eye(V, dtype=torch.bool)
    fs, vs = plan.frame_slice(), plan.view_slice()
    T_loc = plan.T_loc
    kv_loc = kv[:, fs, vs].reshape(-1, 2 * C).contiguous()
    kv_all = torch.full((B * T_loc * V * S, 2 * C), float("nan"))
    plan.gather_views_kv(kv_loc, kv_all, items=B * T_loc, async_op=True).wait()
    assert torch.equal(kv_all, kv[:, fs].reshape(-1, 2 * C))

    def rows(t, n):                       # "(b t v) (h w) c -> (b t h) (v w) c"
        return t.reshape(B, T_loc, n, Hp, Wp, t.shape[-1]).permute(0, 1, 3, 2, 4, 5) \
            .reshape(B, T_loc, Hp, n * Wp, t.shape[-1])

    kf, vf = kv_all.view(B, T_loc, V, S, 2 * C).split(C, -1)
    # key column j belongs to view j // Wp; query row i of the shard to view v_offset + i // Wp
    qv = plan.v_offset + torch.arange(plan.V_loc * Wp) // Wp
    kvv = torch.arange(V * Wp) // Wp
    allow = mask[:, qv][:, :, kvv].view(B, 1, 1, plan.V_loc * Wp, V * Wp)
    s = rows(q[:, fs, vs], plan.V_loc) @ rows(kf, V).transpose(-1, -2) / C ** 0.5
    att = torch.softmax(s.masked_fill(~allow, float("-inf")), -1) @ rows(vf, V)
    full_allow = mask[:, kvv][:, :, kvv].view(B, 1, 1, V * Wp, V * Wp)
    s = rows(q[:, fs], V) @ rows(kv[:, fs, :, :, :C], V).transpose(-1, -2) / C ** 0.5
    ref = torch.softmax(s.masked_fill(~full_allow, float("-inf")), -1) @ rows(kv[:, fs, :, :, C:], V)
    ref = ref.view(B, T_loc, Hp, V, Wp, C)[:, :, :, vs].reshape(att.shape)
    torch.testing.assert_close(att, ref)
    lat = torch.arange(B * T * V * 2, dtype=torch.float32).view(B, T, V, 2)
    assert torch.equal(plan.gather_latents(plan.local_latents(lat)), lat)
    # temporal-conv halo frames come from the frame neighbours of the same branch and views
    buf = torch.full((B * plan.V_loc, T_loc + 2, 3), -1.0)
    buf[:, 1:T_loc + 1] = (torch.arange(T_loc) + plan.t_offset).view(1, -1, 1).float() \
        + 100 * (plan.v_offset + plan.cfg_rank * V)
    plan.exchange_halo(buf)
    own = 100 * (plan.v_offset + plan.cfg_rank * V)
    first = plan.t_offset - 1 + own if plan.t_rank > 0 else -1.0
    last = plan.t_offset + T_loc + own if plan.t_rank + 1 < plan.t_ways else -1.0
    assert (buf[:, 0] == first).all() and (buf[:, T_loc + 1] == last).all(), (rank, buf[0])


@pytest.mark.parametrize("world,T,V,view_ways,cfg", [
    (2, 1, 6, 2, False),           # views 3,3
    (4, 1, 6, 4, False),           # views 2,2,1,1
    (4, 1, 6, 2, True),            # config 2 on 4 ranks: cfg2 x views2
    (4, 5, 6, 2, False),           # views2 x frames 3,2
    (8, 5, 6, 2, True),            # config 5 on 8 ranks: cfg2 x views2 x frames2
])
def test_view_sharded_exchange_gloo(world, T, V, view_ways, cfg):
    _run(_view_exchange, world, T, V, view_ways, cfg)
