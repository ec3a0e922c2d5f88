"""The view-sharded DiT forward at its real call site, every rank emulated in one process:
sharded == unsharded bit for bit, for view shards alone (views 2, views 3, views 2,2,1,1) and
for views x frames, with both K,V exchanges (fused peer scatter and all-gather), in 16 bit and
with the FP8 linears.

Rank r runs its own model instance (same state dict) with `model.shard = ShardPlan(world, r,
T, cfg=False, make_groups=False, views=V, view_ways=k)` on its frames and views.  The
exchanges are replaced by same-device buffers, one per (group, block): the all-gathers by stubs
that write the rank's rows into a shared full buffer and copy it out, the symmetric-memory
`PeerKV` by a fake that hands out the other group members' buffers as peer pointers.  Ranks run
one after another, so a block reads the K,V rows of later ranks from the previous round: rounds
repeat until the stitched tokens stop changing.

6 views of a 4 x 12 patch grid: the cross-view sequence (6 x 12 = 72 keys) runs on the wgmma
kernel, unsharded and (separate K,V with the view offset into the mask) sharded."""
import functools

import pytest
import torch

from common import TINY, seeded_oracle, synthetic_inputs

pytestmark = pytest.mark.gpu
NAN = float("nan")
V, H, W = 6, 8, 24


@functools.lru_cache(maxsize=None)
def _state_dict():
    return seeded_oracle(dict(TINY)).state_dict()


class _Done:
    def wait(self):
        return True


class _Handle:
    def barrier(self, channel=0):
        return None


def _group_key(plan, axis):
    """(axis, the coordinates the group members share) and this rank's index in the group."""
    if axis == "t":
        return (axis, plan.cfg_rank, plan.v_rank), plan.t_rank
    return (axis, plan.cfg_rank, plan.t_rank), plan.v_rank


def _blocks(axis):
    return len(TINY["temporal_block_layers"] if axis == "t" else TINY["crossview_block_layers"])


class _AllGatherStub:
    """`plan.gather_frames_kv` / `plan.gather_views_kv` of every emulated rank: one shared full
    K,V buffer per (group, block); a call writes the rank's rows into it, copies it out."""

    def __init__(self):
        self.shared, self.calls, self.same = {}, {}, []

    def bind(self, plan):
        def gather(axis, kv_local, kv_full, items):
            gk, _ = _group_key(plan, axis)
            ck = (gk, plan.rank)
            k = self.calls.get(ck, 0)
            self.calls[ck] = k + 1
            key = (gk, k % _blocks(axis))
            if key not in self.shared:
                self.shared[key] = torch.full_like(kv_full, NAN)
            full = self.shared[key]
            C = kv_local.shape[1]
            n, off, cnt = (plan.T, plan.t_offset, plan.T_loc) if axis == "t" else \
                (plan.V, plan.v_offset, plan.V_loc)
            dst = full.view(items, n, -1, C)[:, off:off + cnt]
            src = kv_local.view(items, cnt, -1, C)
            self.same.append(torch.equal(dst, src))     # the previous round's rows
            dst.copy_(src)
            kv_full.copy_(full)
            return _Done()
        plan.gather_frames_kv = lambda kl, kf, batch=1, async_op=False: gather("t", kl, kf, batch)
        plan.gather_views_kv = lambda kl, kf, items, async_op=False: gather("v", kl, kf, items)

    def begin_round(self):
        self.same = []

    def check_final_round(self):
        assert self.same and all(self.same), self.same


class _PeerExchange:
    """Stand-in for the symmetric-memory buffers: one gathered buffer per (group member, block),
    never alternated (sequential emulation would let a later block overwrite rows an earlier
    block of another rank still has to read)."""

    def __init__(self):
        self.bufs, self.before = {}, {}
        ex = self

        class FakePeerKV:
            def __init__(self, plan, rows_full, width, dtype, device, axis="t"):
                self.plan, self.axis, self.k = plan, axis, 0
                self.gk, self.me = _group_key(plan, axis)
                self.ways = plan.t_ways if axis == "t" else plan.v_ways
                for r in range(self.ways):
                    for k in range(_blocks(axis)):
                        if (self.gk, r, k) not in ex.bufs:
                            ex.bufs[(self.gk, r, k)] = torch.full((rows_full, width), NAN,
                                                                  dtype=dtype, device=device)

            def next(self):
                k = self.k
                self.k = (k + 1) % _blocks(self.axis)
                peers = [ex.bufs[(self.gk, q, k)].data_ptr() for q in range(self.ways)
                         if q != self.me]
                return ex.bufs[(self.gk, self.me, k)], peers, _Handle()
        self.cls = FakePeerKV

    def begin_round(self):
        self.before = {key: buf.clone() for key, buf in self.bufs.items()}

    def check_final_round(self):
        assert self.bufs
        for (gk, r, k), buf in self.bufs.items():
            assert not torch.isnan(buf).any(), (gk, r, k)
            assert torch.equal(buf, self.bufs[(gk, 0, k)]), (gk, r, k)
            assert torch.equal(buf, self.before[(gk, r, k)]), (gk, r, k)


# (world, T, view_ways): views 2 (3,3), views 3 (2,2,2), views 4 (2,2,1,1), views2 x frames2
CASES = [(2, 4, 2), (3, 4, 3), (4, 4, 4), (4, 4, 2), (4, 5, 2)]
CASE_IDS = ["views2", "views3", "views2211", "views2xframes2", "views2xframes3+2"]


def _run_ranks(ranks, B, ref_shape, rounds, exchange):
    prev = None
    for _ in range(rounds):
        exchange.begin_round()
        full = torch.full((B, ranks[0][1].T, V) + ref_shape, NAN, device="cuda")
        for m, plan, s_loc, t_loc, c_loc in ranks:
            tok, _ = m.forward_tokens(s_loc, t_loc, **c_loc, t_offset=plan.t_offset,
                                      T_total=plan.T, v_offset=plan.v_offset, V_total=plan.V)
            full[:, plan.frame_slice(), plan.view_slice()] = \
                tok.view(B, plan.T_loc, plan.V_loc, *ref_shape)
        if prev is not None and torch.equal(full, prev):
            return full, True
        prev = full
    return prev, False


@pytest.mark.parametrize("use_peer_scatter", [False, True], ids=["allgather", "peer"])
@pytest.mark.parametrize("world,T,view_ways", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("dtype,fp8", [(torch.float16, False), (torch.bfloat16, False),
                                       (torch.bfloat16, True)], ids=["fp16", "bf16", "fp8"])
def test_view_sharded_forward_equals_unsharded(dtype, fp8, world, T, view_ways,
                                               use_peer_scatter, monkeypatch):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from opendwm_b200 import sharding
    from opendwm_b200.sharding import ShardPlan
    sd = _state_dict()

    def model():
        m = DiTCrossviewTemporalConditionModel(
            **TINY, compute_dtype=dtype, gemm_dtype=torch.float8_e4m3fn if fp8 else None)
        m.load_state_dict(sd)
        return m.cuda()

    sample, timestep, cond = synthetic_inputs(TINY, T=T, V=V, H=H, W=W, device="cuda")
    B = sample.shape[0]
    if use_peer_scatter:
        exchange = _PeerExchange()
        monkeypatch.setattr(sharding, "PeerKV", exchange.cls)
    else:
        exchange = _AllGatherStub()
    ranks = []
    for r in range(world):
        plan = ShardPlan(world, r, T, cfg=False, make_groups=False, views=V,
                         view_ways=view_ways)
        assert plan.v_ways == view_ways
        plan.use_peer_scatter = use_peer_scatter
        if not use_peer_scatter:
            exchange.bind(plan)
        m = model()
        m.shard = plan
        ranks.append((m, plan, plan.local_latents(sample),
                      timestep[:, plan.frame_slice(), plan.view_slice()].contiguous(),
                      plan.local_conditions(cond, cfg_doubled=False)))
    ref = model().forward_tokens(sample, timestep, **cond)[0].clone()
    rows = ref.shape[0] // (B * T * V)
    n_rounds = len(TINY["temporal_block_layers"]) + len(TINY["crossview_block_layers"]) + 2
    got, settled = _run_ranks(ranks, B, (rows, ref.shape[1]), n_rounds, exchange)
    torch.cuda.synchronize()
    assert settled, "stitched tokens still changing after {} rounds".format(n_rounds)
    exchange.check_final_round()
    got = got.reshape(ref.shape)
    assert torch.equal(got, ref), ((got - ref).abs().max() / ref.abs().max()).item()


def test_crossview_full_under_a_view_shard_is_refused():
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from opendwm_b200.sharding import ShardPlan
    cfg = dict(TINY, crossview_attention_type="full")
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.bfloat16)
    m.load_state_dict(seeded_oracle(cfg).state_dict())
    m = m.cuda()
    plan = ShardPlan(2, 0, 4, cfg=False, make_groups=False, views=V, view_ways=2)
    plan.use_peer_scatter = False
    m.shard = plan
    sample, timestep, cond = synthetic_inputs(cfg, T=4, V=V, H=H, W=W, device="cuda")
    cond["crossview_attention_mask"] = None
    with pytest.raises(NotImplementedError, match="only 'rowwise'"):
        m.forward_tokens(plan.local_latents(sample),
                         timestep[:, :, plan.view_slice()].contiguous(),
                         **plan.local_conditions(cond, cfg_doubled=False),
                         v_offset=plan.v_offset, V_total=V)
