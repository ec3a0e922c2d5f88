"""The frame-sharded DiT forward at its real call site, every rank of a frame group emulated in
one process: sharded == unsharded bit for bit, for every temporal attention type and both K,V
exchanges (fused peer scatter and all-gather).

Rank r runs its own model instance (same state dict) with `model.shard = ShardPlan(t_ways, r,
T, cfg=False, make_groups=False)` on its frames.  The exchange is replaced by same-device
buffers: the all-gather by a stub that keeps one shared full K,V buffer per temporal block, the
symmetric-memory `PeerKV` by a fake that keeps one gathered buffer per (rank, temporal block)
and hands out the other ranks' buffers as peer pointers.  Ranks run one after another, so a
rank's temporal block reads the K,V rows of later ranks from the previous round: rounds over
all ranks repeat until the stitched tokens stop changing, which takes one round per temporal
block plus one."""
import functools

import pytest
import torch

from common import TINY, seeded_oracle, synthetic_inputs

pytestmark = pytest.mark.gpu
NAN = float("nan")


@functools.lru_cache(maxsize=None)
def _state_dict(kind):
    return seeded_oracle(dict(TINY, temporal_attention_type=kind)).state_dict()


class _Done:
    def wait(self):
        return True


class _Handle:
    def barrier(self, channel=0):
        return None


class _AllGatherStub:
    """`plan.gather_frames_kv` of every emulated rank: one shared full K,V buffer per temporal
    block; a call writes the rank's local rows into it and copies it into `kv_all`."""

    def __init__(self, n_blocks):
        self.n_blocks, self.shared, self.calls, self.same = n_blocks, {}, {}, []

    def bind(self, plan):
        def gather(kv_local, kv_full, batch=1, async_op=False):
            k = self.calls.get(plan.t_rank, 0)
            self.calls[plan.t_rank] = k + 1
            k %= self.n_blocks
            if k not in self.shared:
                self.shared[k] = torch.full_like(kv_full, NAN)
            full = self.shared[k]
            C = kv_local.shape[1]
            dst = full.view(batch, plan.T, -1, C)[:, plan.t_offset:plan.t_offset + plan.T_loc]
            src = kv_local.view(batch, plan.T_loc, -1, C)
            self.same.append(torch.equal(dst, src))     # the previous round's rows
            dst.copy_(src)
            kv_full.copy_(full)
            return _Done()
        plan.gather_frames_kv = gather

    def begin_round(self):
        self.same = []

    def check_final_round(self):
        assert self.same and all(self.same), self.same


class _PeerExchange:
    """Stand-in for the symmetric-memory buffers: one gathered buffer per (rank, temporal
    block), never alternated (sequential emulation would let a later block overwrite the rows
    an earlier block of another rank still has to read)."""

    def __init__(self, n_blocks):
        self.n_blocks, self.bufs, self.before = n_blocks, {}, {}
        ex = self

        class FakePeerKV:
            def __init__(self, plan, rows_full, width, dtype, device):
                self.plan, self.k = plan, 0
                for r in range(plan.t_ways):
                    for k in range(ex.n_blocks):
                        if (r, k) not in ex.bufs:
                            ex.bufs[(r, k)] = torch.full((rows_full, width), NAN, dtype=dtype,
                                                         device=device)

            def next(self):
                k, r = self.k, self.plan.t_rank
                self.k = (k + 1) % ex.n_blocks
                peers = [ex.bufs[(q, k)].data_ptr() for q in range(self.plan.t_ways) if q != r]
                return ex.bufs[(r, k)], peers, _Handle()
        self.cls = FakePeerKV

    def begin_round(self):
        self.before = {key: buf.clone() for key, buf in self.bufs.items()}

    def check_final_round(self):
        assert self.bufs
        for (r, k), buf in self.bufs.items():
            assert not torch.isnan(buf).any(), (r, k)
            assert torch.equal(buf, self.bufs[(0, k)]), (r, k)
            assert torch.equal(buf, self.before[(r, k)]), (r, k)


CASES = [
    ("pointwise", 4, 2, torch.float16, None),
    ("rowwise", 4, 2, torch.float16, None),
    ("full", 4, 2, torch.float16, None),
    ("pointwise", 5, 4, torch.float16, None),
    ("rowwise", 5, 4, torch.float16, None),
    ("full", 5, 4, torch.float16, None),
    ("full", 5, 4, torch.bfloat16, None),
    ("rowwise", 4, 2, torch.float16, [False, True]),
]


@pytest.mark.parametrize("use_peer_scatter", [False, True], ids=["allgather", "peer"])
@pytest.mark.parametrize("kind,T,t_ways,dtype,disable_temporal", CASES,
                         ids=lambda v: {torch.bfloat16: "bf16", torch.float16: "fp16"}.get(v)
                         if isinstance(v, torch.dtype) else None)
def test_sharded_forward_equals_unsharded(kind, T, t_ways, dtype, disable_temporal,
                                          use_peer_scatter, monkeypatch):
    """B = 2, V = 3, 4 x 6 patches: the unsharded GEMMs have M >= 512 (2-CTA kernel) and the
    sharded ones fewer rows, so the STORE / QKNORM / GEGLU / RESID epilogues also cross the
    M-dependent kernel choices.  attn_tc = 0 in both runs (the sharded attention is always the
    mma.sync kernel)."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from opendwm_b200 import lib, sharding
    from opendwm_b200.sharding import ShardPlan
    cfg = dict(TINY, temporal_attention_type=kind)
    sd = _state_dict(kind)
    n_blocks = len(cfg["temporal_block_layers"])

    def model():
        m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=dtype)
        m.load_state_dict(sd)
        return m.cuda()

    sample, timestep, cond = synthetic_inputs(cfg, T=T, device="cuda")
    if disable_temporal is not None:
        cond["disable_temporal"] = torch.tensor(disable_temporal, device="cuda")
    B = sample.shape[0]

    if use_peer_scatter:
        exchange = _PeerExchange(n_blocks)
        monkeypatch.setattr(sharding, "PeerKV", exchange.cls)
    else:
        exchange = _AllGatherStub(n_blocks)
    ranks = []
    for r in range(t_ways):
        plan = ShardPlan(t_ways, r, T, cfg=False, make_groups=False)
        plan.use_peer_scatter = use_peer_scatter
        if not use_peer_scatter:
            exchange.bind(plan)
        m = model()
        m.shard = plan
        fs = plan.frame_slice()
        ranks.append((m, plan, sample[:, fs].contiguous(), timestep[:, fs].contiguous(),
                      plan.local_conditions(cond, cfg_doubled=False)))
    try:
        lib.set_option("attn_tc", 0)
        ref = model().forward_tokens(sample, timestep, **cond)[0].clone()
        prev, settled = None, False
        for _ in range(n_blocks + 2):
            exchange.begin_round()
            parts = []
            for m, plan, s_loc, t_loc, c_loc in ranks:
                tok, _ = m.forward_tokens(s_loc, t_loc, **c_loc, t_offset=plan.t_offset,
                                          T_total=T)
                parts.append(tok.view(B, plan.T_loc, -1, tok.shape[1]).clone())
            stitched = torch.cat(parts, 1).reshape(ref.shape)
            if prev is not None and torch.equal(stitched, prev):
                settled = True
                break
            prev = stitched
        torch.cuda.synchronize()
    finally:
        lib.set_option("attn_tc", -1)
    assert settled, "stitched tokens still changing after {} rounds".format(n_blocks + 2)
    exchange.check_final_round()
    assert torch.equal(stitched, ref), \
        ((stitched - ref).abs().max() / ref.abs().max()).item()
