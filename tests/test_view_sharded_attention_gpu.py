"""Cross-view row-wise attention of a view shard on one GPU: local query views (with the view
offset into the [B, V, V] mask) against the K,V of all views in a separate buffer, on the wgmma
kernel and on the mma.sync kernel.  Every shard of a split is launched in turn; the rows it
writes must equal, bit for bit, the same rows of the unsharded launch of the same kernel, and
no row outside the shard may be written."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# view splits of V = 6: 2,2,1,1 / 3,3 / 6 x 1
SPLITS = {"2211": [2, 2, 1, 1], "33": [3, 3], "111111": [1] * 6}
DTYPES = [torch.bfloat16, torch.float16]


def _ids(v):
    return {torch.bfloat16: "bf16", torch.float16: "fp16"}.get(v) if isinstance(v, torch.dtype) \
        else None


def _masks(BT, V, ring):
    """[BT, V, V] uint8: a ring (each view sees itself and its two neighbours; the second batch
    entry also sees the opposite view), or all ones."""
    if not ring:
        return torch.ones(BT, V, V, dtype=torch.uint8, device="cuda")
    i = torch.arange(V)
    d = (i.view(-1, 1) - i.view(1, -1)) % V
    m = ((d == 0) | (d == 1) | (d == V - 1)).to(torch.uint8)
    ms = [m.clone() for _ in range(BT)]
    for b in range(1, BT, 2):
        ms[b][d == V // 2] = 1
    return torch.stack(ms).cuda()


def _unsharded(ops, qkv, out, BT, V, Hp, Wp, D, heads, mask):
    """The arguments of DiTCrossviewTemporalConditionModel._crossview_attend ("rowwise", T = 1)."""
    S = Hp * Wp
    ops.attention(qkv, out, D=D, heads=heads, group_dims=[BT, Hp], group_strides=[V * S, Wp],
                  seq=V * Wp, inner=Wp, stride_outer=S, stride_inner=1, mask=mask, mask_div=1)


def _shard(ops, q_loc, kv_all, out, BT, V, v_off, V_loc, Hp, Wp, D, heads, mask):
    """Local views [v_off, v_off + V_loc) against all V views; the output goes straight to the
    shard's rows of a full-size [BT * V * S, D] buffer."""
    S = Hp * Wp
    ops.attention(q_loc, out[v_off * S:], D=D, heads=heads, group_dims=[BT, Hp],
                  group_strides=[V_loc * S, Wp], seq=V_loc * Wp, inner=Wp, stride_outer=S,
                  stride_inner=1, out_group_strides=[V * S, Wp], out_stride_outer=S,
                  out_stride_inner=1, mask=mask, mask_div=1, mask_q_offset=v_off,
                  kv=kv_all, k_col=0, v_col=D, kv_group_strides=[V * S, Wp], seq_kv=V * Wp,
                  inner_kv=Wp, kv_stride_outer=S, kv_stride_inner=1)


def _reference(qkv, BT, V, Hp, Wp, D, heads, mask):
    """fp32 softmax attention of "(bt v) (h w) c -> (bt h) (v w) c", in the (bt, v, s) layout."""
    S = Hp * Wp
    x = qkv.float().view(BT, V, Hp, Wp, 3, heads, 64).permute(4, 0, 2, 5, 1, 3, 6)
    q, k, v = (t.reshape(BT, Hp, heads, V * Wp, 64) for t in x)
    s = q @ k.transpose(-1, -2) * 0.125
    allow = mask.bool().repeat_interleave(Wp, 1).repeat_interleave(Wp, 2)
    s = s.masked_fill(~allow.view(BT, 1, 1, V * Wp, V * Wp), float("-inf"))
    o = torch.softmax(s, -1) @ v
    return o.view(BT, Hp, heads, V, Wp, 64).permute(0, 3, 1, 4, 2, 5).reshape(BT * V * S, D)


@pytest.mark.parametrize("attn_tc", [1, 0], ids=["wgmma", "mmasync"])
@pytest.mark.parametrize("ring", [True, False], ids=["ring", "nomask"])
@pytest.mark.parametrize("Wp,heads", [(28, 2), (64, 1), (16, 3)])
@pytest.mark.parametrize("split", list(SPLITS), ids=list(SPLITS))
@pytest.mark.parametrize("dtype", DTYPES, ids=_ids)
def test_view_shard_rows_equal_unsharded_rows(dtype, split, Wp, heads, ring, attn_tc):
    """Wp = 28 (the DiT at 32 x 56 latents: 4 views per key block, the second block ragged),
    64 (2 views per block) and 16 (all six views in one block).  Without the ring mask the
    unsharded call has no mask and the shards an all-ones one: the view-shard call needs a mask
    to take the wgmma kernel, and the two calls compute the same thing."""
    from opendwm_b200 import lib, ops
    BT, V, Hp = 2, 6, 3
    S, D = Hp * Wp, heads * 64
    counts = SPLITS[split]
    offsets = [sum(counts[:i]) for i in range(len(counts))]
    g = torch.Generator(device="cpu").manual_seed(Wp * 10 + heads)
    qkv = torch.randn(BT * V * S, 3 * D, generator=g).to(dtype).cuda()
    kv_all = qkv[:, D:].contiguous()
    mask = _masks(BT, V, ring)
    try:
        lib.set_option("attn_tc", attn_tc)
        unsharded = torch.zeros(BT * V * S, D, dtype=dtype, device="cuda")
        _unsharded(ops, qkv, unsharded, BT, V, Hp, Wp, D, heads, mask if ring else None)
        stitched = torch.full((BT * V * S, D), float("nan"), dtype=dtype, device="cuda")
        for v_off, V_loc in zip(offsets, counts):
            q_loc = qkv.view(BT, V, S, 3 * D)[:, v_off:v_off + V_loc, :, :D] \
                .reshape(-1, D).contiguous()
            before = stitched.clone()
            _shard(ops, q_loc, kv_all, stitched, BT, V, v_off, V_loc, Hp, Wp, D, heads, mask)
            mine = torch.zeros(BT, V, S, dtype=torch.bool, device="cuda")
            mine[:, v_off:v_off + V_loc] = True
            mine = mine.view(-1)
            assert torch.equal(stitched[mine], unsharded[mine]), (v_off, V_loc)
            assert torch.equal(stitched[~mine].isnan(), before[~mine].isnan()), (v_off, V_loc)
        assert torch.equal(stitched, unsharded)
    finally:
        lib.set_option("attn_tc", -1)
    ref = _reference(qkv, BT, V, Hp, Wp, D, heads, mask)
    err = ((unsharded.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < (1.2e-2 if dtype == torch.bfloat16 else 2e-3), err


@pytest.mark.parametrize("dtype", DTYPES, ids=_ids)
def test_all_ones_mask_equals_no_mask(dtype):
    """The unsharded wgmma launch gives the same bits with an all-ones view mask as without a
    mask: the all-ones mask a view shard passes when the model has none changes nothing."""
    from opendwm_b200 import ops
    BT, V, Hp, Wp, heads = 4, 6, 16, 28, 2
    S, D = Hp * Wp, heads * 64
    qkv = (torch.randn(BT * V * S, 3 * D, generator=torch.Generator().manual_seed(3))
           .to(dtype).cuda())
    a = torch.empty(BT * V * S, D, dtype=dtype, device="cuda")
    b = torch.empty_like(a)
    _unsharded(ops, qkv, a, BT, V, Hp, Wp, D, heads, None)
    _unsharded(ops, qkv, b, BT, V, Hp, Wp, D, heads, _masks(BT, V, False))
    assert torch.equal(a, b)


def test_view_shard_rejects_offsets_outside_the_mask():
    from opendwm_b200 import ops
    BT, V, Hp, Wp, D = 1, 6, 2, 28, 64
    S = Hp * Wp
    q_loc = torch.zeros(BT * 2 * S, D, dtype=torch.bfloat16, device="cuda")
    kv_all = torch.zeros(BT * V * S, 2 * D, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(BT * V * S, D, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="outside the 6 mask rows"):
        _shard(ops, q_loc, kv_all, out, BT, V, 5, 2, Hp, Wp, D, 1, _masks(BT, V, True))
