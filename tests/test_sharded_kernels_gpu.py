"""Kernel paths of frame-sharded temporal attention and of separate-K,V attention, checked on
one GPU against fp32 PyTorch on the same 16-bit inputs.

Every rank of a frame group is emulated in one process: the "peer" buffers are other buffers
on the same device, so the fused K,V projection scatter (`peer_out` of dwm_b200_linear) and
the attention of local queries against all frames (`kv` of dwm_b200_attention) run exactly
as in a multi-GPU step.  Where the sharded step claims the bits of the unsharded one, the
comparison is torch.equal."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# (T, t_ways): even shards, and the uneven 2,1,1,1 / 3,3,3,2 / 5,5,5,4 splits
SHARDS = [(16, 2), (16, 8), (5, 4), (11, 4), (19, 4)]
SHARD_IDS = ["16over2", "16over8", "5over4", "11over4", "19over4"]
DTYPES = [torch.bfloat16, torch.float16]


def _ids(v):
    """Test ids: dtypes by their short names, everything else as pytest names it."""
    return {torch.bfloat16: "bf16", torch.float16: "fp16"}.get(v) if isinstance(v, torch.dtype) \
        else None


def _split(T, t_ways):
    """(counts, offsets) of the frame shards, as ShardPlan computes them."""
    from opendwm_b200.sharding import ShardPlan
    plans = [ShardPlan(t_ways, r, T, cfg=False, make_groups=False) for r in range(t_ways)]
    return [p.T_loc for p in plans], [p.t_offset for p in plans]


def _mk(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _relerr(y, ref):
    return ((y.float() - ref).abs().max() / ref.abs().max().clamp_min(1e-20)).item()


def _frames(t, B, T, off, cnt):
    """Rows of frames [off, off + cnt) of a [B * T * R, C] buffer, as [B * cnt * R, C]."""
    C = t.shape[1]
    return t.view(B, T, -1, C)[:, off:off + cnt].reshape(-1, C)


def _frame_mask(B, T, R, off, cnt):
    m = torch.zeros(B, T, R, dtype=torch.bool, device="cuda")
    m[:, off:off + cnt] = True
    return m.view(-1)


# ---- 1a. K,V projection scattered into every peer's gathered buffer -------------------------

@pytest.fixture(params=[(0, 128), (0, 256), (1, 128), (1, 256)],
                ids=["1cta-bn128", "1cta-bn256", "2cta-bn128", "2cta-bn256"])
def gemm_variant(request):
    """The 1-CTA and the 2-CTA (M >= 512) GEMM, each at both tile widths (GEGLU always uses
    256); defaults restored afterwards."""
    from opendwm_b200 import lib
    two, bn = request.param
    lib.set_option("gemm_2cta", two)
    lib.set_option("gemm_bn", bn)
    yield request.param
    lib.set_option("gemm_2cta", 1)
    lib.set_option("gemm_bn", 0)


def _rms(t, w, eps):
    return t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + eps) * w


@pytest.mark.parametrize("D", [128, 1536])
@pytest.mark.parametrize("T,t_ways", SHARDS, ids=SHARD_IDS)
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("dtype", DTYPES, ids=_ids)
def test_kv_projection_peer_scatter(dtype, B, T, t_ways, D, gemm_variant):
    """Every emulated rank projects its local frames (rows_per_item = T_loc * R, items = batch
    entries) into its own gathered buffer and, through `peer_out`, into every other rank's, in
    the unsharded (b, t, r) row layout: the arguments of `_temporal_qkv_attend_sharded.project`
    (QKNORM with one normalised region and no k weight; STORE when qk_norm is off) and GEGLU,
    which the ABI allows as well.  Buffers start as NaN so stray or missing stores show."""
    from opendwm_b200 import ops, lib
    counts, offsets = _split(T, t_ways)
    R, K = 32, D + 64                     # rows per frame (V * S), input width
    a_full = _mk((B * T * R, K), dtype, seed=1)
    w = _mk((2 * D, K), dtype, 0.05, seed=2)
    b = _mk((2 * D,), torch.float32, 0.5, seed=3)
    nk = _mk((64,), torch.float32, seed=4) * 0.2 + 1
    tol = 6e-3 if dtype == torch.bfloat16 else 1e-3
    eps = 1e-5

    z = a_full.float() @ w.float().t() + b
    k32 = _rms(z[:, :D].reshape(-1, D // 64, 64), nk, eps).reshape(-1, D)
    wg, bg = ops.pack_geglu(w, b)
    h, gate = z.chunk(2, dim=-1)
    cases = {
        "qknorm": (dict(epilogue=lib.EPI_QKNORM, qk_region=D, qk_norm_regions=1,
                        q_norm_weight=nk, k_norm_weight=None, eps=eps), w, b,
                   torch.cat([k32, z[:, D:]], 1), 2 * D),
        "store": (dict(), w, b, z, 2 * D),
        "geglu": (dict(epilogue=lib.EPI_GEGLU), wg, bg, h * torch.nn.functional.gelu(gate), D),
    }
    for name, (kw, wt, bias, ref32, width) in cases.items():
        unsharded = ops.linear(a_full, wt, bias, **kw)
        assert _relerr(unsharded, ref32) < tol, name
        bufs = [torch.full((B * T * R, width), float("nan"), dtype=dtype, device="cuda")
                for _ in range(t_ways)]
        for r in range(t_ways):
            a_loc = _frames(a_full, B, T, offsets[r], counts[r]).contiguous()
            peers = [bufs[q].data_ptr() for q in range(t_ways) if q != r]
            ops.linear(a_loc, wt, bias, out=bufs[r], peer_out=peers,
                       rows_per_item=counts[r] * R, out_item_stride=T * R,
                       out_row_offset=offsets[r] * R, **kw)
            if r == 0:
                mine = _frame_mask(B, T, R, offsets[0], counts[0])
                for q in range(t_ways):
                    assert torch.equal(bufs[q][mine], bufs[0][mine]), (name, q)
                    assert torch.isnan(bufs[q][~mine]).all(), (name, q)
                assert not torch.isnan(bufs[0][mine]).any(), name
        for q in range(t_ways):
            assert torch.equal(bufs[q], unsharded), (name, q)


def test_peer_scatter_errors():
    from opendwm_b200 import ops, lib
    a = _mk((128, 64), torch.bfloat16)
    w = _mk((256, 64), torch.bfloat16, 0.05)
    out = torch.empty(128, 256, dtype=torch.bfloat16, device="cuda")
    bufs = [torch.empty_like(out) for _ in range(9)]
    with pytest.raises(ValueError, match="at most 8 peer"):
        ops.linear(a, w, out=out, peer_out=[t.data_ptr() for t in bufs])
    for epi in (lib.EPI_RESID, lib.EPI_F32):
        with pytest.raises(RuntimeError, match="peer_out needs a 16-bit epilogue"):
            ops.linear(a, w, epilogue=epi, peer_out=[bufs[0].data_ptr()])


# ---- 1b. local queries against the gathered K,V of all frames --------------------------------

def _ref_attention(q, k, v, heads):
    """q [G, sq, D], k / v [G, sk, D] fp32 -> softmax(q k^T / 8) v, [G, sq, D]."""
    G, sq, D = q.shape
    sk = k.shape[1]
    qh = q.view(G, sq, heads, 64).transpose(1, 2)
    kh = k.view(G, sk, heads, 64).transpose(1, 2)
    vh = v.view(G, sk, heads, 64).transpose(1, 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * 0.125, -1)
    return (p @ vh).transpose(1, 2).reshape(G, sq, D)


def _temporal_geometry(kind):
    """(H, W) of the latent patch grid per temporal attention type: row-wise and full at
    W = 28 (row-wise T x W up to 19 x 28 = 532 keys, full T x S up to 532 as well)."""
    return {"pointwise": (2, 6), "rowwise": (2, 28), "full": (1, 28)}[kind]


def _temporal_index(kind, B, T, V, H, W):
    """Rows of the (b, t, v, s) layout in the groups / sequence order of each type."""
    S = H * W
    if kind == "pointwise":      # (b v hw) t
        b, r, t = torch.meshgrid(torch.arange(B), torch.arange(V * S), torch.arange(T),
                                 indexing="ij")
        idx = (b * T * V * S + t * V * S + r).reshape(B * V * S, T)
    elif kind == "rowwise":      # (b v h) (t w)
        b, v, h, t, w = torch.meshgrid(torch.arange(B), torch.arange(V), torch.arange(H),
                                       torch.arange(T), torch.arange(W), indexing="ij")
        idx = (((b * T + t) * V + v) * S + h * W + w).reshape(B * V * H, T * W)
    else:                        # (b v) (t hw)
        b, v, t, s = torch.meshgrid(torch.arange(B), torch.arange(V), torch.arange(T),
                                    torch.arange(S), indexing="ij")
        idx = (((b * T + t) * V + v) * S + s).reshape(B * V, T * S)
    return idx.cuda()


def _attend_unsharded(ops, kind, qkv, out, B, T, V, H, W, D, heads):
    """The arguments of DiTCrossviewTemporalConditionModel._temporal_attend."""
    S = H * W
    if kind == "full":
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V],
                      group_strides=[T * V * S, S], seq=T * S, inner=S,
                      stride_outer=V * S, stride_inner=1)
    elif kind == "rowwise":
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V, H],
                      group_strides=[T * V * S, S, W], seq=T * W,
                      inner=W, stride_outer=V * S, stride_inner=1)
    else:
        ops.attention(qkv, out, D=D, heads=heads,
                      group_dims=[B, V * S], group_strides=[T * V * S, 1],
                      seq=T, inner=1, stride_outer=V * S, stride_inner=0)


def _attend_sharded(ops, kind, q_loc, kv_all, out, B, T_loc, T, V, H, W, D, heads):
    """The arguments of DiTCrossviewTemporalConditionModel._temporal_qkv_attend_sharded.attend."""
    S, Hp, Wp = H * W, H, W
    if kind == "full":
        ops.attention(
            q_loc, out, D=D, heads=heads, group_dims=[B, V],
            group_strides=[T_loc * V * S, S], seq=T_loc * S, inner=S,
            stride_outer=V * S, stride_inner=1, kv=kv_all, k_col=0, v_col=D,
            kv_group_strides=[T * V * S, S], seq_kv=T * S, inner_kv=S,
            kv_stride_outer=V * S, kv_stride_inner=1)
    elif kind == "rowwise":
        ops.attention(
            q_loc, out, D=D, heads=heads, group_dims=[B, V, Hp],
            group_strides=[T_loc * V * S, S, Wp], seq=T_loc * Wp, inner=Wp,
            stride_outer=V * S, stride_inner=1, kv=kv_all, k_col=0, v_col=D,
            kv_group_strides=[T * V * S, S, Wp], seq_kv=T * Wp, inner_kv=Wp,
            kv_stride_outer=V * S, kv_stride_inner=1)
    else:
        ops.attention(
            q_loc, out, D=D, heads=heads, group_dims=[B, V * S],
            group_strides=[T_loc * V * S, 1], seq=T_loc, inner=1,
            stride_outer=V * S, stride_inner=0, kv=kv_all, k_col=0, v_col=D,
            kv_group_strides=[T * V * S, 1], seq_kv=T, inner_kv=1,
            kv_stride_outer=V * S, kv_stride_inner=0)


TEMPORAL_CASES = [(kind, T, t_ways, heads, dtype)
                  for kind in ("pointwise", "rowwise", "full")
                  for T, t_ways in SHARDS
                  for heads in (1, 2, 3)
                  for dtype in DTYPES]
TEMPORAL_CASES += [("rowwise", 19, 4, 24, torch.bfloat16), ("full", 11, 4, 24, torch.float16),
                   ("pointwise", 16, 8, 24, torch.bfloat16)]


@pytest.mark.parametrize("kind,T,t_ways,heads,dtype", TEMPORAL_CASES, ids=_ids)
def test_frame_sharded_temporal_attention(kind, T, t_ways, heads, dtype):
    """Each emulated rank attends its local query frames (a contiguous [rows_loc, D] buffer)
    to the K,V of all frames (`kv`, unsharded row layout).  B = 2, so the query and key group
    strides differ.  With attn_tc = 0 both runs use the same mma.sync tile configuration
    (chosen from max(seq, seq_kv)), so the stitched output equals the unsharded call bit for
    bit; both, and the unsharded default kernel, are within tolerance of fp32."""
    from opendwm_b200 import ops, lib
    B, V = 2, 2
    H, W = _temporal_geometry(kind)
    S, D = H * W, heads * 64
    counts, offsets = _split(T, t_ways)
    rows = B * T * V * S
    qkv = _mk((rows, 3 * D), dtype, seed=T * 10 + heads)
    kv_all = qkv[:, D:].contiguous()
    tol = 1.2e-2 if dtype == torch.bfloat16 else 2e-3

    idx = _temporal_index(kind, B, T, V, H, W)
    x = qkv.float()[idx.reshape(-1)].view(*idx.shape, 3 * D)
    ref = _ref_attention(x[..., :D], x[..., D:2 * D], x[..., 2 * D:], heads)

    def gathered(out):
        return out.float()[idx.reshape(-1)].view(*idx.shape, D)

    try:
        lib.set_option("attn_tc", 0)
        unsharded = torch.zeros(rows, D, dtype=dtype, device="cuda")
        _attend_unsharded(ops, kind, qkv, unsharded, B, T, V, H, W, D, heads)
        stitched = torch.full((rows, D), float("nan"), dtype=dtype, device="cuda")
        for r in range(t_ways):
            q_loc = _frames(qkv, B, T, offsets[r], counts[r])[:, :D].contiguous()
            out = torch.empty(q_loc.shape[0], D, dtype=dtype, device="cuda")
            _attend_sharded(ops, kind, q_loc, kv_all, out, B, counts[r], T, V, H, W, D, heads)
            stitched.view(B, T, V * S, D)[:, offsets[r]:offsets[r] + counts[r]] = \
                out.view(B, counts[r], V * S, D)
        lib.set_option("attn_tc", -1)
        default = torch.zeros(rows, D, dtype=dtype, device="cuda")
        _attend_unsharded(ops, kind, qkv, default, B, T, V, H, W, D, heads)
    finally:
        lib.set_option("attn_tc", -1)
    assert torch.equal(stitched, unsharded)
    for got in (unsharded, default):
        err = _relerr(gathered(got), ref)
        assert err < tol, err


# ---- 1c. UNet cross-attention: strided queries, separate text K,V ---------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=_ids)
@pytest.mark.parametrize("heads", [5, 10, 20])
@pytest.mark.parametrize("seq", [5, 12, 30, 40, 112, 1792])
@pytest.mark.parametrize("Lc", [1, 7, 16, 17, 32, 33, 64, 65, 77, 154])
def test_separate_kv_cross_attention(Lc, seq, heads, dtype):
    """Queries are the q columns of the fused self-attention buffer (row pitch 3 x inner),
    keys / values a [N * Lc, 2 x inner] text projection, as in the UNet's spatial transformer.
    Lengths sit on both sides of the kernel's tile switches at max(seq, seq_kv) = 16 / 32 and of
    the 64-query tiles; short queries meet long keys and the reverse."""
    from opendwm_b200 import ops
    N = 2
    inner = heads * 64
    qkv_s = _mk((N * seq, 3 * inner), dtype, seed=seq)
    q = qkv_s[:, :inner]
    kv = _mk((N * Lc, 2 * inner), dtype, seed=1000 + Lc)
    out = torch.full((N * seq, inner), float("nan"), dtype=dtype, device="cuda")
    ops.attention(q, out, D=inner, heads=heads, group_dims=[N], group_strides=[seq], seq=seq,
                  kv=kv, k_col=0, v_col=inner, kv_group_strides=[Lc], seq_kv=Lc)
    kf = kv.float().view(N, Lc, 2 * inner)
    ref = _ref_attention(q.float().reshape(N, seq, inner), kf[..., :inner], kf[..., inner:],
                         heads)
    err = _relerr(out.view(N, seq, inner), ref)
    assert err < (1.2e-2 if dtype == torch.bfloat16 else 2e-3), err
