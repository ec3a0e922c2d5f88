"""Parity of the gathered attention kernel against fp32 softmax(QK^T)V on the same
16-bit q|k|v, for every regrouping the CTSD DiT uses."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _qkv(rows, D, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, 3 * D, generator=g).to(dtype).cuda()


def _ref(qkv, rows_idx, D, heads, mask=None):
    """rows_idx: long [G, seq]; mask: bool [G, seq, seq] or None -> fp32 [G, seq, D]."""
    G, seq = rows_idx.shape
    x = qkv.float()[rows_idx.reshape(-1)].view(G, seq, 3, heads, 64)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))
    s = q @ k.transpose(-1, -2) * 0.125
    if mask is not None:
        s = s.masked_fill(~mask[:, None], float("-inf"))
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(G, seq, D)


def _tol(dtype):
    return 1.2e-2 if dtype == torch.bfloat16 else 2e-3


@pytest.fixture(params=[0, 2], ids=["mma", "tc2"])
def tc_variant(request):
    """Both attention kernels: 0 = attention.cu (mma.sync, gathered addressing), 2 =
    attention_wgmma.cu (warpgroup MMA, S / P / O in registers; contiguous and gathered-unit
    sequences)."""
    from opendwm_b200 import lib
    lib.set_option("attn_tc", request.param)
    yield request.param
    lib.set_option("attn_tc", -1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_joint_split(dtype, tc_variant):
    from opendwm_b200 import ops
    N, S, L, heads = 3, 448, 154, 3
    D = heads * 64
    qkv = _qkv(N * (S + L), D, dtype)
    out = torch.zeros(N * S, D, dtype=dtype, device="cuda")
    out2 = torch.zeros(N * L, D, dtype=dtype, device="cuda")
    ops.attention(qkv, out, D=D, heads=heads, group_dims=[N], group_strides=[S + L],
                  seq=S + L, out_group_strides=[S], out_stride_outer=0, out_stride_inner=1,
                  split=S, out2=out2)
    idx = torch.arange(N * (S + L), device="cuda").view(N, S + L)
    ref = _ref(qkv, idx, D, heads)
    err = (out.view(N, S, D).float() - ref[:, :S]).abs().max() / ref.abs().max()
    err2 = (out2.view(N, L, D).float() - ref[:, S:]).abs().max() / ref.abs().max()
    assert err < _tol(dtype) and err2 < _tol(dtype), (err, err2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("use_mask", [False, True])
@pytest.mark.parametrize("V,W", [(6, 28), (3, 12), (6, 56), (5, 128), (7, 20)])
def test_crossview_rowwise(use_mask, V, W, dtype, tc_variant):
    """(bt v) (h w) -> (bt h) (v w) with the [B,V,V] view mask.  V x W = 6 x 28 is the
    north-star regrouping (seq 168: tiles of 4 + 2 views); 6 x 56 has 2 views per tile, 5 x 128
    one view per tile, 7 x 20 a ragged last tile, 3 x 12 (seq 36) stays on the small kernel."""
    from opendwm_b200 import ops
    B, T, H, heads = 2, 2, 4, 2
    S, D = H * W, heads * 64
    qkv = _qkv(B * T * V * S, D, dtype)
    out = torch.zeros(B * T * V * S, D, dtype=dtype, device="cuda")
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    m = torch.stack([ring, torch.ones(V, V, dtype=torch.bool)]).cuda()  # batch 1 unmasked
    ops.attention(qkv, out, D=D, heads=heads, group_dims=[B * T, H], group_strides=[V * S, W],
                  seq=V * W, inner=W, stride_outer=S, stride_inner=1,
                  mask=m.to(torch.uint8).contiguous() if use_mask else None, mask_div=T)
    bt, h, v, w = torch.meshgrid(torch.arange(B * T), torch.arange(H), torch.arange(V),
                                 torch.arange(W), indexing="ij")
    idx = ((bt * V + v) * S + h * W + w).view(B * T * H, V * W).cuda()
    mask = None
    if use_mask:
        mask = m.repeat_interleave(W, 2).repeat_interleave(W, 1).repeat_interleave(T * H, 0)
    ref = _ref(qkv, idx, D, heads, mask)
    got = out.float()[idx.reshape(-1)].view(B * T * H, V * W, D)
    assert ((got - ref).abs().max() / ref.abs().max()).item() < _tol(dtype)


@pytest.mark.parametrize("T,kind,W", [(16, "pointwise", 6), (19, "pointwise", 6),
                                      (5, "pointwise", 6), (5, "rowwise", 6), (3, "full", 6),
                                      (19, "rowwise", 28), (16, "rowwise", 28), (6, "rowwise", 28)])
def test_temporal(T, kind, W, tc_variant):
    """Row-wise with W = 28 are the full-size sequences (T x W = 532 / 448 / 168: three group
    dims, tiles of 4 frames) that take the gathered wgmma path."""
    from opendwm_b200 import ops
    B, V, H, heads = 2, 2, 2, 2
    S, D, dtype = H * W, heads * 64, torch.bfloat16
    qkv = _qkv(B * T * V * S, D, dtype, seed=T)
    out = torch.zeros(B * T * V * S, D, dtype=dtype, device="cuda")
    if kind == "pointwise":   # (b v hw) t
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V * S],
                      group_strides=[T * V * S, 1], seq=T, inner=1, stride_outer=V * S,
                      stride_inner=0)
        b, r, t = torch.meshgrid(torch.arange(B), torch.arange(V * S), torch.arange(T), indexing="ij")
        idx = (b * T * V * S + t * V * S + r).view(B * V * S, T)
    elif kind == "rowwise":   # (b v h) (t w)
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V, H],
                      group_strides=[T * V * S, S, W], seq=T * W, inner=W, stride_outer=V * S,
                      stride_inner=1)
        b, v, h, t, w = torch.meshgrid(torch.arange(B), torch.arange(V), torch.arange(H),
                                       torch.arange(T), torch.arange(W), indexing="ij")
        idx = (((b * T + t) * V + v) * S + h * W + w).view(B * V * H, T * W)
    else:                     # (b v) (t hw)
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V],
                      group_strides=[T * V * S, S], seq=T * S, inner=S, stride_outer=V * S,
                      stride_inner=1)
        b, v, t, s = torch.meshgrid(torch.arange(B), torch.arange(V), torch.arange(T),
                                    torch.arange(S), indexing="ij")
        idx = (((b * T + t) * V + v) * S + s).view(B * V, T * S)
    idx = idx.cuda()
    ref = _ref(qkv, idx, D, heads)
    got = out.float()[idx.reshape(-1)].view(*idx.shape, D)
    assert ((got - ref).abs().max() / ref.abs().max()).item() < _tol(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("seq,N,heads", [(448, 5, 4), (129, 3, 2), (200, 7, 1), (640, 2, 3),
                                         (65, 4, 2), (602, 40, 24)])
def test_contiguous_sequences_tcgen05(seq, N, heads, dtype, tc_variant):
    """Contiguous unmasked groups take the wgmma kernel (attention_wgmma.cu)."""
    from opendwm_b200 import ops
    D = heads * 64
    qkv = _qkv(N * seq, D, dtype, seed=seq)
    out = torch.zeros(N * seq, D, dtype=dtype, device="cuda")
    ops.attention(qkv, out, D=D, heads=heads, group_dims=[N], group_strides=[seq], seq=seq)
    idx = torch.arange(N * seq, device="cuda").view(N, seq)
    ref = _ref(qkv, idx, D, heads)
    err = ((out.view(N, seq, D).float() - ref).abs().max() / ref.abs().max()).item()
    assert err < _tol(dtype), err


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_growing_logits_exercise_rescale(dtype, tc_variant):
    """Keys of later blocks carry much larger logits, so the running max grows by far more
    than 2^8 between key blocks and also by small steps: the online-softmax rescale of the
    running output must stay exact in both regimes."""
    from opendwm_b200 import ops
    N, seq, heads = 3, 602, 2
    D = heads * 64
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N * seq, 3 * D, generator=g)
    ramp = torch.linspace(0.2, 6.0, seq).repeat(N).unsqueeze(1)     # |k| grows along the sequence
    x[:, D:2 * D] *= ramp
    x[:, :D] *= 2.0
    qkv = x.to(dtype).cuda()
    out = torch.zeros(N * seq, D, dtype=dtype, device="cuda")
    ops.attention(qkv, out, D=D, heads=heads, group_dims=[N], group_strides=[seq], seq=seq)
    idx = torch.arange(N * seq, device="cuda").view(N, seq)
    ref = _ref(qkv, idx, D, heads)
    err = ((out.view(N, seq, D).float() - ref).abs().max() / ref.abs().max()).item()
    assert err < _tol(dtype), err
