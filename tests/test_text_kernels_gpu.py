"""Element-wise conformance of the text-encoder kernels against float64 on the same 16-bit
operands: causal (CLIP) and biased (T5) attention at tile edges, the RMSNorm operand
(T5LayerNorm), the QuickGELU and gated tanh-GELU GEMM epilogues, and the embedding gather
(bit-exact)."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_attention_conformance_gpu import bound_violations, unit_roundoff  # noqa: E402

pytestmark = pytest.mark.gpu

# half the spacing of fp16 subnormals: the absolute error of rounding a value below 2^-14 to fp16
FP16_SUB = 2.0 ** -25


def subnormal_slack(dtype):
    """Absolute error a 16-bit rounding can add beyond u|x|: fp16 subnormals (bf16 has fp32's
    exponent range, so none at these magnitudes)."""
    return FP16_SUB if dtype == torch.float16 else 0.0


SEQS = [1, 63, 64, 65, 77, 128, 129, 300]
HEADS = [12, 20, 64]
DTYPES = [torch.bfloat16, torch.float16]


def _reference(q, k, v, scale, causal, bias):
    """float64 (softmax(q k^T scale + bias) v, same softmax applied to |v|, sum of |v| over the
    attended keys); q, k, v [G, H, S, 64], bias [H, S, S]."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.transpose(-1, -2) * scale
    S = s.shape[-1]
    if bias is not None:
        s = s + bias.double()[None]
    if causal:
        keep = torch.ones(S, S, dtype=torch.bool, device=s.device).tril()
        s = s.masked_fill(~keep, float("-inf"))
    p = torch.softmax(s, -1)
    return p @ v, p @ v.abs(), torch.isfinite(s).double() @ v.abs()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("heads", HEADS)
@pytest.mark.parametrize("seq", SEQS)
@pytest.mark.parametrize("mode", ["causal", "bias"])
def test_text_attention_conforms(mode, seq, heads, dtype):
    from opendwm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seq * 131 + heads)
    G, D = 3, heads * 64
    qkv = (torch.randn(G * seq, 3 * D, device="cuda", generator=g) * 1.5).to(dtype)
    bias = None
    scale = 0.125
    if mode == "bias":
        bias = torch.randn(heads, seq, seq, device="cuda", generator=g) * 3.0
        scale = 1.0 if heads != 20 else 0.125   # T5 runs unscaled
    sentinel = torch.full((G * seq + 2, D + 16), -7.0, device="cuda", dtype=dtype)
    out = sentinel[1:-1, :D]
    kw = dict(D=D, heads=heads, group_dims=[G], group_strides=[seq], seq=seq, scale=scale)
    ops.attention(qkv, out, causal=mode == "causal", bias=bias, **kw)
    again = torch.empty_like(out)
    ops.attention(qkv, again, causal=mode == "causal", bias=bias, **kw)
    torch.cuda.synchronize()
    x = qkv.view(G, seq, 3, heads, 64).permute(2, 0, 3, 1, 4)
    ref, pv, vsum = _reference(x[0], x[1], x[2], scale, mode == "causal", bias)
    got = out.view(G, seq, heads, 64).permute(0, 2, 1, 3)
    # bound_violations' bound, plus the P values that fp16 rounds to subnormals: each such p_j
    # (unnormalised, the row max is 1 so l >= 1) moves by up to 2^-25 absolutely, which is not
    # relative to P|V| when the winning keys' |v| is small: up to 2^-25 sum_j |v_j| in all.  The
    # unscaled T5 logits here (std ~20) put most keys there.
    u = unit_roundoff(dtype)
    bad, worst = bound_violations(got, ref, pv + subnormal_slack(dtype) * vsum / (2 * u + 1e-6), u)
    assert not bad.any(), "{} of {} elements outside the bound, worst ratio {:.3g}".format(
        int(bad.sum()), bad.numel(), worst)
    assert torch.equal(out, again)
    # nothing outside the output rows / columns was written
    assert (sentinel[0] == -7).all() and (sentinel[-1] == -7).all() and (sentinel[:, D:] == -7).all()


def test_text_attention_refusals():
    from opendwm_b200 import ops
    qkv = torch.zeros(2 * 77, 3 * 128, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(2 * 77, 128, device="cuda", dtype=torch.bfloat16)
    bias = torch.zeros(2, 77, 77, device="cuda")
    kw = dict(D=128, heads=2, group_dims=[2], group_strides=[77], seq=77)
    with pytest.raises(RuntimeError, match="one of causal and bias"):
        ops.attention(qkv, out, causal=True, bias=bias, **kw)
    with pytest.raises(RuntimeError, match="contiguous sequences"):   # padded groups
        ops.attention(torch.zeros(2 * 80, 3 * 128, device="cuda", dtype=torch.bfloat16), out,
                      causal=True, **dict(kw, group_strides=[80]))
    with pytest.raises(RuntimeError, match="contiguous sequences"):   # gathered units
        ops.attention(qkv, out, causal=True, **dict(kw, inner=7, stride_outer=7))
    with pytest.raises(ValueError, match="bias must be"):
        ops.attention(qkv, out, bias=bias[:, :76], **kw)


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16, torch.float32],
                         ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("M,D", [(1, 128), (77, 768), (300, 4096), (5, 1284)])
def test_rmsnorm_conforms(M, D, out_dtype):
    from opendwm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(M + D)
    xbuf = torch.randn(M, D + 12, device="cuda", generator=g) * 3 + 0.5
    x = xbuf[:, :D]                                   # row pitch != D
    w = torch.randn(D, device="cuda", generator=g)
    out = torch.empty(M, D + 4, device="cuda", dtype=out_dtype)[:, :D]
    ops.rmsnorm(x, w, out, eps=1e-6)
    xd = x.double()
    ref = w.double() * (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6))
    u = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}[out_dtype]
    # fp32 statistics and products: a few ulps of fp32 relative to |w x / rms|
    tol = u * ref.abs() + 2.0 ** -20 * ref.abs() + (FP16_SUB if out_dtype == torch.float16 else 0)
    assert ((out.double() - ref).abs() <= tol).all()


def _gemm_case(M, N, K, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(dtype)
    b = torch.randn(N, device="cuda", generator=g) * 0.5
    acc = a.double() @ w.double().t() + b.double()
    mag = a.double().abs() @ w.double().abs().t() + b.double().abs()
    return a, w, b, acc, mag


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("M", [77, 300, 924])
def test_quick_gelu_epilogue_conforms(M, dtype):
    from opendwm_b200 import lib, ops
    a, w, b, acc, mag = _gemm_case(M, 384, 256, dtype, M)
    out = ops.linear(a, w, b, act=lib.ACT_QUICK_GELU)
    sig = torch.sigmoid(1.702 * acc)
    ref = acc * sig
    slope = (sig + 1.702 * acc.abs() * sig * (1 - sig)).abs()     # |d quick_gelu / dx|
    tol = unit_roundoff(dtype) * ref.abs() + 2.0 ** -18 * (slope * mag + ref.abs()) + \
        subnormal_slack(dtype)
    err = (out.double() - ref).abs()
    assert (err <= tol).all(), float((err / tol).max())


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("M", [77, 300, 924])
def test_gated_tanh_gelu_epilogue_conforms(M, dtype):
    from opendwm_b200 import lib, ops
    F = 384
    a, w, b, acc, mag = _gemm_case(M, 2 * F, 256, dtype, M + 1)
    # rows [0, F) gate (wi_0), [F, 2F) value (wi_1), as T5 stores them; packed value-first
    gate_w, val_w = w[:F], w[F:]
    wp, bp = ops.pack_geglu(torch.cat([val_w, gate_w]), torch.cat([b[F:], b[:F]]))
    out = ops.linear(a, wp, bp, epilogue=lib.EPI_GEGLU_TANH)
    assert out.shape == (M, F)
    g, v = acc[:, :F], acc[:, F:]
    k = math.sqrt(2 / math.pi)
    th = torch.tanh(k * (g + 0.044715 * g ** 3))
    gelu = 0.5 * g * (1 + th)
    dgelu = (0.5 * (1 + th) + 0.5 * g * (1 - th ** 2) * k * (1 + 3 * 0.044715 * g ** 2)).abs()
    ref = v * gelu
    tol = unit_roundoff(dtype) * ref.abs() + 2.0 ** -18 * (
        gelu.abs() * mag[:, F:] + v.abs() * dgelu * mag[:, :F] + ref.abs()) + subnormal_slack(dtype)
    err = (out.double() - ref).abs()
    assert (err <= tol).all(), float((err / tol).max())


def test_text_epilogue_refusals():
    from opendwm_b200 import lib, ops
    a = torch.zeros(64, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(256, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="QUICK_GELU needs the DWM_EPI_STORE"):
        ops.linear(a, w, act=lib.ACT_QUICK_GELU, epilogue=lib.EPI_F32)
    with pytest.raises(RuntimeError, match="GEGLU needs N"):
        ops.linear(a, w[:128], epilogue=lib.EPI_GEGLU_TANH)


@pytest.mark.parametrize("D,seq,pos", [(768, 77, True), (1280, 77, True), (4096, 77, False),
                                       (128, 5, True)])
def test_embed_gather_is_bit_exact(D, seq, pos):
    from opendwm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(D + seq)
    vocab, n = 1000, 7
    tok = torch.randn(vocab, D, device="cuda", generator=g)
    p = torch.randn(seq + 3, D, device="cuda", generator=g) if pos else None
    ids = torch.randint(0, vocab, (n * seq,), device="cuda", generator=g)
    out = torch.full((n * seq, D + 8), float("nan"), device="cuda")[:, :D]
    ops.embed(ids, tok, out, pos=p, seq=seq)
    want = torch.nn.functional.embedding(ids, tok)
    if pos:
        want = want + p[:seq].repeat(n, 1)
    assert torch.equal(out, want)
