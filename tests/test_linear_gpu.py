"""Parity of the wgmma GEMM + fused epilogues (dwm_b200_linear) against a plain
fp32 PyTorch evaluation of the same math on the same 16-bit inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["1cta", "2cta"])
def gemm_variant(request):
    """Every test runs on the 1-CTA kernel and on the kernel for clusters of two CTAs that
    share the weight tile by TMA multicast (the latter is used for M >= 512)."""
    from opendwm_b200 import lib
    lib.set_option("gemm_2cta", 1 if request.param == "2cta" else 0)
    yield
    lib.set_option("gemm_2cta", 1)


def _mk(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _relerr(y, ref):
    return ((y.float() - ref).abs().max() / ref.abs().max().clamp_min(1e-20)).item()


SHAPES = [
    (128, 256, 64), (128, 256, 128), (256, 512, 1536), (192, 1536, 256),
    (448 * 3, 4608, 1536), (77, 320, 320), (1000, 64, 1536), (130, 288, 72),
    (4096, 6144, 1536), (700, 512, 192), (513, 288, 64),
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_store(M, N, K, dtype):
    from opendwm_b200 import ops, lib
    a = _mk((M, K), dtype, seed=1)
    w = _mk((N, K), dtype, 0.05, seed=2)
    b = _mk((N,), torch.float32, seed=3)
    y = ops.linear(a, w, b)
    ref = a.float() @ w.float().t() + b
    # 16-bit output rounding: 2^-8 (bf16) / 2^-11 (fp16) relative per element
    tol = 6e-3 if dtype == torch.bfloat16 else 1e-3
    assert _relerr(y, ref) < tol
    y2 = ops.linear(a, w, b, epilogue=lib.EPI_F32)
    assert _relerr(y2, ref) < 2e-5
    torch.testing.assert_close(y2, ref, rtol=1e-3, atol=1e-3 * ref.abs().max().item())


@pytest.mark.parametrize("act", ["gelu_tanh", "gelu_erf", "silu", "relu"])
def test_activation(act):
    from opendwm_b200 import ops, lib
    code = {"gelu_tanh": lib.ACT_GELU_TANH, "gelu_erf": lib.ACT_GELU_ERF, "silu": lib.ACT_SILU,
            "relu": lib.ACT_RELU}[act]
    a = _mk((300, 512), torch.bfloat16, seed=1)
    w = _mk((1024, 512), torch.bfloat16, 0.05, seed=2)
    b = _mk((1024,), torch.float32, seed=3)
    z = a.float() @ w.float().t() + b
    ref = {"gelu_tanh": lambda t: torch.nn.functional.gelu(t, approximate="tanh"),
           "gelu_erf": torch.nn.functional.gelu,
           "silu": torch.nn.functional.silu, "relu": torch.relu}[act](z)
    y = ops.linear(a, w, b, epilogue=lib.EPI_F32, act=code)
    assert _relerr(y, ref) < 1e-5
    y16 = ops.linear(a, w, b, act=code)
    assert _relerr(y16, ref) < 6e-3


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_geglu(dtype):
    from opendwm_b200 import ops, lib
    D, M = 512, 700
    a = _mk((M, D), dtype, seed=1)
    w = _mk((8 * D, D), dtype, 0.05, seed=2)
    b = _mk((8 * D,), torch.float32, 0.5, seed=3)
    wp, bp = ops.pack_geglu(w, b)
    y = ops.linear(a, wp, bp, epilogue=lib.EPI_GEGLU)
    z = a.float() @ w.float().t() + b
    h, gate = z.chunk(2, dim=-1)
    ref = h * torch.nn.functional.gelu(gate)
    assert y.shape == (M, 4 * D)
    assert _relerr(y, ref) < (6e-3 if dtype == torch.bfloat16 else 1e-3)


@pytest.mark.parametrize("with_bias", [False, True])
def test_qknorm_with_row_remap(with_bias):
    from opendwm_b200 import ops, lib
    D, items, S, L = 512, 3, 100, 30
    dtype = torch.bfloat16
    a = _mk((items * S, D), dtype, seed=1)
    w = _mk((3 * D, D), dtype, 0.05, seed=2)
    b = _mk((3 * D,), torch.float32, 0.5, seed=3) if with_bias else None
    qw = _mk((64,), torch.float32, seed=4) * 0.2 + 1
    kw = _mk((64,), torch.float32, seed=5) * 0.2 + 1
    out = torch.zeros((items * (S + L), 3 * D), dtype=dtype, device="cuda")
    ops.linear(a, w, b, epilogue=lib.EPI_QKNORM, out=out, rows_per_item=S,
               out_item_stride=S + L, out_row_offset=0, q_norm_weight=qw,
               k_norm_weight=kw, qk_region=D, eps=1e-6)
    z = a.float() @ w.float().t()
    if b is not None:
        z = z + b
    q, k, v = z.view(items, S, 3, D // 64, 64).unbind(2)

    def rms(t, wt):
        return t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * wt
    ref = torch.stack([rms(q, qw), rms(k, kw), v], 2).reshape(items, S, 3 * D)
    got = out.view(items, S + L, 3 * D)
    assert _relerr(got[:, :S], ref) < 6e-3
    assert got[:, S:].abs().max().item() == 0  # context rows untouched


def test_resid_gate_blend():
    from opendwm_b200 import ops, lib
    D, K, B, items_per_b, S = 512, 1024, 2, 3, 50
    M = B * items_per_b * S
    a = _mk((M, K), torch.bfloat16, seed=1)
    w = _mk((D, K), torch.bfloat16, 0.05, seed=2)
    b = _mk((D,), torch.float32, seed=3)
    resid = _mk((M, D), torch.float32, seed=4)
    gate = _mk((B * items_per_b, 6 * D), torch.float32, seed=5)
    z = a.float() @ w.float().t() + b
    # gated residual (JointTransformerBlock): x + gate[item] * (acc + bias)
    g = gate[:, 2 * D:3 * D]
    ref = resid + g.repeat_interleave(S, 0) * z
    y = ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=resid, gate=g, rows_per_item=S)
    assert _relerr(y, ref) < 1e-5
    # in place
    r2 = resid.clone()
    ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=r2, out=r2, gate=g, rows_per_item=S)
    assert _relerr(r2, ref) < 1e-5
    # residual + AlphaBlender: alpha*x + (1-alpha)*(y + acc + bias)
    x = _mk((M, D), torch.float32, seed=6)
    alpha = torch.tensor([0.88, 1.0], device="cuda")
    ref2 = alpha.repeat_interleave(items_per_b * S)[:, None] * x + \
        (1 - alpha.repeat_interleave(items_per_b * S)[:, None]) * (resid + z)
    y2 = ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=resid, blend_x=x, alpha=alpha,
                    rows_per_batch=items_per_b * S)
    assert _relerr(y2, ref2) < 1e-5
    # positional table broadcast: resid row = m % S
    pos = _mk((S, D), torch.float32, seed=7)
    y3 = ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=pos, resid_row_mod=S)
    assert _relerr(y3, z + pos.repeat(B * items_per_b, 1)) < 1e-5


def test_errors_are_loud():
    from opendwm_b200 import ops
    a = _mk((128, 60), torch.bfloat16)
    w = _mk((256, 60), torch.bfloat16)
    with pytest.raises(RuntimeError, match="multiples of 8"):
        ops.linear(a, w)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(a.cpu(), w.cpu())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", [
    (512, 256, 64),            # one tile per cluster
    (3 * 448 + 77, 1536, 256),  # M tail (not a multiple of 32), 6 N-tiles
    (700, 320, 192),           # N % 256 != 0: dead chunks keep the stream in step
    (148 * 256 + 999, 512, 128),   # more tile pairs than clusters: several tiles per persistent CTA
    (5376, 1536, 1536),        # north-star out-proj shape (one frame group)
])
@pytest.mark.parametrize("bn", [256, 128])
def test_resid_tma_epilogue_equals_register_epilogue(M, N, K, dtype, bn, gemm_variant):
    """RESID epilogue against fp32 PyTorch (plain residual, in place, separate output, gate,
    bias, AlphaBlender) with the residual / blend rows prefetched into L2 by the TMA unit while
    the tile's MMAs run (`resid_tma` = 1) on the `bn`-column tile, and bit for bit against the
    OTHER tile width run without the prefetch: a second kernel instantiation whose epilogue
    drains differently split chunks must produce the same bits (same K order, explicit
    roundings in resid_elem / blend_elem)."""
    from opendwm_b200 import ops, lib
    S = 50
    items = (M + S - 1) // S
    B = 2
    rpb = (M + B - 1) // B
    a = _mk((M, K), dtype, seed=1)
    w = _mk((N, K), dtype, 0.05, seed=2)
    b = _mk((N,), torch.float32, seed=3)
    resid = _mk((M, N), torch.float32, seed=4)
    gate = _mk((items, 2 * N), torch.float32, seed=5)[:, N:]
    x = _mk((M, N), torch.float32, seed=6)
    alpha = torch.tensor([0.3, 1.0], device="cuda")
    z = a.float() @ w.float().t() + b
    rows = torch.arange(M, device="cuda")
    ref_gate = resid + gate[rows // S] * z
    al = alpha[rows // rpb][:, None]
    ref_blend = al * x + (1 - al) * (resid + z)

    def run(tma, tile_n):
        lib.set_option("resid_tma", tma)
        lib.set_option("gemm_bn", tile_n)      # 128: the narrow-tile variant (tail-wave repair)
        try:
            y1 = ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=resid, gate=gate,
                            rows_per_item=S)
            r2 = resid.clone()
            ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=r2, out=r2, gate=gate,
                       rows_per_item=S)
            y3 = ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=resid, blend_x=x,
                            alpha=alpha, rows_per_batch=rpb)
            x4 = x.clone()          # VT-block form: out = blend operand, in place
            ops.linear(a, w, b, epilogue=lib.EPI_RESID, resid=resid, out=x4, blend_x=x4,
                       alpha=alpha, rows_per_batch=rpb)
            y5 = ops.linear(a, w, None, epilogue=lib.EPI_RESID, resid=resid)
            torch.cuda.synchronize()
            return y1, r2, y3, x4, y5
        finally:
            lib.set_option("resid_tma", 1)
            lib.set_option("gemm_bn", 0)
    new, old = run(1, bn), run(0, 384 - bn)
    for got, ref in zip(new, (ref_gate, ref_gate, ref_blend, ref_blend, resid + z - b)):
        assert _relerr(got, ref) < 2e-5
    for g, o in zip(new, old):      # explicit roundings (resid_elem / blend_elem): same bits
        assert torch.equal(g, o)
