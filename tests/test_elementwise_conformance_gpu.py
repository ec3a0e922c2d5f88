"""Element-wise conformance of the scheduler updates and pixel kernels of rowops.cu / vae.cu
against float64: cfg_ddim_step, euler_step_by_indices, cfg_euler_step, lincomb2, axpy,
softmax_rows, act_cast, sinusoid, patchify, upsample_nearest and the text encoders' embed.

Bounds.  The arithmetic kernels are restated as float64 expressions over `Fe` values, which carry
a first-order bound on the fp32 kernel's error: every fp32 operation rounds once (U32 = 2^-24 of
its result), a product, sum or quotient propagates its operands' bounds (|b| e_a + |a| e_b;
e_a + e_b; (e_a + |a / b| e_b) / |b|), sqrtf is correctly rounded, and a fused multiply-add is
bounded by the same terms as the product and the sum, so the bound holds whether or not nvcc
contracts a product into the following addition.  A result rounded to bf16 / fp16 adds u |ref|
(2^-8, 2^-11).  The transcendental kernels use their CUDA accuracy: silu / gelu as
`act_reference` of the GEMM suite states; exp2f (softmax) 2 ulps plus the rounding of its
argument, |arg| 4 U32 ln 2 (the subtraction, the product and the fp32 scale log2(e)); expf /
sinf / cosf (sinusoid) 2 ulps each, with the timestep times the frequency rounded in fp32
(absolute error |t f| (3 U32 a + 5 U32), a = ln(1e4) k / (half - shift)).  softmax: max is
exact; the sum of c exponentials in a 256-thread, 8-warp tree adds (ceil(c / 256) + 13) U32
relative error.  Results below 2^-120 (softmax rows whose scaled range underflows exp2f,
gelu_tanh where __fdividef flushes to 0) are held to that absolute floor.  patchify and upsample_nearest move values
and round once: bit-exact against torch.  embed gathers fp32 rows and adds the position row with
one fp32 addition: bit-exact against torch.nn.functional.embedding (+ pos).

Every deterministic kernel is called twice and must repeat its bits.  groupnorm_stats (atomics)
is not here: see test_norm_conformance_gpu.

Worst ratio |out - ref| / tol over this file's cases, measured on an H100 80GB HBM3 at a 700 W
power limit (bf16 / fp16 / fp32 rounding): cfg_ddim_step 0.991 / 0.992 / 0.496,
euler_step_by_indices 0.959 / 0.975 / 0.927, cfg_euler_step 0.988 (bf16) / 0.941 (fp32),
lincomb2 0.924, axpy 0.976, softmax_rows 0.993 / 0.999, act_cast 0.991 / 0.992, sinusoid
0.977 / 0.922.  The 16-bit maxima sit in the output rounding, which is exact; the fp32 ones in
the single roundings of the update.
"""
import math

import pytest
import torch

from opendwm_b200 import lib
from test_gemm_conformance_gpu import (GELU_ERF, GELU_TANH, NONE, SILU, U32, act_reference,
                                       bound_violations, unit_roundoff)

pytestmark = pytest.mark.gpu

SENT16 = -21555
POISON = (float("nan"), float("inf"), float("-inf"))


class Fe:
    """float64 value and a bound on the fp32 kernel's error in computing it."""

    def __init__(self, v, e=None):
        self.v = v.double() if torch.is_tensor(v) else torch.tensor(float(v), dtype=torch.float64)
        self.e = torch.zeros_like(self.v) if e is None else e

    @staticmethod
    def of(x):
        return x if isinstance(x, Fe) else Fe(x)

    def _r(self, v, e):
        return Fe(v, e + U32 * v.abs())

    def __add__(self, o):
        o = Fe.of(o)
        return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = Fe.of(o)
        return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return Fe.of(o) - self

    def __mul__(self, o):
        o = Fe.of(o)
        return self._r(self.v * o.v, o.v.abs() * self.e + self.v.abs() * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Fe.of(o)
        q = self.v / o.v
        return self._r(q, (self.e + q.abs() * o.e) / o.v.abs())

    def sqrt(self):
        r = self.v.sqrt()
        return self._r(r, self.e / (2 * r.clamp_min(1e-300)))


def f32(t):
    """Fe of an fp32 operand (exact)."""
    return Fe(t.double())


def tol_for(fe, dtype):
    u = unit_roundoff(dtype)
    sub = 2.0 ** -25 if dtype == torch.float16 else 0.0
    return (1 + u) * fe.e + u * fe.v.abs() + sub


def check(out, ref, tol, what):
    bad, worst = bound_violations(out.cpu(), ref.cpu(), tol.cpu())
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d outside the bound (worst %.3g); first at %s: got %r ref %r tol %r" % (
            what, bad.sum(), bad.numel(), worst, i, out.cpu()[i].item(), ref.cpu()[i].item(), tol.cpu()[i].item()))
    print("BOUND_RATIO elementwise %s %.4g" % (what, worst))
    return worst


def _poison(n):
    return torch.tensor(POISON).repeat(n // 3 + 1)[:n]


def in_poison(t, pad=64):
    n = t.numel()
    x = _poison(n + 2 * pad).to(t.dtype)
    x[pad:pad + n] = t.reshape(-1)
    return x.cuda()[pad:pad + n].view(t.shape)


def in_block(t, pad=64):
    """t.cuda() as a view inside a larger, poisoned allocation: a missing check reads in-bounds
    memory instead of faulting."""
    return in_poison(t, pad)


def _g(seed):
    return torch.Generator().manual_seed(seed)


# --------------------------------------------------------------------------------------------
# cfg_ddim_step
# --------------------------------------------------------------------------------------------
def ddim_reference(pred, pred_c, lat, ts, step_ratio, alphas, final_alpha, ptype, gs):
    """Fe of the kernel's fp32 formula (cfg_ddim_kernel), per element."""
    v = f32(pred)
    if pred_c is not None:
        v = v + Fe(gs) * (f32(pred_c) - v)
    inner = lat.numel() // ts.numel()
    t = ts.long().repeat_interleave(inner).view(lat.shape)
    tp = t - step_ratio
    a_t = Fe(alphas.double()[t])
    a_p = Fe(torch.where(tp >= 0, alphas.double()[tp.clamp_min(0)], torch.tensor(float(final_alpha)).double()))
    b_t = 1.0 - a_t
    x = f32(lat)
    if ptype == "epsilon":
        x0 = (x - b_t.sqrt() * v) / a_t.sqrt()
        eps = v
    elif ptype == "sample":
        x0 = v
        eps = (x - a_t.sqrt() * x0) / b_t.sqrt()
    else:
        x0 = a_t.sqrt() * x - b_t.sqrt() * v
        eps = a_t.sqrt() * v + b_t.sqrt() * x
    return a_p.sqrt() * x0 + (1.0 - a_p).sqrt() * eps


@pytest.mark.parametrize("rdt", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("cfg", [1, 2])
@pytest.mark.parametrize("ptype", ["epsilon", "sample", "v_prediction"])
def test_cfg_ddim_step_conforms(ptype, cfg, rdt):
    """Per-item timesteps [B, T, V] = [2, 3, 2] from 999 down to 1, step_ratio 20: items with
    t - 20 < 0 take final_alpha_cumprod."""
    from opendwm_b200 import ops
    g = _g(7)
    B, T, V, C, H, W = 2, 3, 2, 4, 5, 7
    shape = (B, T, V, C, H, W)
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2
    alphas = torch.cumprod(1 - betas, 0).float()
    ts = torch.tensor([999, 500, 19, 0, 20, 1, 700, 40, 5, 250, 998, 21], dtype=torch.int32).view(B, T, V)
    lat = torch.randn(shape, generator=g)
    pred = torch.randn((cfg * B,) + shape[1:], generator=g)
    pc = pred[B:] if cfg == 2 else None
    ref = ddim_reference(pred[:B], pc, lat, ts, 20, alphas, 0.9991, ptype, 2.5)

    def run():
        out = in_block(lat)
        ops.cfg_ddim_step(in_block(pred), out, in_block(ts), in_block(alphas), cfg=cfg,
                          guidance_scale=2.5, step_ratio=20, final_alpha_cumprod=0.9991,
                          prediction_type=ptype, round_dtype=rdt)
        torch.cuda.synchronize()
        return out.cpu()

    out = run()
    check(out, ref.v, tol_for(ref, rdt), "cfg_ddim_%s_cfg%d_%s" % (ptype, cfg, rdt))
    assert torch.equal(run(), out), "the repeated call gave other bits"


# --------------------------------------------------------------------------------------------
# Euler updates
# --------------------------------------------------------------------------------------------
SIGMAS = torch.linspace(1.0, 0.0, 13)


@pytest.mark.parametrize("rdt", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
def test_euler_step_by_indices_conforms(rdt):
    from opendwm_b200 import ops
    g = _g(3)
    sample = torch.randn(2, 5, 3, 7, 9, generator=g)
    mo = torch.randn(sample.shape, generator=g)
    idx = torch.tensor([[0, 3, 11, 5, 7], [1, 2, 10, 4, 6]], dtype=torch.int32)
    k = idx.long().repeat_interleave(3 * 7 * 9).view(sample.shape)
    s = SIGMAS
    ref = f32(sample) + (Fe(s.double()[k + 1]) - Fe(s.double()[k])) * f32(mo)

    def run():
        x = in_block(sample)
        ops.euler_step_by_indices(in_block(mo), x, in_block(idx), in_block(s), round_dtype=rdt)
        torch.cuda.synchronize()
        return x.cpu()

    out = run()
    check(out, ref.v, tol_for(ref, rdt), "euler_idx_%s" % rdt)
    assert torch.equal(run(), out), "the repeated call gave other bits"
    with pytest.raises(ValueError):
        ops.euler_step_by_indices(in_block(mo), in_block(sample), in_block(idx.view(-1)[:4]), in_block(s))


def cfg_euler_reference(tok, ld, cfg, gs, shape, P, idx, sig, in_range, lat):
    """float64 un-patchify of the token rows (row r, column ((py P + px) C + c)), CFG, Euler."""
    B, T, V, C, H, W = shape
    Hp, Wp = H // P, W // P
    t6 = tok[:, :P * P * C].reshape(cfg, B, T, V, Hp, Wp, P, P, C)
    pix = t6.permute(0, 1, 2, 3, 8, 4, 6, 5, 7).reshape((cfg,) + shape)
    v = f32(pix[0])
    if cfg == 2:
        v = v + Fe(gs) * (f32(pix[1]) - v)
    k = idx.long().view(B, T, V, 1, 1, 1).expand(shape)
    new = f32(lat) + (Fe(sig.double()[k + 1]) - Fe(sig.double()[k])) * v
    keep = torch.ones(T, dtype=torch.bool) if in_range is None else in_range.bool()
    return new, v, keep.view(1, T, 1, 1, 1, 1).expand(shape)


@pytest.mark.parametrize("rdt", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("cfg,P,with_range,with_npred", [(2, 2, True, True), (1, 1, False, False),
                                                          (2, 1, False, True), (1, 2, True, False)])
def test_cfg_euler_step_conforms(cfg, P, with_range, with_npred, rdt):
    """ld_tok > P P C with a NaN / Inf pitch, V = 3; in_range / noise_pred optional."""
    from opendwm_b200 import ops
    g = _g(cfg * 10 + P)
    B, T, V, C, H, W = 2, 3, 3, 4, 6, 8
    shape = (B, T, V, C, H, W)
    rows = cfg * B * T * V * (H // P) * (W // P)
    cols = P * P * C
    ld = cols + 12
    tok = _poison(rows * ld).view(rows, ld)
    tok[:, :cols] = torch.randn(rows, cols, generator=g)
    lat = torch.randn(shape, generator=g)
    idx = torch.randint(0, 12, (B, T, V), generator=g, dtype=torch.int32)
    rng = torch.tensor([1, 0, 1], dtype=torch.uint8) if with_range else None
    new, v, keep = cfg_euler_reference(tok, ld, cfg, 3.0, shape, P, idx, SIGMAS, rng, lat)
    tokd = tok.cuda()[:, :cols]

    def run():
        x = in_block(lat)
        npred = in_block(torch.full(shape, float("nan"))) if with_npred else None
        ops.cfg_euler_step(tokd, x, in_block(idx), in_block(SIGMAS), cfg=cfg, guidance_scale=3.0,
                           patch=P, in_range=None if rng is None else rng.cuda(), noise_pred=npred,
                           round_dtype=rdt)
        torch.cuda.synchronize()
        return x.cpu(), None if npred is None else npred.cpu()

    out, npred = run()
    ref = torch.where(keep, new.v, lat.double())
    tol = torch.where(keep, tol_for(new, rdt), torch.zeros_like(new.e))
    check(out, ref, tol, "cfg_euler_cfg%d_P%d_%s" % (cfg, P, rdt))
    if with_npred:
        check(npred, v.v, v.e, "cfg_euler_npred_cfg%d_P%d" % (cfg, P))
    o2, n2 = run()
    assert torch.equal(o2, out) and (npred is None or torch.equal(n2, npred)), "the repeated call gave other bits"


# --------------------------------------------------------------------------------------------
# lincomb2, axpy
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,items", [(1, 1), (3, 1), (6, 2), (1001, 7), (4099, 1)])
def test_lincomb2_and_axpy_conform(n, items):
    from opendwm_b200 import ops
    g = _g(n)
    x, y = torch.randn(n * items, generator=g), torch.randn(n * items, generator=g)
    s0, s1 = torch.randn(items, generator=g), torch.randn(items, generator=g)
    it = torch.arange(n * items) // n
    ref = Fe(s0.double()[it]) * f32(x) + Fe(s1.double()[it]) * f32(y)

    def run():
        out = in_block(torch.full((n * items,), float("nan")))
        ops.lincomb2(in_block(x), in_block(y), in_block(s0), in_block(s1), out)
        torch.cuda.synchronize()
        return out.cpu()

    out = run()
    check(out, ref.v, ref.e, "lincomb2_n%d_items%d" % (n, items))
    assert torch.equal(run(), out)
    ref = f32(y) + Fe(0.37) * f32(x)

    def run_axpy():
        yy = in_block(y)
        ops.axpy(in_block(x), yy, 0.37)
        torch.cuda.synchronize()
        return yy.cpu()

    out = run_axpy()
    check(out, ref.v, ref.e, "axpy_n%d" % (n * items))
    assert torch.equal(run_axpy(), out)
    with pytest.raises(ValueError):
        ops.lincomb2(in_block(x), in_block(y[:-1]), in_block(s0), in_block(s1), in_block(x))
    with pytest.raises(ValueError):
        ops.lincomb2(in_block(x), in_block(y), in_block(s0), in_block(s1), in_block(torch.zeros(n * items + 1)))


# --------------------------------------------------------------------------------------------
# softmax_rows
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("cols", [1, 255, 256, 257, 1792, 7168])
def test_softmax_rows_conforms(cols, dtype):
    """ld > cols with NaN / Inf in the pitch; a constant row; a row whose scaled range underflows
    exp2f for all but a few entries; rows of mixed scale.  1792 and 7168 are the key counts of
    the 2-D VAE mid-block at 256 x 448 and 512 x 896 pixels."""
    from opendwm_b200 import ops
    g = _g(cols)
    R = 6
    x = torch.randn(R, cols, generator=g) * torch.tensor([1.0, 30.0, 0.1, 1.0, 1.0, 300.0])[:, None]
    x[3] = 2.5
    x[4] = torch.randn(cols, generator=g) * 0.01 - 1e3
    x[4, ::97] = 0.0
    scale = 0.125
    ld = cols + 5
    xp = _poison(R * ld).view(R, ld)
    xp[:, :cols] = x
    xd = xp.cuda()[:, :cols]
    xs = x.double() * scale
    ref = torch.softmax(xs, -1)
    arg = (x.double() - x.double().amax(-1, keepdim=True)) * scale * math.log2(math.e)
    e_elem = arg.abs() * 4 * U32 * math.log(2) + 5 * U32
    e_sum = (math.ceil(cols / 256) + 13) * U32 + e_elem.amax(-1, keepdim=True)
    err = ref * (e_elem + e_sum + 2 * U32)
    u = unit_roundoff(dtype)
    tol = (1 + u) * err + u * ref + 2.0 ** -120 + (2.0 ** -25 if dtype == torch.float16 else 0.0)

    def run():
        buf = torch.full((R, cols + 9), SENT16, dtype=torch.int16, device="cuda")
        ops.softmax_rows(xd, scale, buf.view(dtype)[:, :cols])
        torch.cuda.synchronize()
        return buf

    buf = run()
    assert (buf[:, cols:] == SENT16).all(), "wrote into the output pitch"
    check(buf.view(dtype)[:, :cols].float(), ref, tol, "softmax_c%d_%s" % (cols, dtype))
    assert torch.equal(run(), buf)


# --------------------------------------------------------------------------------------------
# act_cast
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("act", [NONE, SILU, GELU_TANH, GELU_ERF], ids=["none", "silu", "gelu_tanh", "gelu_erf"])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 4099])
def test_act_cast_conforms(n, act, dtype):
    from opendwm_b200 import ops
    x = torch.randn(n, generator=_g(n)) * 4
    x[::5] *= 1e-3
    y, e = act_reference(x.double(), act)
    u = unit_roundoff(dtype)
    # 2^-120: gelu_tanh's __fdividef returns 0 once 1 + e^-u2 exceeds 2^126 (|ref| < 2^-119)
    tol = (1 + u) * e + u * y.abs() + 2.0 ** -120 + (2.0 ** -25 if dtype == torch.float16 else 0.0)

    def run():
        buf = torch.full((n + 8,), SENT16, dtype=torch.int16, device="cuda")
        ops.act_cast(in_block(x), buf[:n].view(dtype), act)
        torch.cuda.synchronize()
        return buf

    buf = run()
    assert (buf[n:] == SENT16).all(), "wrote past n"
    check(buf[:n].view(dtype).float(), y, tol, "act_cast_n%d_act%d_%s" % (n, act, dtype))
    assert torch.equal(run(), buf)


def test_act_cast_rejects_relu():
    """act_cast does not implement ReLU; it used to return the input unchanged."""
    from opendwm_b200 import ops
    with pytest.raises(RuntimeError, match="not implemented"):
        ops.act_cast(torch.zeros(8, device="cuda"), torch.empty(8, device="cuda", dtype=torch.bfloat16),
                     lib.ACT_RELU)


# --------------------------------------------------------------------------------------------
# sinusoid
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("flip,shift", [(True, 0.0), (False, 1.0), (True, 1.0), (False, 0.0)])
def test_sinusoid_conforms(flip, shift, dtype):
    from opendwm_b200 import ops
    t = torch.tensor([0.0, 1.0, 999.0, -1000.0, 0.5, 250.25, 1000.0])
    ch = 320
    half = ch // 2
    k = torch.arange(half, dtype=torch.float64)
    a = math.log(10000.0) * k / (half - shift)
    freq = torch.exp(-a)
    arg = t.double()[:, None] * freq
    s, c = torch.sin(arg), torch.cos(arg)
    ref = torch.cat([c, s] if flip else [s, c], 1)
    e_arg = arg.abs() * (3 * U32 * a + 5 * U32)
    err = torch.cat([e_arg, e_arg], 1) + 2.0 ** -22
    u = unit_roundoff(dtype)
    tol = (1 + u) * err + u * ref.abs() + (2.0 ** -25 if dtype == torch.float16 else 0.0)
    ldo = ch + 12

    def run():
        buf = torch.full((len(t), ldo), SENT16, dtype=torch.int16, device="cuda")
        ops.sinusoid(in_block(t), ch, buf.view(dtype)[:, :ch], flip_sin_to_cos=flip, downscale_freq_shift=shift)
        torch.cuda.synchronize()
        return buf

    buf = run()
    assert (buf[:, ch:] == SENT16).all(), "wrote into the output pitch"
    check(buf.view(dtype)[:, :ch].float(), ref, tol, "sinusoid_flip%d_shift%d_%s" % (flip, shift, dtype))
    assert torch.equal(run(), buf)


# --------------------------------------------------------------------------------------------
# patchify, upsample_nearest (bit-exact)
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("P", [1, 2])
def test_patchify_bit_exact(P, dtype):
    from opendwm_b200 import ops
    n, C, H, W = 3, 5, 6, 10
    x = torch.randn(n, C, H, W, generator=_g(P)) * 3
    Hp, Wp = H // P, W // P
    ref = x.view(n, C, Hp, P, Wp, P).permute(0, 2, 4, 1, 3, 5).reshape(n * Hp * Wp, C * P * P).to(dtype)
    cols = C * P * P
    ldo = cols + 7

    def run():
        buf = torch.full((n * Hp * Wp, ldo), SENT16, dtype=torch.int16, device="cuda")
        ops.patchify(in_block(x), P, buf.view(dtype)[:, :cols])
        torch.cuda.synchronize()
        return buf

    buf = run()
    assert (buf[:, cols:] == SENT16).all(), "wrote into the output pitch"
    assert torch.equal(buf[:, :cols].cpu(), ref.view(torch.int16))
    assert torch.equal(run(), buf)


def upsample_reference(x, compress_time):
    """CogVideoXUpsample3D: nearest x2 in space; with compress_time, an even T doubles every
    frame, an odd T > 1 keeps the first frame and doubles the rest, T = 1 stays one frame."""
    y = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
    T = x.shape[1]
    if compress_time and T > 1:
        if T % 2 == 0:
            y = y.repeat_interleave(2, 1)
        else:
            y = torch.cat([y[:, :1], y[:, 1:].repeat_interleave(2, 1)], 1)
    return y


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("T,compress", [(1, True), (4, True), (5, True), (3, False)])
@pytest.mark.parametrize("C", [4, 64])
def test_upsample_nearest_bit_exact(T, compress, C, dtype):
    from opendwm_b200 import ops
    x = torch.randn(2, T, 3, 5, C, generator=_g(T + C)) * 3
    ref = upsample_reference(x, compress).to(dtype)
    xd = in_block(x)
    out = ops.upsample_nearest(xd, compress, dtype)
    torch.cuda.synchronize()
    assert out.shape == ref.shape
    assert torch.equal(out.cpu().view(torch.int16), ref.view(torch.int16))
    assert torch.equal(ops.upsample_nearest(xd, compress, dtype), out)
    with pytest.raises(ValueError):
        ops.upsample_nearest(xd.transpose(2, 3), compress, dtype)


# --------------------------------------------------------------------------------------------
# embed (bit-exact)
# --------------------------------------------------------------------------------------------
SENT32 = 0x7FABCDEF
EMBED_GUARD = 3
EMBED_CASES = [
    # (D, seq, M, pos): D on both sides of the 128 / 256-thread switch at D = 1024; M not a
    # multiple of seq (the C API allows a partial last sequence)
    (4, 5, 23, True),
    (1020, 77, 251, True),
    (1024, 77, 251, True),
    (1284, 77, 160, True),
    (4096, 77, 100, False),
    (4096, 16, 50, True),
]


@pytest.mark.parametrize("D,seq,M,pos", EMBED_CASES, ids=["D%d_seq%d_M%d_pos%d" % c for c in EMBED_CASES])
def test_embed_bit_exact(D, seq, M, pos):
    """ids 0 and vocab - 1 among random ones; the table inside a NaN / +-Inf allocation; pos
    [seq + 3, D] whose rows past seq are NaN (the kernel must not read them); the output rows
    with a pitch of D + 8 inside sentinel guard rows.  Out-of-range ids trap by design and are
    not called here."""
    from opendwm_b200 import ops
    g = _g(D + seq + M)
    vocab = 1000
    tok = torch.randn(vocab, D, generator=g)
    ids = torch.randint(0, vocab, (M,), generator=g)
    ids[0], ids[M // 2], ids[-1] = vocab - 1, 0, vocab - 1
    p = torch.cat([torch.randn(seq, D, generator=g), torch.full((3, D), float("nan"))]) if pos else None
    want = torch.nn.functional.embedding(ids, tok)
    if pos:
        want = want + p[torch.arange(M) % seq]
    tokd, posd, idsd = in_poison(tok), None if p is None else in_block(p), ids.cuda()

    def run():
        buf = torch.full((M + 2 * EMBED_GUARD, D + 8), SENT32, dtype=torch.int32, device="cuda")
        ops.embed(idsd, tokd, buf[EMBED_GUARD:-EMBED_GUARD, :D].view(torch.float32), pos=posd, seq=seq)
        torch.cuda.synchronize()
        return buf

    buf = run()
    inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    inside[EMBED_GUARD:-EMBED_GUARD, :D] = True
    assert (buf[~inside] == SENT32).all(), "wrote outside the [M, D] rows"
    assert torch.equal(buf[EMBED_GUARD:-EMBED_GUARD, :D].cpu(), want.view(torch.int32))
    assert torch.equal(run(), buf), "the repeated call gave other bits"
