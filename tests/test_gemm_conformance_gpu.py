"""Element-wise conformance of the wgmma GEMM (dwm_b200_linear) and the implicit-GEMM
convolution (dwm_b200_conv) against float64, at the tile, remap and layout edges.

Both kernels share one fused epilogue (drain_tile) and pick their kernel variant silently:
tile width (pick_tile_n, conv_pick_bn), 1-CTA or a cluster of two CTAs, and for kw = 3 the
halo-row convolution.  Every GPU case therefore:

  * writes into views of sentinel-filled buffers with guard rows before and after and a row
    pitch `ldo > out_cols`: every element outside the expected write set (the gaps a row remap
    leaves included) must keep the sentinel's bits, every element inside must be finite and
    within `epilogue_reference`'s bound.  16-bit epilogues also scatter to two sentinel-filled
    peer buffers, which must equal `out` bit for bit;
  * reads operands whose padding the kernel must not read: A / W columns [K, ld) and the rows
    of the allocation past M / N hold NaN / +-Inf, and so does the bias past N and the pitch of
    resid / gate / blend_x; convolution inputs and weights sit inside NaN-filled allocations;
  * scales every third row of A and output channel of W up and every third one by 1e-3, so
    that an error in a small row or column cannot hide under a max-relative norm;
  * runs every kernel variant the options reach (gemm_2cta x gemm_bn, resid_tma; conv_2cta x
    conv_halo), restating the selection rules in `linear_kernel` / `conv_kernel`: variants
    that claim the same accumulation order must give the same bits, the halo-row kernel (other
    tap order) is held to the bound.  The default call is repeated and must repeat its bits.
    `test_kernel_selection` checks with torch.profiler that the rules pick the launched kernel.

The CPU self-test checks the bound itself against an emulated kernel and ten wrong ones.

Worst ratio |out - ref| / tol over this file's cases, measured on an H100 80GB HBM3 at a 700 W
power limit (bf16 / fp16): linear 16-bit and F32 0.995 / 0.996, linear RESID 0.909 / 0.909,
per-tap convolution 0.955 / 0.942, halo-row convolution 0.684 / 0.934; the text encoders'
QuickGELU STORE 0.994 / 0.988 and GEGLU_TANH 0.992 / 0.990 (same card, same limit).  These maxima sit in
the one-rounding terms (the 16-bit output, the fp32 fma of a residual far larger than the
product), which are exact.  Where the accumulation term dominates, fp32 outputs of sums of
K = 648 to 2880 products, the error is 0.2 to 0.8 % of acc_bound: the model's linear growth
and worst-case truncation are that loose for Hopper's accumulator on random data.
"""
import math
import re
import subprocess
import sys

import pytest
import torch

from opendwm_b200 import lib

STORE, GEGLU, QKNORM, RESID, F32 = lib.EPI_STORE, lib.EPI_GEGLU, lib.EPI_QKNORM, lib.EPI_RESID, lib.EPI_F32
GEGLU_TANH = lib.EPI_GEGLU_TANH
NONE, GELU_TANH, GELU_ERF, SILU, RELU, QUICK_GELU = (lib.ACT_NONE, lib.ACT_GELU_TANH, lib.ACT_GELU_ERF,
                                                     lib.ACT_SILU, lib.ACT_RELU, lib.ACT_QUICK_GELU)
EPI_STORE_QUICK_GELU = 16  # gemm_epilogue.cuh: the EPI template argument of STORE with act = QUICK_GELU
SENT16 = -21555          # int16 0xABCD: bits of every 16-bit element the call must not write
SENT32 = 0x7FABCDEF      # int32 bits of every fp32 element the call must not write (a NaN)
GUARD = 3                # sentinel rows before and after each output buffer
LDO_PAD = 24             # sentinel columns after the result in each output row
LD_PAD = 8               # poisoned columns after K in each A / W row (lda = K + 8)
ROW_PAD = 5              # poisoned rows after the M rows of A and the N rows of W
AUX_PAD = 8              # NaN columns after N in each resid / gate / blend_x row
POISON = (float("nan"), float("inf"), float("-inf"))
U32 = 2.0 ** -24         # fp32 unit roundoff (round to nearest)
K_GRP = 16               # products per accumulation block (one k16 wgmma)
C_ACC = K_GRP + 2        # ulps lost per block: K_GRP aligned products, the running sum, the normalisation
H100_SMS = 132           # the case labels name the kernels chosen on an H100 SXM


def unit_roundoff(dtype):
    return {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}[dtype]


def cdiv(a, b):
    return (a + b - 1) // b


# --------------------------------------------------------------------------------------------
# reference and bound
# --------------------------------------------------------------------------------------------
def acc_bound(P, K):
    """Bound on |acc - z| for the fp32 wgmma accumulator of z = sum_k a_k w_k, P = sum_k |a_k w_k|.

    Model: products of 16-bit values are exact in fp32.  The tensor core adds them in blocks of
    at most K_GRP = 16 (one k16 instruction; Hopper's internal blocking is not documented and
    published measurements of earlier NVIDIA tensor cores found blocks of 4 to 16).  Per block,
    the products and the running sum are aligned to the largest exponent among them with the
    bits below fp32's 24-bit significand truncated, added, and the sum normalised with
    truncation.  Each of the K_GRP products and the running sum then loses less than one ulp
    of the block's largest magnitude, and the normalisation one ulp of the result: C_ACC =
    K_GRP + 2 ulps, each at most 2^-23 of a magnitude that is at most the running P.  Over
    ceil(K / K_GRP) blocks:  |acc - z| <= C_ACC 2^-23 ceil(K / K_GRP) P.
    Reordering the blocks (the halo-row convolution sums its taps in another order) does not
    change the bound.  It is linear in the number of blocks, while truncation errors of random
    sign grow like its square root, so it is loose by design (see the measured ratios below)."""
    return C_ACC * 2.0 ** -23 * math.ceil(K / K_GRP) * P


# QuickGELU's derivative is SiLU's at u = 1.702 x, times 1.702 x / u = 1: the same constant
LIPSCHITZ = {NONE: 1.0, RELU: 1.0, GELU_TANH: 1.13, GELU_ERF: 1.13, SILU: 1.1, QUICK_GELU: 1.1}


def act_reference(x, act):
    """float64 act(x), and a bound on the error of the kernel's fp32 formula at x (common.cuh).
    gelu_tanh = x / (1 + __expf(-u2)) (__fdividef) and silu = x / (1 + __expf(-x)): __expf is
    accurate to (2 + 1.2 |u2|) ulps and the rounded u2 adds ~4 ulps of |u2|, which moves the
    result by (1 - sigmoid(u2)) times that relative error; the division and 1 + e add 2^-21.
    quick_gelu = x / (1 + __expf(-1.702f * x)) (gemm_epilogue.cuh, built without fast math: the
    division is IEEE) is silu's formula at u2 = 1.702 x: the constant 1.702f and the rounded
    product -1.702f * x move u2 by at most 2 ulps of |u2|, inside the 4 above, so it takes
    silu's bound with that u2.
    gelu_erf = 0.5 x (1 + erff(x / sqrt2)): erff is within 2 ulps, so 1 + erff has an absolute
    error below 2^-22, times |x| / 2."""
    zero = torch.zeros_like(x)
    if act == NONE:
        return x, zero
    if act == RELU:
        return x.clamp_min(0), zero
    if act == GELU_ERF:
        y = 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
        return y, 2.0 ** -22 * (x.abs() + y.abs())
    if act == SILU:
        u2 = x
    elif act == QUICK_GELU:
        u2 = 1.702 * x
    else:
        u2 = 2 * 0.7978845608028654 * (x + 0.044715 * x ** 3)
    s = torch.sigmoid(u2)
    y = x * s
    return y, y.abs() * (2.0 ** -21 + (2.0 ** -22 + 2.0 ** -20 * u2.abs()) * (1 - s))


class Epi:
    """One epilogue as include/dwm_b200.h defines it, with its fp32 operands (logical views)."""

    def __init__(self, kind, act=NONE, bias=None, resid=None, resid_row_mod=0, gate=None,
                 blend_x=None, alpha=None, rows_per_batch=0, rows_per_item=0, out_item_stride=0,
                 out_row_offset=0, qw=None, kw=None, qk_region=0, regions=0, eps=1e-6):
        self.kind, self.act, self.bias = kind, act, bias
        self.resid, self.resid_row_mod, self.gate = resid, resid_row_mod, gate
        self.blend_x, self.alpha, self.rows_per_batch = blend_x, alpha, rows_per_batch
        self.rows_per_item, self.out_item_stride, self.out_row_offset = \
            rows_per_item, out_item_stride, out_row_offset
        self.qw, self.kw, self.qk_region, self.regions = qw, kw, qk_region, regions or 2
        self.eps = torch.tensor(eps, dtype=torch.float32).item()

    @property
    def out16(self):
        return self.kind in (STORE, GEGLU, QKNORM, GEGLU_TANH)

    @property
    def gated(self):
        return self.kind in (GEGLU, GEGLU_TANH)

    def out_cols(self, N):
        return N // 2 if self.gated else N

    def out_rows(self, M):
        """Output row of each of the M result rows (16-bit outputs are remapped)."""
        m = torch.arange(M)
        if not self.out16:
            return m
        rpi = self.rows_per_item
        o = (m // rpi) * self.out_item_stride + m % rpi if rpi > 0 else m
        return o + self.out_row_offset

    def operands(self, M, bug=None):
        """float64 residual, gate, blend rows and alpha of each result row (None if absent).
        `bug` reads one of them from the wrong row (the self-test's wrong kernels)."""
        m = torch.arange(M)
        dev = next((t.device for t in (self.resid, self.gate, self.blend_x) if t is not None), None)
        item = m // self.rows_per_item if self.rows_per_item > 0 else torch.zeros_like(m)
        R = G = X = al = None
        if self.resid is not None:
            mod = self.resid_row_mod
            if mod > 0:
                rr = (m + (1 if bug == "resid row + 1" else 0)) % mod
            else:
                rr = item if mod < 0 else m
            R = self.resid.double()[rr.to(dev)]
        if self.gate is not None:
            gi = item + 1 if bug == "gate of item + 1" else item
            G = self.gate.double()[gi.clamp_max(self.gate.shape[0] - 1).to(dev)]
        if self.blend_x is not None:
            X = self.blend_x.double()[:M]
            b = m // self.rows_per_batch if self.rows_per_batch > 0 else torch.zeros_like(m)
            if bug == "alpha of the next batch":
                b = (b + 1) % self.alpha.numel()
            al = self.alpha.double()[b.to(dev)][:, None]
        return R, G, X, al


def geglu_columns(N):
    """(value, gate) accumulator columns of each GEGLU output column (256-column packing)."""
    j = torch.arange(N // 2)
    v = 256 * (j // 128) + j % 128
    return v, v + 128


def epilogue_reference(z, P, K, e, out_dtype, acc_err=None):
    """float64 (ref, tol) of the epilogue `e` applied to z = A W^T (float64, from the 16-bit
    operands the kernel reads), P = |A| |W|^T, [M, out_cols].  The kernel conforms where
    |out - ref| <= tol.

    tol propagates the accumulation bound E = acc_bound(P, K) (or `acc_err`, a bound on
    |acc - z| the caller derived otherwise, e.g. for FP8 operands) through the epilogue's fp32 steps
    (unit roundoff U32 = 2^-24 each, round to nearest):
      * pre = acc + bias: E_pre = E + U32 |pre|;
      * STORE / F32: L E_pre + the activation's own error (act_reference), with L its Lipschitz
        constant (1.13 for both GELUs, 1.1 for SiLU, 1 for ReLU / none);
      * RESID: v = fma(pre, g, r): |g| E_pre + U32 |v|; blend, fma(a, x, (1 - a) v) with 1 - a
        rounded in fp32: |1 - a| E_v + 2 U32 |(1 - a) v| + U32 |out|;
      * GEGLU / GEGLU_TANH: x * gelu(y), gelu_erf / gelu_tanh: |gelu(y)| E_x + |x| (1.13 E_y +
        the activation's own error) + U32 |out|;
      * QKNORM: y = v r w with r = rsqrt(mean(v^2) + eps): to first order |w| r (E_v +
        |v| r max_head E_v) (the perturbation of r is at most r^2 max E_v), plus 2^-18 |y| for
        the fp32 64-term sum of squares (<= 2^-19 relative), rsqrtf and the two products;
      * a 16-bit output is rounded once more: (1 + u) tol + u |ref|, u = 2^-8 (bf16), 2^-11 (fp16).
    Floors: 2^-20 (P + |bias|) (scaled by |gate| for RESID, by |w| r for a normalised head)
    covers results far below their operands' magnitude, e.g. gelu_tanh's __fdividef returning 0
    where the true value is about -1e-37; fp16 outputs add 2^-25, half the spacing of fp16
    subnormals."""
    M, N = z.shape
    u = unit_roundoff(out_dtype)
    sub = 2.0 ** -25 if out_dtype == torch.float16 else 0.0
    b = e.bias.double()[:N].to(z.device) if e.bias is not None else torch.zeros(N, dtype=z.dtype, device=z.device)
    pre = z + b
    e_pre = (acc_bound(P, K) if acc_err is None else acc_err) + U32 * pre.abs()
    scale = P + b.abs()
    floor = 2.0 ** -20 * scale
    if e.kind in (STORE, F32):
        y, e_act = act_reference(pre, e.act)
        err = LIPSCHITZ[e.act] * e_pre + e_act
    elif e.kind == RESID:
        R, G, X, al = e.operands(M)
        g = G if G is not None else torch.ones_like(pre)
        v = pre * g + (R if R is not None else 0.0)
        err = g.abs() * e_pre + U32 * v.abs()
        floor = floor * g.abs()
        y = v
        if X is not None:
            a1 = 1 - al
            y = al * X + a1 * v
            err = a1.abs() * err + 2 * U32 * (a1 * v).abs() + U32 * y.abs()
            floor = floor * a1.abs()
    elif e.gated:
        vc, gc = (c.to(z.device) for c in geglu_columns(N))
        x, yg = pre[:, vc], pre[:, gc]
        ge, e_ge = act_reference(yg, GELU_ERF if e.kind == GEGLU else GELU_TANH)
        y = x * ge
        err = ge.abs() * e_pre[:, vc] + x.abs() * (1.13 * e_pre[:, gc] + e_ge) + U32 * y.abs()
        floor = 2.0 ** -20 * (scale[:, vc] * ge.abs() + x.abs() * scale[:, gc])
    else:  # QKNORM
        y, err, floor = pre.clone(), e_pre.clone(), floor.clone()
        for h in range(N // 64):
            c = slice(64 * h, 64 * h + 64)
            region = 64 * h // e.qk_region
            if region >= e.regions:
                continue
            w = (e.qw if region == 0 else e.kw).double().to(z.device)
            v, ev = pre[:, c], e_pre[:, c]
            r = torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + e.eps)
            y[:, c] = v * r * w
            err[:, c] = w.abs() * r * (ev + v.abs() * r * ev.amax(-1, keepdim=True)) + 2.0 ** -18 * y[:, c].abs()
            floor[:, c] = 2.0 ** -20 * w.abs() * r * scale[:, c]
    tol = (1 + u) * err + u * y.abs() + floor + sub
    return y, tol


def bound_violations(out, ref, tol):
    """Elements outside |out - ref| <= tol (NaN / Inf count as violations), and the worst ratio."""
    err = (out.double() - ref).abs()
    bad = ~(err <= tol)
    ratio = torch.where(err == 0, 0.0, err / tol)
    ratio = torch.where(torch.isnan(ratio), math.inf, ratio)
    return bad, ratio.max().item() if ratio.numel() else 0.0


# --------------------------------------------------------------------------------------------
# emulated kernel (CPU)
# --------------------------------------------------------------------------------------------
def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _act32(x, act):
    if act == QUICK_GELU:
        return x * torch.sigmoid(1.702 * x)
    if act == GELU_TANH:
        return x * torch.sigmoid(2 * 0.7978845608028654 * (x + 0.044715 * x * x * x))
    if act == GELU_ERF:
        return torch.nn.functional.gelu(x)
    if act == SILU:
        return torch.nn.functional.silu(x)
    if act == RELU:
        return x.clamp_min(0)
    return x


def emulate(a, w, e, out_dtype, bug=None):
    """fp32 kernel: the accumulator adds each 64-wide k-block of A W^T with one rounding (the
    order the pipeline consumes them), then the epilogue in fp32 with its explicit roundings,
    then one rounding to the output type.  `bug` makes it one of the wrong kernels."""
    M, K = a.shape
    N = w.shape[0]
    a64, w64 = a.double(), w.double()
    acc = torch.zeros(M, N)
    starts = list(range(0, K, 64))
    if bug == "last k-block dropped":
        starts = starts[:-1]
    for k0 in starts:
        acc = (acc.double() + a64[:, k0:k0 + 64] @ w64[:, k0:k0 + 64].T).float()
    b = e.bias.float().clone() if e.bias is not None else torch.zeros(N)
    if bug == "no bias on chunk 1":
        b[32:64] = 0
    return emulate_epilogue(acc + b, e, out_dtype, bug)


def emulate_epilogue(pre, e, out_dtype, bug=None):
    """The fp32 epilogue after the bias, pre = acc + bias [M, N] fp32, then one rounding to the
    output type."""
    M, N = pre.shape
    if e.kind in (STORE, F32):
        act = SILU if bug == "sigmoid(x) for sigmoid(1.702 x)" else e.act
        y = _act32(pre, act)
    elif e.kind == RESID:
        R, G, X, al = e.operands(M, bug)
        y = _fma(pre, G if G is not None else torch.ones_like(pre), R if R is not None else torch.zeros_like(pre))
        if X is not None:
            a_ = al.float()
            y = _fma(a_, X, (1 - a_) * y)
    elif e.gated:
        vc, gc = geglu_columns(N)
        if bug == "GEGLU halves swapped":
            vc, gc = gc, vc
        tanh = e.kind == GEGLU_TANH and bug != "erf GELU on the gate"
        y = pre[:, vc] * _act32(pre[:, gc], GELU_TANH if tanh else GELU_ERF)
    else:
        y = pre.clone()
        for h in range(N // 64):
            c = slice(64 * h, 64 * h + 64)
            region = 64 * h // e.qk_region
            if region >= e.regions:
                continue
            v = pre[:, c]
            n = 63 if bug == "RMS over 63 columns" else 64
            inv = torch.rsqrt((v[:, :n] * v[:, :n]).sum(-1, keepdim=True) / n + e.eps)
            y[:, c] = v * inv * (e.qw if region == 0 else e.kw).float()
    return y.to(out_dtype)


def row_scales(n, big):
    """1 on rows 0, 3, 6, ...; `big` on rows 1, 4, ...; 1e-3 on rows 2, 5, ..."""
    s = torch.ones(n)
    s[1::3] = big
    s[2::3] = 1e-3
    return s


def make_operands(M, N, K, dtype, big, seed):
    """16-bit A [M, K] (std 1) and W [N, K] (std K^-1/2) with scaled rows / output channels."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g) * row_scales(M, big)[:, None]
    w = torch.randn(N, K, generator=g) * K ** -0.5 * row_scales(N, big)[:, None]
    return a.to(dtype), w.to(dtype)


def big_scale(dtype, out16):
    """Largest row / channel scale: 1e3, but 4 for fp16 outputs (GEGLU squares it; fp16 <= 65504)."""
    return 4.0 if (dtype == torch.float16 and out16) else 1e3


# --------------------------------------------------------------------------------------------
# CPU self-test of the bound
# --------------------------------------------------------------------------------------------
def _selftest_specs():
    g = torch.Generator().manual_seed(7)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    M = 48
    return [
        ("STORE gelu_tanh", 96, Epi(STORE, GELU_TANH, bias=rn(96)), ["last k-block dropped"]),
        ("STORE bias", 96, Epi(STORE, bias=rn(96)), ["no bias on chunk 1"]),
        ("F32 silu", 96, Epi(F32, SILU, bias=rn(96)), ["last k-block dropped"]),
        ("RESID gate", 96, Epi(RESID, bias=rn(96), resid=rn(M, 96), gate=rn(6, 96), rows_per_item=8),
         ["gate of item + 1"]),
        ("RESID row mod", 96, Epi(RESID, resid=rn(12, 96), resid_row_mod=12), ["resid row + 1"]),
        ("RESID blend", 96, Epi(RESID, bias=rn(96), resid=rn(M, 96), blend_x=rn(M, 96),
                                alpha=torch.tensor([0.3, 0.8]), rows_per_batch=24),
         ["alpha of the next batch"]),
        ("QKNORM", 192, Epi(QKNORM, bias=rn(192), qw=rn(64) * 0.2 + 1, kw=rn(64) * 0.2 + 1,
                            qk_region=64), ["RMS over 63 columns"]),
        ("GEGLU", 256, Epi(GEGLU, bias=rn(256)), ["GEGLU halves swapped"]),
        ("STORE quick_gelu", 96, Epi(STORE, QUICK_GELU, bias=rn(96)), ["sigmoid(x) for sigmoid(1.702 x)"]),
        ("GEGLU_TANH", 256, Epi(GEGLU_TANH, bias=rn(256)), ["GEGLU halves swapped", "erf GELU on the gate"]),
    ]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_bound_accepts_emulated_kernel_and_rejects_wrong_ones(dtype):
    """Per epilogue (M = 48, K = 256 = four k-blocks, scaled rows and channels): the fp32
    emulation passes the bound, and each wrong kernel fails it."""
    M, K = 48, 256
    for name, N, e, bugs in _selftest_specs():
        out_dtype = dtype if e.out16 else torch.float32
        a, w = make_operands(M, N, K, dtype, big_scale(dtype, e.out16), seed=N)
        z = a.double() @ w.double().T
        P = a.double().abs() @ w.double().abs().T
        ref, tol = epilogue_reference(z, P, K, e, out_dtype)
        bad, worst = bound_violations(emulate(a, w, e, out_dtype), ref, tol)
        assert not bad.any(), (name, worst)
        if e.out16:
            assert worst > 0.05, (name, worst)   # the 16-bit rounding alone nearly fills it
        for bug in bugs:
            bad, worst = bound_violations(emulate(a, w, e, out_dtype, bug), ref, tol)
            assert bad.any(), (name, bug, worst)


# --------------------------------------------------------------------------------------------
# kernel selection, restated from gemm.cu / conv.cu
# --------------------------------------------------------------------------------------------
def pick_tile_n(M, N, kind, cl, sms, gemm_bn=0):
    if kind in (GEGLU, GEGLU_TANH):
        return 256
    if gemm_bn in (128, 256):
        return gemm_bn
    slots = sms // cl
    m_groups = cdiv(cdiv(M, 128), cl)
    w256 = cdiv(m_groups * cdiv(N, 256), slots)
    w128 = cdiv(m_groups * cdiv(N, 128), slots)
    return 128 if w128 * 128 * 10 < w256 * 256 * 9 else 256


def linear_kernel(M, N, kind, sms, gemm_2cta=1, gemm_bn=0):
    """(NT, CL) of the gemm_wgmma_kernel dwm_b200_linear launches."""
    cl = 2 if gemm_2cta == 1 and M >= 512 else 1
    return pick_tile_n(M, N, kind, cl, sms, gemm_bn), cl


def conv_kernel(nb, t_out, h, w, c_out, kw, sms, conv_2cta=1, conv_halo=1):
    """(CBN, CL, HALO) of the conv_wgmma_kernel dwm_b200_conv launches."""
    cbn = next(n for n in (256, 128, 64, 32) if c_out % n == 0)
    bw = min(w, 128)
    bh = max(1, min(128 // bw, h))
    m_tiles = nb * t_out * cdiv(w, bw) * cdiv(h, bh)
    seg_tiles = nb * t_out * h * cdiv(w, 128)
    n_blocks = c_out // cbn
    if cbn <= 128 and conv_halo == 1 and kw == 3 and w >= 128 and seg_tiles * n_blocks >= sms:
        return cbn, 1, True
    if cbn >= 64 and conv_2cta == 1 and m_tiles * n_blocks >= 2 * sms:
        return cbn, 2, False
    return cbn, 1, False


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _label(k):
    return "NT%d_CL%d" % k[:2] + ("_HALO" if len(k) > 2 and k[2] else "")


# --------------------------------------------------------------------------------------------
# GPU buffers
# --------------------------------------------------------------------------------------------
def _poison(n):
    return torch.tensor(POISON).repeat(n // 3 + 1)[:n]


def poisoned_2d(t, ld_pad=LD_PAD):
    """CUDA view of t [R, C] inside an allocation with `ld_pad` poisoned columns per row and
    ROW_PAD poisoned rows after it (E4M3: the NaN bytes 0x7F / 0xFF)."""
    R, C = t.shape
    x = _poison((R + ROW_PAD) * (C + ld_pad)).view(R + ROW_PAD, C + ld_pad).to(t.dtype)
    x[:R, :C] = t
    return x.cuda()[:R, :C]


def pitched(t):
    """CUDA fp32 view of t [R, C] with AUX_PAD NaN / Inf columns after each row."""
    R, C = t.shape
    x = _poison(R * (C + AUX_PAD)).view(R, C + AUX_PAD)
    x[:, :C] = t
    return x.cuda()[:, :C]


def padded_vec(t, pad=32):
    x = _poison(t.numel() + pad)
    x[:t.numel()] = t
    return x.cuda()[:t.numel()]


def in_nan_block(t, pad=4096):
    """Contiguous CUDA tensor of t's shape placed `pad` elements into a NaN-filled allocation."""
    n = t.numel()
    x = torch.full((n + 2 * pad,), float("nan"), dtype=t.dtype)
    x[pad:pad + n] = t.reshape(-1)
    return x.cuda()[pad:pad + n].view(t.shape)


def sentinel_buffer(rows, cols, dtype):
    """[rows + 2 GUARD, cols + LDO_PAD] of sentinel bits, as `dtype`."""
    if dtype == torch.float32:
        return torch.full((rows + 2 * GUARD, cols + LDO_PAD), SENT32, dtype=torch.int32,
                          device="cuda").view(torch.float32)
    return torch.full((rows + 2 * GUARD, cols + LDO_PAD), SENT16, dtype=torch.int16,
                      device="cuda").view(dtype)


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _record(family, name, worst):
    print("BOUND_RATIO %s %s %.4g" % (family, name, worst))


def check_output(buf, orows, out_cols, ref, tol, what):
    """Sentinel bits outside rows `orows` x columns [0, out_cols); finite values within the bound
    inside.  Returns the worst bound ratio."""
    rows = (orows + GUARD).to(buf.device)
    w = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    w[rows, :out_cols] = True
    sent = SENT32 if buf.dtype == torch.float32 else SENT16
    stray = _bits(buf)[~w] != sent
    assert not stray.any(), "%s: %d element(s) written outside the result" % (what, stray.sum())
    got = buf[rows, :out_cols]
    bad, worst = bound_violations(got, ref, tol)
    if bad.any():
        m, n = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(
            "%s: %d of %d outside the float64 bound (worst ratio %.3g, non-finite %d); first at "
            "row %d col %d: got %r ref %r tol %r" % (
                what, bad.sum(), bad.numel(), worst, (~torch.isfinite(got)).sum(), m, n,
                got[m, n].item(), ref[m, n].item(), tol[m, n].item()))
    return worst


class _Options:
    """Sets dwm_b200 options for a block and restores their defaults."""
    DEFAULTS = {"gemm_2cta": 1, "gemm_bn": 0, "resid_tma": 1, "conv_2cta": 1, "conv_halo": 1}

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        for k, v in self.kw.items():
            lib.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            lib.set_option(k, self.DEFAULTS[k])


# --------------------------------------------------------------------------------------------
# linear cases
# --------------------------------------------------------------------------------------------
def _lin(name, M, N, K, kind, label, **opt):
    return (name, (M, N, K, kind, opt), label)


LINEAR_CASES = [
    # STORE: no bias, each activation, every M / N / K edge
    _lin("store_M1_N32_K8", 1, 32, 8, STORE, "NT128_CL1"),
    _lin("store_gelu_tanh_M127_N96_K72", 127, 96, 72, STORE, "NT128_CL1", act=GELU_TANH, bias=True),
    _lin("store_gelu_erf_M129_N288_K1536", 129, 288, 1536, STORE, "NT128_CL1", act=GELU_ERF, bias=True),
    _lin("store_silu_M511_N6144_K72", 511, 6144, 72, STORE, "NT256_CL1", act=SILU, bias=True),
    _lin("store_relu_M512_N288_K6144", 512, 288, 6144, STORE, "NT128_CL2", act=RELU, bias=True),
    _lin("store_M513_N6144_K1536", 513, 6144, 1536, STORE, "NT128_CL2", bias=True),
    _lin("store_silu_M513_N96_K6144", 513, 96, 6144, STORE, "NT128_CL2", act=SILU),
    _lin("store_remap_M300_N288_K72", 300, 288, 72, STORE, "NT128_CL1", bias=True,
         rows_per_item=100, out_item_stride=130, out_row_offset=7),
    # F32: rows_per_item / offsets must not remap fp32 outputs
    _lin("f32_gelu_tanh_M513_N288_K1536", 513, 288, 1536, F32, "NT128_CL2", act=GELU_TANH, bias=True),
    _lin("f32_items_M129_N96_K8", 129, 96, 8, F32, "NT128_CL1", bias=True, rows_per_item=50,
         out_row_offset=5),
    # RESID
    _lin("resid_M513_N288_K1536", 513, 288, 1536, RESID, "NT128_CL2", bias=True, resid="full"),
    _lin("resid_mod_gate_M511_N96_K72", 511, 96, 72, RESID, "NT128_CL1", bias=True, resid="mod",
         gate=True, rows_per_item=100),
    _lin("resid_item_M129_N6144_K1536", 129, 6144, 1536, RESID, "NT128_CL1", bias=True,
         resid="item", rows_per_item=43),
    _lin("resid_blend_gate_M513_N288_K1536", 513, 288, 1536, RESID, "NT128_CL2", bias=True,
         resid="full", gate=True, rows_per_item=57, blend=(0.0, 0.3, 1.0)),
    _lin("resid_inplace_gate_M512_N96_K6144", 512, 96, 6144, RESID, "NT128_CL2", bias=True,
         resid="full", gate=True, rows_per_item=128, inplace="resid"),
    _lin("resid_inplace_blend_M127_N288_K72", 127, 288, 72, RESID, "NT128_CL1", bias=True,
         resid="full", blend=(0.3, 1.0), inplace="blend"),
    _lin("resid_nobias_M1_N32_K8", 1, 32, 8, RESID, "NT128_CL1", resid="full"),
    # GEGLU (always 256 wide)
    _lin("geglu_M513_N512_K1536", 513, 512, 1536, GEGLU, "NT256_CL2", bias=True),
    _lin("geglu_nobias_M127_N256_K72", 127, 256, 72, GEGLU, "NT256_CL1"),
    _lin("geglu_remap_M300_N768_K72", 300, 768, 72, GEGLU, "NT256_CL1", bias=True,
         rows_per_item=100, out_item_stride=110, out_row_offset=3),
    # QKNORM, D = 320: region boundaries inside 256-wide tiles
    _lin("qknorm2_M513_N960_K1536", 513, 960, 1536, QKNORM, "NT128_CL2", bias=True, qk_region=320,
         regions=2),
    _lin("qknorm1_M129_N960_K72", 129, 960, 72, QKNORM, "NT128_CL1", qk_region=320, regions=1),
    # the DiT's joint q|k|v buffer: items of S = 100 sample and L = 30 context rows
    _lin("qknorm_joint_sample_M300_N960_K72", 300, 960, 72, QKNORM, "NT128_CL1", bias=True,
         qk_region=320, regions=2, rows_per_item=100, out_item_stride=130, out_row_offset=0,
         out_total=390),
    _lin("qknorm_joint_context_M90_N960_K72", 90, 960, 72, QKNORM, "NT128_CL1", bias=True,
         qk_region=320, regions=2, rows_per_item=30, out_item_stride=130, out_row_offset=100,
         out_total=390),
    # text encoders.  CLIP-L's fc1 for one prompt of 77 tokens, and for 12 (a CFG window's
    # distinct prompts)
    _lin("store_quick_gelu_M77_N3072_K768", 77, 3072, 768, STORE, "NT128_CL1", act=QUICK_GELU,
         bias=True),
    _lin("store_quick_gelu_M924_N3072_K768", 924, 3072, 768, STORE, "NT256_CL2", act=QUICK_GELU,
         bias=True),
    _lin("store_quick_gelu_remap_M301_N352_K72", 301, 352, 72, STORE, "NT128_CL1", act=QUICK_GELU,
         bias=True, rows_per_item=77, out_item_stride=90, out_row_offset=4),
    # T5's gated tanh-GELU (always 256 wide)
    _lin("geglu_tanh_nobias_M77_N512_K256", 77, 512, 256, GEGLU_TANH, "NT256_CL1"),
    _lin("geglu_tanh_M616_N1536_K1024", 616, 1536, 1024, GEGLU_TANH, "NT256_CL2", bias=True),
    _lin("geglu_tanh_remap_M300_N768_K72", 300, 768, 72, GEGLU_TANH, "NT256_CL1", bias=True,
         rows_per_item=100, out_item_stride=110, out_row_offset=3),
]


def _family(kind, act):
    """The BOUND_RATIO family of a linear case."""
    if kind == RESID:
        return "linear_resid"
    if kind == GEGLU_TANH:
        return "linear_geglu_tanh"
    return "linear_quick_gelu" if act == QUICK_GELU else "linear"


def _linear_inputs(M, N, K, kind, opt, dtype):
    a, w = make_operands(M, N, K, dtype, big_scale(dtype, Epi(kind).out16), seed=M * 7 + N + K)
    g = torch.Generator().manual_seed(M + N + K)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    rpi = opt.get("rows_per_item", 0)
    items = cdiv(M, rpi) if rpi else 1
    e = Epi(kind, act=opt.get("act", NONE), rows_per_item=rpi,
            out_item_stride=opt.get("out_item_stride", 0), out_row_offset=opt.get("out_row_offset", 0))
    if opt.get("bias"):
        e.bias = padded_vec(rn(N) * 0.5)
    if kind == RESID:
        mode = opt.get("resid")
        if mode == "mod":
            e.resid_row_mod = 37
            e.resid = pitched(rn(37, N))
        elif mode == "item":
            e.resid_row_mod = -1
            e.resid = pitched(rn(items, N))
        elif mode == "full":
            e.resid = pitched(rn(M, N))
        if opt.get("gate"):
            e.gate = pitched(rn(items, N))
        if opt.get("blend"):
            e.blend_x = pitched(rn(M, N))
            e.alpha = torch.tensor(opt["blend"], dtype=torch.float32).cuda()
            e.rows_per_batch = cdiv(M, len(opt["blend"]))
    if kind == QKNORM:
        e.qw, e.kw = (rn(64) * 0.2 + 1).cuda(), (rn(64) * 0.2 + 1).cuda()
        e.qk_region, e.regions = opt["qk_region"], opt["regions"]
    return poisoned_2d(a), poisoned_2d(w), e


def _launch_linear(A, W, e, opt, dtype, gemm_2cta=1, gemm_bn=0, resid_tma=1):
    """One call into fresh sentinel buffers; returns [out buffer, peer buffers...]."""
    from opendwm_b200 import ops
    M, N = A.shape[0], W.shape[0]
    odt = dtype if e.out16 else torch.float32
    cols = e.out_cols(N)
    rows = max(int(e.out_rows(M).max()) + 1, opt.get("out_total", 0))
    bufs = [sentinel_buffer(rows, cols, odt) for _ in range(3 if e.out16 else 1)]
    view = lambda b: b[GUARD:GUARD + rows, :cols]  # noqa: E731
    out = view(bufs[0])
    resid, blend_x = e.resid, e.blend_x
    if opt.get("inplace") == "resid":
        out[:M, :N] = resid
        resid = out
    elif opt.get("inplace") == "blend":
        out[:M, :N] = blend_x
        blend_x = out
    with _Options(gemm_2cta=gemm_2cta, gemm_bn=gemm_bn, resid_tma=resid_tma):
        ops.linear(A, W, e.bias, epilogue=e.kind, act=e.act, out=out,
                   rows_per_item=e.rows_per_item, out_item_stride=e.out_item_stride,
                   out_row_offset=e.out_row_offset, q_norm_weight=e.qw, k_norm_weight=e.kw,
                   qk_region=e.qk_region, eps=e.eps, qk_norm_regions=e.regions if e.kind == QKNORM else 0,
                   peer_out=[view(b).data_ptr() for b in bufs[1:]] or None,
                   resid=resid, resid_row_mod=e.resid_row_mod, gate=e.gate, blend_x=blend_x,
                   alpha=e.alpha, rows_per_batch=e.rows_per_batch)
        torch.cuda.synchronize()
    return bufs


DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,shape,label", LINEAR_CASES,
                         ids=["%s_%s" % (c[0], c[2]) for c in LINEAR_CASES])
def test_linear_conforms(name, shape, label, dtype):
    """`label` is the kernel (tile width, CTAs per cluster) the default options reach on an H100."""
    M, N, K, kind, opt = shape
    sms = _sms()
    if sms == H100_SMS:
        assert _label(linear_kernel(M, N, kind, sms)) == label
    A, W, e = _linear_inputs(M, N, K, kind, opt, dtype)
    z = A.double() @ W.double().T
    P = A.double().abs() @ W.double().abs().T
    ref, tol = epilogue_reference(z, P, K, e, dtype if e.out16 else torch.float32)
    b0 = _launch_linear(A, W, e, opt, dtype)
    worst = check_output(b0[0], e.out_rows(M), e.out_cols(N), ref, tol, name)
    for i, p in enumerate(b0[1:]):
        assert torch.equal(_bits(p), _bits(b0[0])), "peer_out[%d] differs from out" % i
    same = lambda bufs: all(torch.equal(_bits(x), _bits(y)) for x, y in zip(bufs, b0))  # noqa: E731
    assert same(_launch_linear(A, W, e, opt, dtype)), "the repeated call gave other bits"
    # every other kernel the options reach accumulates in the same order: the same bits
    seen = {linear_kernel(M, N, kind, sms)}
    for two in (1, 0):
        for bn in (128, 256):
            k = linear_kernel(M, N, kind, sms, two, bn)
            if k not in seen:
                seen.add(k)
                assert same(_launch_linear(A, W, e, opt, dtype, two, bn)), \
                    "%s gave other bits than %s" % (_label(k), label)
    if kind == RESID:
        assert same(_launch_linear(A, W, e, opt, dtype, resid_tma=0)), "resid_tma = 0 gave other bits"
    _record(_family(kind, opt.get("act", NONE)), "%s_%s" % (name, dtype), worst)


# --------------------------------------------------------------------------------------------
# convolution cases
# --------------------------------------------------------------------------------------------
def _cv(name, nb, t_out, h, w, c_in, c_out, kernel, epi, label):
    return (name, (nb, t_out, h, w, c_in, c_out, kernel, epi), label)


CONV_CASES = [
    _cv("w1_k133_cin8_cout32_store_silu", 2, 1, 7, 1, 8, 32, (1, 3, 3), "store_silu", "NT32_CL1"),
    _cv("w3_k333_cin72_cout96_f32", 1, 2, 5, 3, 72, 96, (3, 3, 3), "f32", "NT32_CL1"),
    _cv("w56_h5_k133_cin72_cout320_resid", 2, 1, 5, 56, 72, 320, (1, 3, 3), "resid", "NT64_CL1"),
    _cv("w56_h65_k133_cin72_cout384_f32_pair_odd", 3, 1, 65, 56, 72, 384, (1, 3, 3), "f32",
        "NT128_CL2"),
    _cv("w127_k111_cin320_cout384_resid_item", 2, 1, 3, 127, 320, 384, (1, 1, 1), "resid_item",
        "NT128_CL1"),
    _cv("w128_h48_k133_cin72_cout96_f32_halo", 1, 1, 48, 128, 72, 96, (1, 3, 3), "f32",
        "NT32_CL1_HALO"),
    _cv("w129_h40_k333_cin8_cout384_blend_self_halo", 1, 2, 40, 129, 8, 384, (3, 3, 3), "blend_self",
        "NT128_CL1_HALO"),
    _cv("w130_h17_k311_cin320_cout512_resid_item_pair", 1, 4, 17, 130, 320, 512, (3, 1, 1),
        "resid_item", "NT256_CL2"),
    _cv("w200_h14_k133_cin320_cout320_store_silu_halo", 1, 1, 14, 200, 320, 320, (1, 3, 3),
        "store_silu", "NT64_CL1_HALO"),
    _cv("w448_h3_k333_cin72_cout512_blend", 1, 1, 3, 448, 72, 512, (3, 3, 3), "blend", "NT256_CL1"),
    _cv("w448_h12_k133_cin8_cout384_resid_halo", 1, 1, 12, 448, 8, 384, (1, 3, 3), "resid",
        "NT128_CL1_HALO"),
    _cv("w130_h6_k111_cin72_cout32_f32", 2, 1, 6, 130, 72, 32, (1, 1, 1), "f32", "NT32_CL1"),
]


def _conv_inputs(shape, dtype):
    nb, t_out, h, w, c_in, c_out, kernel, epi = shape
    kt, kh, kw = kernel
    tp = t_out + kt - 1
    rows = nb * t_out * h * w
    g = torch.Generator().manual_seed(rows + c_in + c_out)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    big = big_scale(dtype, epi == "store_silu")
    x = rn(nb, tp, h, w, c_in) * row_scales(nb * tp * h * w, big).view(nb, tp, h, w, 1)
    taps = kt * kh * kw
    wt = rn(taps, c_out, c_in) * (taps * c_in) ** -0.5 * row_scales(c_out, big).view(1, c_out, 1)
    x, wt = in_nan_block(x.to(dtype)), in_nan_block(wt.to(dtype))
    e = Epi(STORE if epi.startswith("store") else F32 if epi == "f32" else RESID,
            act=SILU if epi == "store_silu" else NONE, bias=padded_vec(rn(c_out) * 0.5))
    if epi == "resid":
        e.resid = pitched(rn(rows, c_out))
    elif epi == "resid_item":
        e.resid_row_mod, e.rows_per_item = -1, h * w
        e.resid = pitched(rn(nb * t_out, c_out))
    elif epi in ("blend", "blend_self"):
        e.resid = pitched(rn(rows, c_out))
        e.blend_x = e.resid if epi == "blend_self" else pitched(rn(rows, c_out))
        e.alpha = torch.tensor([0.3, 0.0, 1.0][:nb * t_out] if nb * t_out > 1 else [0.3]).cuda()
        e.rows_per_batch = cdiv(rows, e.alpha.numel())
    return x, wt, e


def _launch_conv(x, wt, e, kernel, conv_2cta=1, conv_halo=1):
    from opendwm_b200 import ops
    rows = x.shape[0] * (x.shape[1] - kernel[0] + 1) * x.shape[2] * x.shape[3]
    c_out = wt.shape[1]
    buf = sentinel_buffer(rows, c_out, x.dtype if e.out16 else torch.float32)
    with _Options(conv_2cta=conv_2cta, conv_halo=conv_halo):
        ops.conv(x, wt, e.bias, kernel=kernel, epilogue=e.kind, act=e.act,
                 out=buf[GUARD:GUARD + rows, :c_out], resid=e.resid,
                 resid_rows_per_item=e.rows_per_item if e.resid_row_mod < 0 else 0,
                 blend_x=e.blend_x, alpha=e.alpha, rows_per_batch=e.rows_per_batch)
        torch.cuda.synchronize()
    return buf


def conv_reference_inputs(x, wt, kernel):
    """float64 (z, P) as [pixels, c_out] for x [nb, tp, h, w, c_in], wt [taps, c_out, c_in]."""
    kt, kh, kw = kernel
    _, c_out, c_in = wt.shape
    X = x.double().permute(0, 4, 1, 2, 3)
    Wt = wt.double().view(kt, kh, kw, c_out, c_in).permute(3, 4, 0, 1, 2)
    f = lambda a, b: torch.nn.functional.conv3d(a, b, padding=(0, kh // 2, kw // 2)).permute(  # noqa: E731
        0, 2, 3, 4, 1).reshape(-1, c_out)
    return f(X, Wt), f(X.abs(), Wt.abs())


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,shape,label", CONV_CASES,
                         ids=["%s_%s" % (c[0], c[2]) for c in CONV_CASES])
def test_conv_conforms(name, shape, label, dtype):
    """`label` is the kernel (C_out tile, CTAs per cluster, halo rows) the default options reach
    on an H100.  Every other variant the options reach runs too: the per-tap kernels (1-CTA and
    pair) must give the same bits, the halo-row kernel is held to the bound."""
    nb, t_out, h, w, c_in, c_out, kernel, _ = shape
    sms = _sms()
    k0 = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms)
    if sms == H100_SMS:
        assert _label(k0) == label
    x, wt, e = _conv_inputs(shape, dtype)
    z, P = conv_reference_inputs(x, wt, kernel)
    K = kernel[0] * kernel[1] * kernel[2] * c_in
    ref, tol = epilogue_reference(z, P, K, e, dtype if e.out16 else torch.float32)
    rows = torch.arange(z.shape[0])
    outs = {}
    for two in (1, 0):
        for halo in (1, 0):
            k = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms, two, halo)
            if k not in outs:
                outs[k] = _launch_conv(x, wt, e, kernel, two, halo)
    assert torch.equal(_bits(_launch_conv(x, wt, e, kernel)), _bits(outs[k0])), \
        "the repeated call gave other bits"
    per_tap = [b for k, b in outs.items() if not k[2]]
    for b in per_tap[1:]:
        assert torch.equal(_bits(b), _bits(per_tap[0])), "1-CTA and pair kernels gave other bits"
    for k, b in outs.items():
        worst = check_output(b, rows, c_out, ref, tol, "%s (%s)" % (name, _label(k)))
        _record("conv_halo" if k[2] else "conv", "%s_%s_%s" % (name, _label(k), dtype), worst)


# --------------------------------------------------------------------------------------------
# which kernel ran
# --------------------------------------------------------------------------------------------
def _launched(fn, types=False, epi=False):
    """Template arguments of every gemm / conv wgmma kernel `fn` launches, in order; with `epi`,
    each gemm entry also carries its EPI template argument; with `types`, each entry ends with
    the operand and 16-bit output type names (TA, T)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    found = []
    for ev in prof.events():
        m = re.search(r"(gemm|conv)_wgmma_kernel<(.*)>", ev.name)
        if not m:
            continue
        args = [re.sub(r"^\((int|bool)\)", "", s.strip()) for s in m.group(2).split(",")]
        if m.group(1) == "gemm":
            k = (int(args[3]), int(args[4])) + ((int(args[2]),) if epi else ())
        else:
            k = (int(args[3]), int(args[4]), args[5] in ("true", "1"))
        found.append(k + tuple(a.split("::")[-1] for a in args[:2]) if types else k)
    return found


def run_isolated(module, func):
    """Runs module.func() (a check built on _launched) in a fresh Python process and fails with
    its output if it fails.  The profiler loses kernels in a process with a history: on an H100
    (torch 2.11, CUDA 12.8) a kernel launched in a profile went unrecorded once a CUDA graph had
    been captured since the process's first profile, or, with CUPTI kept up between profiles,
    once 20 s had passed.  A fresh process profiles only this check's own launches."""
    code = "import sys; sys.path[:0] = %r; import %s as m; m.%s()" % (sys.path, module, func)
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, "%s.%s failed:\n%s\n%s" % (module, func, r.stdout[-3000:], r.stderr[-6000:])


def _selection_shapes(sms):
    """Linear (M, N, kind) and conv (nb, t_out, h, w, c_out, kernel) shapes on both sides of each
    threshold: M = 512 for pairs; a shape whose 128-wide tiles save a tenth of the waves and one
    where they do not; C_out 32 / 96 / 320 / 384 / 512; the halo rule's kw, W and segment count;
    the conv pair rule's 2 x SMs pixel tiles.  Then the text encoders' 16-bit-only linears
    (M, N, kind, act): QuickGELU on both sides of the M = 512 and NT128 / NT256 thresholds
    (CLIP-L's fc1 for 12 prompts is the NT256_CL2 one), and GEGLU_TANH on both sides of M = 512."""
    lin = [(511, 288, STORE), (512, 288, STORE), (4096, 1536, RESID), (2048, 1536, RESID),
           (2048, 1536, GEGLU), (513, 6144, F32), (1, 64, QKNORM)]
    conv = [(1, 1, 4, 14, c, (1, 3, 3)) for c in (32, 96, 320, 384, 512)]
    conv += [(1, 1, sms - 1, 128, 128, (1, 3, 3)), (1, 1, sms, 128, 128, (1, 3, 3)),
             (1, 1, sms, 127, 128, (1, 3, 3)), (1, 1, sms, 128, 128, (1, 1, 1)),
             (1, 1, 2 * sms - 1, 128, 128, (1, 1, 1)), (1, 1, 2 * sms, 128, 128, (1, 1, 1)),
             (1, 1, 2 * sms, 128, 256, (1, 3, 3)), (1, 1, sms, 128, 32, (1, 3, 3)),
             (1, 1, cdiv(sms, 5), 128, 320, (1, 3, 3))]
    text = [(511, 288, STORE, QUICK_GELU), (512, 288, STORE, QUICK_GELU),
            (511, 6144, STORE, QUICK_GELU), (924, 3072, STORE, QUICK_GELU),
            (511, 512, GEGLU_TANH, NONE), (512, 512, GEGLU_TANH, NONE)]
    return lin, conv, text


@pytest.mark.gpu
def test_kernel_selection():
    """check_kernel_selection, in a process of its own (run_isolated)."""
    run_isolated("test_gemm_conformance_gpu", "check_kernel_selection")


def _epi_arg(kind, act):
    """The EPI template argument dwm_b200_linear instantiates for (epilogue, act)."""
    return EPI_STORE_QUICK_GELU if kind == STORE and act == QUICK_GELU else kind


def check_kernel_selection():
    """The launched kernel's template arguments (NT, CL, EPI; CBN, CL, HALO) are the ones
    linear_kernel / conv_kernel / _epi_arg predict, on both sides of each threshold, for every
    option setting the conformance cases use; and every kernel named in a case label is among
    them.  QuickGELU must reach its own instantiation (EPI 16): the generic STORE kernel's
    run-time activation switch has no QuickGELU branch."""
    from opendwm_b200 import ops
    sms = _sms()
    lin, conv, text = _selection_shapes(sms)
    seen = set()
    seen_text = set()
    for M, N, kind, act in text:
        for dt in (torch.bfloat16, torch.float16):
            a = torch.randn(M, 64, device="cuda").to(dt)
            w = torch.randn(N, 64, device="cuda").to(dt)
            for two in (1, 0):
                for bn in (0, 128, 256):
                    want = linear_kernel(M, N, kind, sms, two, bn) + (_epi_arg(kind, act),)
                    with _Options(gemm_2cta=two, gemm_bn=bn):
                        got = _launched(lambda: ops.linear(a, w, epilogue=kind, act=act), epi=True)
                    assert got == [want], ((M, N, kind, act, dt, two, bn), got, want)
                    seen_text.add((_label(want[:2]), want[2], dt))
                    seen.add(_label(want[:2]))
    for dt in (torch.bfloat16, torch.float16):
        want = {("NT%d_CL%d" % (nt, cl), EPI_STORE_QUICK_GELU, dt) for nt in (128, 256) for cl in (1, 2)}
        want |= {("NT256_CL%d" % cl, GEGLU_TANH, dt) for cl in (1, 2)}
        assert want <= seen_text, want - seen_text
    if sms == H100_SMS:
        named = {(c[2], _epi_arg(c[1][3], c[1][4].get("act", NONE)), dt) for c in LINEAR_CASES
                 for dt in (torch.bfloat16, torch.float16)
                 if c[1][3] == GEGLU_TANH or c[1][4].get("act") == QUICK_GELU}
        assert named <= seen_text, named - seen_text
    for M, N, kind in lin:
        a = torch.randn(M, 64, device="cuda").bfloat16()
        w = torch.randn(N, 64, device="cuda").bfloat16()
        kw = {}
        if kind == RESID:
            kw = dict(resid=torch.zeros(M, N, device="cuda"))
        elif kind == QKNORM:
            kw = dict(q_norm_weight=torch.ones(64, device="cuda"), qk_region=N, qk_norm_regions=1)
        for two in (1, 0):
            for bn in (0, 128, 256):
                want = linear_kernel(M, N, kind, sms, two, bn)
                with _Options(gemm_2cta=two, gemm_bn=bn):
                    got = _launched(lambda: ops.linear(a, w, epilogue=kind, **kw), epi=True)
                assert got == [want + (kind,)], ((M, N, kind, two, bn), got, want)
                seen.add(_label(want))
    for nb, t_out, h, w_, c_out, kernel in conv:
        x = torch.randn(nb, t_out + kernel[0] - 1, h, w_, 64, device="cuda").bfloat16()
        wt = torch.randn(kernel[0] * kernel[1] * kernel[2], c_out, 64, device="cuda").bfloat16()
        for two in (1, 0):
            for halo in (1, 0):
                want = conv_kernel(nb, t_out, h, w_, c_out, kernel[2], sms, two, halo)
                with _Options(conv_2cta=two, conv_halo=halo):
                    got = _launched(lambda: ops.conv(x, wt, kernel=kernel))
                assert got == [want], ((nb, t_out, h, w_, c_out, kernel, two, halo), got, want)
                seen.add(_label(want))
    if sms == H100_SMS:
        named = {c[2] for c in LINEAR_CASES + CONV_CASES}
        assert named <= seen, named - seen


# --------------------------------------------------------------------------------------------
# argument checks that keep short or misaligned operands from reaching the device
# --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ops_rejects_short_operands():
    """ops.linear / ops.conv refuse every operand shorter than the rows and columns the epilogue
    addresses, before anything is launched."""
    from opendwm_b200 import ops
    dev = "cuda"
    a = torch.zeros(256, 64, device=dev, dtype=torch.bfloat16)
    w = torch.zeros(96, 64, device=dev, dtype=torch.bfloat16)
    f = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
    bad = [
        dict(bias=f(95)),
        dict(out=torch.zeros(255, 96, device=dev, dtype=torch.bfloat16)),
        dict(out=torch.zeros(260, 96, device=dev, dtype=torch.bfloat16), out_row_offset=5),
        dict(out=torch.zeros(295, 96, device=dev, dtype=torch.bfloat16), rows_per_item=100,
             out_item_stride=120),       # the last item writes rows 240 ... 295
        dict(out=torch.zeros(400, 96, device=dev, dtype=torch.bfloat16), rows_per_item=100,
             out_item_stride=99),
        dict(epilogue=lib.EPI_RESID, resid=f(255, 96)),
        dict(epilogue=lib.EPI_RESID, resid=f(256, 95)),
        dict(epilogue=lib.EPI_RESID, resid=f(49, 96), resid_row_mod=50),
        dict(epilogue=lib.EPI_RESID, resid=f(2, 96), resid_row_mod=-1, rows_per_item=100),
        dict(epilogue=lib.EPI_RESID, resid=f(256, 96), gate=f(2, 96), rows_per_item=100),
        dict(epilogue=lib.EPI_RESID, resid=f(256, 96), blend_x=f(255, 96), alpha=f(1)),
        dict(epilogue=lib.EPI_RESID, resid=f(256, 96), blend_x=f(256, 96), alpha=f(2),
             rows_per_batch=80),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            ops.linear(a, w, **kw)
    x = torch.zeros(2, 1, 4, 14, 64, device=dev, dtype=torch.bfloat16)
    wt = torch.zeros(9, 96, 64, device=dev, dtype=torch.bfloat16)
    rows = 2 * 4 * 14
    with pytest.raises(TypeError):
        ops.conv(x, wt, kernel=(1, 3, 3), out=f(rows, 64))
    for kw in (dict(bias=f(64)),
               dict(epilogue=lib.EPI_RESID, resid=f(rows - 1, 96)),
               dict(epilogue=lib.EPI_RESID, resid=f(1, 96), resid_rows_per_item=56),
               dict(epilogue=lib.EPI_RESID, resid=f(rows, 96), blend_x=f(rows, 95), alpha=f(1)),
               dict(epilogue=lib.EPI_RESID, resid=f(rows, 96), blend_x=f(rows, 96), alpha=f(1),
                    rows_per_batch=56)):
        with pytest.raises(ValueError):
            ops.conv(x, wt, kernel=(1, 3, 3), **kw)


@pytest.mark.gpu
def test_conv_store_with_resid_raises():
    """A 16-bit conv store given a per-item residual used to write every item onto the first
    item's rows (rows_per_item remapped the store); it is refused now."""
    from opendwm_b200 import ops
    x = torch.randn(3, 1, 4, 14, 64, device="cuda").bfloat16()
    wt = torch.randn(9, 64, 64, device="cuda").bfloat16()
    with pytest.raises((ValueError, RuntimeError)):
        ops.conv(x, wt, kernel=(1, 3, 3), epilogue=lib.EPI_STORE, resid=torch.zeros(3, 64, device="cuda"),
                 resid_rows_per_item=56)


@pytest.mark.gpu
def test_text_epilogue_refusals():
    """QuickGELU exists only as a STORE epilogue and GEGLU_TANH needs the 256-column packing;
    both are compiled for 16-bit operands only, so E4M3 operands are refused with either."""
    from opendwm_b200 import ops
    a = torch.zeros(64, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(256, 64, device="cuda", dtype=torch.bfloat16)
    for epi in (F32, RESID, GEGLU, QKNORM):
        with pytest.raises(RuntimeError, match="QUICK_GELU needs the DWM_EPI_STORE"):
            kw = dict(resid=torch.zeros(64, 256, device="cuda")) if epi == RESID else {}
            if epi == QKNORM:
                kw = dict(q_norm_weight=torch.ones(64, device="cuda"), qk_region=256, qk_norm_regions=1)
            ops.linear(a, w, act=QUICK_GELU, epilogue=epi, **kw)
    for n in (128, 384):
        with pytest.raises(RuntimeError, match="GEGLU needs N"):
            ops.linear(a, torch.zeros(n, 64, device="cuda", dtype=torch.bfloat16), epilogue=GEGLU_TANH)
    f8 = torch.float8_e4m3fn
    sc = dict(a_scale=torch.ones(64, device="cuda"), w_scale=torch.ones(256, device="cuda"))
    for kw in (dict(act=QUICK_GELU), dict(epilogue=GEGLU_TANH)):
        for od in (torch.bfloat16, torch.float16):
            with pytest.raises(RuntimeError, match="need 16-bit operands"):
                ops.linear(a.to(f8), w.to(f8), out_dtype=od, **sc, **kw)


def test_pack_geglu_matches_geglu_columns():
    """ops.pack_geglu puts value row j and gate row j of cat([value, gate]) at the accumulator
    columns geglu_columns(2F) gives output column j (the layout the references assume), with
    the bias packed alike; T5 packs cat([wi_1, wi_0]) that way."""
    from opendwm_b200 import ops
    F = 384
    w = torch.arange(2 * F, dtype=torch.float32)[:, None].repeat(1, 8)
    b = torch.arange(2 * F, dtype=torch.float32) + 0.5
    wp, bp = ops.pack_geglu(w, b)
    vc, gc = geglu_columns(2 * F)
    assert torch.equal(wp[vc], w[:F]) and torch.equal(wp[gc], w[F:])
    assert torch.equal(bp[vc], b[:F]) and torch.equal(bp[gc], b[F:])
