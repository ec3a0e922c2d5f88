"""Element-wise conformance of the E4M3 paths of the wgmma GEMM (dwm_b200_linear) and the
implicit-GEMM convolution (dwm_b200_conv) against float64, at the tile, remap and layout edges.

Hopper's FP8 accumulator is not documented (it keeps fewer bits than an fp32 add), so a bound
on its error for random data is either a measured guess or too loose to catch a dropped
k-block.  This suite takes the accumulator out of the question instead: every operand is a
small integer times a power of two, A8[m, k] = i 2^e[m] and W8[n, k] = j 2^f[n] with
|i|, |j| <= 8, and each output's budget sum_k |i j| is at most 2^11 (asserted when the operands
are built).  Every partial sum, in any order and any blocking, is then an integer multiple of
2^(e + f) below 2^11 of them: exact in any accumulator that keeps 12 significant bits, and in
fp32.  test_small_integer_accumulation_is_exact checks that premise first, bit for bit.  So:

  * the accumulator equals z / (sa sw) exactly, z the float64 product of the dequantized
    operands; the kernel's dequantization v = fl(acc fl(sa sw)) (dequant_frag) is within
    (2 U32 + U32^2) |z| of z, and the epilogue's steps after it are bounded as in
    test_gemm_conformance_gpu (epilogue_reference with acc_err);
  * every kernel variant the options reach must give the same bits, the halo-row convolution
    (another tap order) included.

The exponents cycle through -9 ... 6: rows at -9 sit in E4M3 subnormals, rows at 6 reach 448.
The scales spread like row_scales (1, big, 1e-3) times a factor that is not a power of two, so
fl(sa sw) rounds and a scale taken from the wrong row or column fails the bound.  Operand
padding holds the NaN bytes 0x7F / 0xFF, scales past M / N NaN / +-Inf; outputs are checked in
sentinel-filled buffers as in the 16-bit suite.

The CPU self-test checks the bound against an emulated FP8 kernel and eight wrong ones.

The premise probe is bit-exact on an H100 80GB HBM3.  Worst ratio |out - ref| / tol over this
file's cases, measured on that card at a 700 W power limit (bf16 / fp16 outputs): linear 16-bit
outputs 0.996 / 0.999 (the output rounding alone), F32 0.097 / 0.097, RESID 0.963 / 0.963;
convolution 0.133.  The fp32-output ratios sit low because the bound's floor, 2^-20 of
sum |a w|, exceeds the scale product's rounding.
"""
import math

import pytest
import torch

from test_gemm_conformance_gpu import (
    F32, GEGLU, GELU_ERF, GELU_TANH, GUARD, H100_SMS, NONE, QKNORM, RELU, RESID, SILU, STORE, U32,
    Epi, _bits, _label, _launched, _Options, _record, _selection_shapes, _sms, big_scale,
    bound_violations, cdiv, check_output, conv_kernel, emulate_epilogue, epilogue_reference,
    in_nan_block, linear_kernel, padded_vec, pitched, poisoned_2d, row_scales, run_isolated,
    sentinel_buffer)

F8 = torch.float8_e4m3fn
BUDGET = 2 ** 11         # largest sum_k |i j| of an output, in units of 2^(e + f)
TARGET = 2 ** 9          # mean budget the density aims at
MEAN_MAG = 4.5           # mean |i| of a nonzero integer uniform in 1 ... 8
E_MIN = -9               # exponents cycle through E_MIN ... E_MIN + 15 = 6
C_A, C_W = 1.2345679, 0.8765432   # scale factors that are not powers of two
NORM = 1.0 / (8 * 8 * math.sqrt(TARGET))   # |z| ~ row scales: |i j| / 64 over ~ sqrt(TARGET) terms
LD_PAD8 = 16             # poisoned E4M3 columns after K (lda, ldw multiples of 16)
K_MMA = 32               # K of one E4M3 wgmma
SCALE_ERR = 2 * U32 + U32 ** 2   # fl(acc fl(sa sw)) against acc sa sw, acc exact


def exponents(n, shift):
    """Power-of-two exponent of each of n rows / channels: -9 ... 6 in turn."""
    return (torch.arange(n) * 7 + shift) % 16 + E_MIN


def densities(k, n_last):
    """Probability that an element is nonzero: the budget's mean stays near TARGET whatever the
    K (k products per output), and the last n_last positions (the last k32 MMA, the last 16
    input channels of a tap) keep enough nonzero products that dropping them is seen."""
    d = min(0.9, math.sqrt(TARGET / (k * MEAN_MAG ** 2)))
    return d, max(d, min(0.5, math.sqrt(2 ** 7 / (n_last * MEAN_MAG ** 2))))


def integers(g, shape, density, cap):
    """float64 integers in [-cap, cap], nonzero with probability `density` (broadcast over the
    last dimension), magnitudes uniform in 1 ... cap (cap broadcast over the first one)."""
    mag = (torch.rand(shape, generator=g, dtype=torch.float64) * cap).floor() + 1
    nz = torch.rand(shape, generator=g, dtype=torch.float64) < density
    sign = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    return mag * sign * nz


def row_caps(exps, dims):
    """8, but 7 where the exponent is -9 (the row stays subnormal) or 6 (8 x 2^6 overflows)."""
    cap = torch.where((exps == E_MIN) | (exps == E_MIN + 15), 7.0, 8.0).double()
    return cap.view(-1, *[1] * (dims - 1))


def to_e4m3(ints, exps):
    """E4M3 tensor of ints * 2^exps (exps per leading index); asserts every code is exact."""
    v = ints * torch.exp2(exps.double()).view(-1, *[1] * (ints.dim() - 1))
    q = v.to(F8)
    assert torch.equal(q.double(), v), "an operand is not an exact E4M3 code"
    return q


# --------------------------------------------------------------------------------------------
# exactly-accumulating operands
# --------------------------------------------------------------------------------------------
class LinearOperands:
    """E4M3 A8 [M, K] = I 2^e[m], W8 [N, K] = J 2^f[n] with a_scale [M] and w_scale [N].

    A8 rows 0 / 1 and W8 rows 0 / 1 share 32 nonzero columns (all K if K < 32) of +-8, with
    equal signs, and +-7 at one of them in row 1: their sums are 2^11, 2040 and 2033 (11
    significant bits) at K >= 32.  `unit_scales` gives a_scale = w_scale = 1."""

    def __init__(self, M, N, K, big, seed, unit_scales=False):
        g = torch.Generator().manual_seed(seed)
        self.M, self.N, self.K = M, N, K
        self.k_last = K_MMA * ((K - 1) // K_MMA)          # first column of the last k32 MMA
        d, d_last = densities(K, K - self.k_last)
        dens = torch.full((K,), d, dtype=torch.float64)
        dens[self.k_last:] = d_last
        self.e, self.f = exponents(M, 0), exponents(N, 3)
        self.I = integers(g, (M, K), dens, row_caps(self.e, 2))
        self.J = integers(g, (N, K), dens, row_caps(self.f, 2))
        cols = torch.randperm(K, generator=g)[:32]
        signs = torch.randint(0, 2, (cols.numel(),), generator=g).double() * 2 - 1
        for I, n in ((self.I, M), (self.J, N)):
            for r in range(min(2, n)):
                I[r] = 0
                I[r, cols] = 8 * signs
            if n > 1:
                I[1, cols[0]] = 7 * signs[0]
        self.budget = self.I.abs() @ self.J.abs().T             # exact: small integers
        assert self.budget.max() <= BUDGET, (M, N, K, self.budget.max().item())
        self.U = self.I @ self.J.T                               # exact integer sums
        self.a8, self.w8 = to_e4m3(self.I, self.e), to_e4m3(self.J, self.f)
        if unit_scales:
            self.sa, self.sw = torch.ones(M), torch.ones(N)
        else:
            self.sa = (C_A * row_scales(M, big).double() * torch.exp2(-self.e.double()) / 8).float()
            self.sw = (C_W * row_scales(N, big).double() * torch.exp2(-self.f.double()) * 8 * NORM).float()
            s = self.sa.double()[:, None] * self.sw.double()[None, :]
            assert (s != s.float().double()).double().mean() > 0.5, "fl(sa sw) should round"
        # float64 dequantized row factors 2^e sa, 2^f sw (exact), and z, P from the integer sums
        ra = torch.exp2(self.e.double()) * self.sa.double()
        rw = torch.exp2(self.f.double()) * self.sw.double()
        self.z = self.U * ra[:, None] * rw[None, :]
        self.P = self.budget * ra[:, None] * rw[None, :]

    @property
    def acc_err(self):
        return SCALE_ERR * self.z.abs()

    def cuda(self):
        """(A8, W8, a_scale, w_scale) on the GPU inside poisoned allocations."""
        return (poisoned_2d(self.a8, LD_PAD8), poisoned_2d(self.w8, LD_PAD8),
                padded_vec(self.sa), padded_vec(self.sw))


VOL_EXP = (-20, 20, 0, 9, -9, 4)   # 2^p: dequantized magnitude of volume n


class ConvOperands:
    """E4M3 x [nb, tp, h, w, c_in] with volume n = I 2^e[n], weight [taps, c_out, c_in] with
    output channel c = J 2^f[c]; a_scale [nb] puts volume n at about 2^VOL_EXP[n], w_scale
    [c_out] spreads like row_scales.  The budget runs over taps x C_in, zero padding included."""

    def __init__(self, nb, tp, h, w, c_in, c_out, kernel, seed):
        g = torch.Generator().manual_seed(seed)
        kt, kh, kw = kernel
        self.kernel, self.nb, self.c_in, self.c_out = kernel, nb, c_in, c_out
        taps = kt * kh * kw
        d, d_last = densities(taps * c_in, taps * 16)
        dens = torch.full((c_in,), d, dtype=torch.float64)
        dens[c_in - 16:] = d_last
        self.e, self.f = exponents(nb, 5), exponents(c_out, 3)
        self.I = integers(g, (nb, tp, h, w, c_in), dens, row_caps(self.e, 5))
        J = integers(g, (c_out, taps, c_in), dens, row_caps(self.f, 3))
        self.J = J.transpose(0, 1).contiguous()                  # tap-major [taps, c_out, c_in]
        self.budget = self.conv(self.I.abs(), self.J.abs())
        assert self.budget.max() <= BUDGET, (kernel, c_in, c_out, self.budget.max().item())
        self.U = self.conv(self.I, self.J)
        self.x8 = to_e4m3(self.I, self.e)
        self.w8 = to_e4m3(self.J.transpose(0, 1), self.f).transpose(0, 1).contiguous()
        p = torch.tensor(VOL_EXP[:nb], dtype=torch.float64)
        self.sa = (C_A * torch.exp2(p - self.e.double())).float()
        self.sw = (C_W * row_scales(c_out, 1e3).double() * torch.exp2(-self.f.double()) * 8 * NORM).float()
        self.vol = torch.arange(self.U.shape[0]) // (self.U.shape[0] // nb)   # volume of each row
        ra = (torch.exp2(self.e.double()) * self.sa.double())[self.vol]
        rw = torch.exp2(self.f.double()) * self.sw.double()
        self.z = self.U * ra[:, None] * rw[None, :]
        self.P = self.budget * ra[:, None] * rw[None, :]

    def conv(self, x, wt):
        """float64 convolution [pixels, c_out] of x [nb, tp, h, w, c_in], wt [taps, c_out, c_in]
        (exact on these integers)."""
        kt, kh, kw = self.kernel
        X = x.permute(0, 4, 1, 2, 3)
        W = wt.reshape(kt, kh, kw, self.c_out, self.c_in).permute(3, 4, 0, 1, 2)
        y = torch.nn.functional.conv3d(X, W, padding=(0, kh // 2, kw // 2))
        return y.permute(0, 2, 3, 4, 1).reshape(-1, self.c_out)

    @property
    def acc_err(self):
        return SCALE_ERR * self.z.abs()


# --------------------------------------------------------------------------------------------
# emulated FP8 kernel (CPU)
# --------------------------------------------------------------------------------------------
def _e5m2(q):
    return q.view(torch.uint8).view(torch.float8_e5m2).double()


def emulate_linear(op, e, out_dtype, bug=None):
    """The FP8 kernel on the CPU: exact accumulation, v = fl(acc fl(sa sw)), + bias in fp32, then
    the 16-bit suite's fp32 epilogue.  `bug` makes it one of the wrong kernels."""
    a = op.a8.double()
    w = op.w8.double()
    if bug == "last k32 MMA dropped":
        a = a.clone()
        a[:, op.k_last:] = 0
    if bug == "operands decoded as E5M2":
        a, w = _e5m2(op.a8), _e5m2(op.w8)
    acc = (a @ w.T).float()
    sa, sw = op.sa.clone(), op.sw.clone()
    if bug == "a_scale rows r, r + 8 swapped":
        r = torch.arange(op.M)
        lo = r[(r % 16 < 8) & (r + 8 < op.M)]
        sa[lo], sa[lo + 8] = op.sa[lo + 8], op.sa[lo]
    if bug == "w_scale pair swapped":
        sw = sw.view(-1, 2).flip(1).reshape(-1)
    if bug == "a_scale ignored":
        sa = torch.ones_like(sa)
    s = sa[:, None] * sw[None, :]
    b = e.bias.float() if e.bias is not None else torch.zeros(op.N)
    pre = (acc + b) * s if bug == "scale after the bias" else acc * s + b
    return emulate_epilogue(pre, e, out_dtype, bug)


def emulate_conv(op, e, bug=None):
    """The FP8 convolution on the CPU (RESID, fp32 output), as emulate_linear."""
    I = op.I
    if bug == "last 16 input channels dropped":
        I = I.clone()
        I[..., -16:] = 0
    x = I * torch.exp2(op.e.double()).view(-1, 1, 1, 1, 1)
    wt = op.J * torch.exp2(op.f.double()).view(1, -1, 1)
    acc = op.conv(x, wt).float()
    vol = (op.vol + 1) % op.nb if bug == "scale of the next volume" else op.vol
    s = op.sa[vol][:, None] * op.sw[None, :]
    b = e.bias.float() if e.bias is not None else torch.zeros(op.c_out)
    return emulate_epilogue(acc * s + b, e, torch.float32, bug)


# --------------------------------------------------------------------------------------------
# CPU self-test of the bound
# --------------------------------------------------------------------------------------------
LINEAR_BUGS = ["a_scale rows r, r + 8 swapped", "w_scale pair swapped", "scale after the bias",
               "a_scale ignored", "last k32 MMA dropped", "operands decoded as E5M2"]
CONV_BUGS = ["scale of the next volume", "last 16 input channels dropped"]


def _selftest_specs(M):
    g = torch.Generator().manual_seed(11)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    return [
        ("STORE gelu_tanh", 96, Epi(STORE, GELU_TANH, bias=rn(96))),
        ("STORE", 96, Epi(STORE)),
        ("F32 silu", 96, Epi(F32, SILU, bias=rn(96))),
        ("RESID gate", 96, Epi(RESID, bias=rn(96), resid=rn(M, 96), gate=rn(6, 96), rows_per_item=8)),
        ("RESID blend", 96, Epi(RESID, bias=rn(96), resid=rn(M, 96), blend_x=rn(M, 96),
                                alpha=torch.tensor([0.3, 0.8]), rows_per_batch=24)),
        ("QKNORM", 192, Epi(QKNORM, bias=rn(192), qw=rn(64) * 0.2 + 1, kw=rn(64) * 0.2 + 1,
                            qk_region=64)),
        ("GEGLU", 256, Epi(GEGLU, bias=rn(256))),
    ]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_bound_accepts_emulated_kernel_and_rejects_wrong_ones(dtype):
    """Per epilogue (M = 48, K = 144: a ragged last k32 MMA) and for a convolution (C_in = 48,
    three volumes): the emulated FP8 kernel passes the bound, and each wrong kernel fails it
    (the scale-after-bias kernel only where there is a bias)."""
    M, K = 48, 144
    for name, N, e in _selftest_specs(M):
        out_dtype = dtype if e.out16 else torch.float32
        op = LinearOperands(M, N, K, big_scale(dtype, e.out16), seed=N)
        ref, tol = epilogue_reference(op.z, op.P, K, e, out_dtype, acc_err=op.acc_err)
        bad, worst = bound_violations(emulate_linear(op, e, out_dtype), ref, tol)
        assert not bad.any(), (name, worst)
        if e.out16:
            assert worst > 0.05, (name, worst)
        for bug in LINEAR_BUGS:
            if bug == "scale after the bias" and e.bias is None:
                continue
            bad, worst = bound_violations(emulate_linear(op, e, out_dtype, bug), ref, tol)
            assert bad.any(), (name, bug, worst)
    g = torch.Generator().manual_seed(5)
    op = ConvOperands(3, 1, 5, 6, 48, 64, (1, 3, 3), seed=3)
    rows = op.U.shape[0]
    for e in (Epi(RESID, bias=torch.randn(64, generator=g) * 1e-6, resid=op.z.float()),
              Epi(RESID, resid=op.z.float() * 0.5, blend_x=op.z.float() * 0.1,
                  alpha=torch.tensor([0.3, 0.0, 1.0]), rows_per_batch=rows // 3)):
        ref, tol = epilogue_reference(op.z, op.P, 9 * 48, e, torch.float32, acc_err=op.acc_err)
        bad, worst = bound_violations(emulate_conv(op, e), ref, tol)
        assert not bad.any(), worst
        for bug in CONV_BUGS:
            bad, worst = bound_violations(emulate_conv(op, e, bug), ref, tol)
            assert bad.any(), (bug, worst)


def test_operands_are_exact_and_within_budget():
    """The constructors' assertions for every GPU case (budget, exact E4M3 codes, rounding scale
    products), and the reach of the data: subnormal and 448-valued elements, the planted 2^11
    sums, the last k32 MMA nonzero for most outputs."""
    for K in PROBE_K:
        op = LinearOperands(520, 288, K, 1.0, seed=K, unit_scales=True)
        if K >= 32:
            assert op.U[0, 0] == BUDGET and op.U[1, 0] == 2040 and op.U[1, 1] == 2033
        last = op.I[:, op.k_last:] @ op.J[:, op.k_last:].T
        assert (last != 0).double().mean() > 0.75, K
        v = op.a8.double().abs()
        assert (v == 448).any() and ((v > 0) & (v < 2 ** -6)).any()
    for _, (M, N, K, kind, opt), _ in LINEAR_CASES:
        LinearOperands(M, N, K, big_scale(torch.float16, kind in (STORE, GEGLU, QKNORM)), seed=M + N + K)
    for _, shape, _ in CONV_CASES:
        nb, t_out, h, w, c_in, c_out, kernel, _ = shape
        ConvOperands(nb, t_out + kernel[0] - 1, h, w, c_in, c_out, kernel, seed=h * w + c_in)


# --------------------------------------------------------------------------------------------
# the premise: small-integer sums are exact in the FP8 accumulator
# --------------------------------------------------------------------------------------------
PROBE_K = [16, 32, 48, 144, 1552, 6144]


@pytest.mark.gpu
@pytest.mark.parametrize("K", PROBE_K)
def test_small_integer_accumulation_is_exact(K):
    """Unit scales, the F32 epilogue, no bias: the output is the integer sum itself, bit for
    bit, for 1-CTA and pair kernels and 128- and 256-wide tiles (M = 520: five 128-row blocks,
    so the pair runs a dummy tile).  Rows 0 / 1 reach 2^11 at K >= 32."""
    from opendwm_b200 import ops
    op = LinearOperands(520, 288, K, 1.0, seed=K, unit_scales=True)
    A, W, sa, sw = op.cuda()
    want = (op.U * torch.exp2((op.e[:, None] + op.f[None, :]).double())).cuda()
    for two in (1, 0):
        for bn in (128, 256):
            with _Options(gemm_2cta=two, gemm_bn=bn):
                out = ops.linear(A, W, epilogue=F32, a_scale=sa, w_scale=sw, out_dtype=torch.bfloat16)
                torch.cuda.synchronize()
            bad = out.double() != want
            if bad.any():
                U = op.U.cuda()
                raise AssertionError(
                    "K = %d, %s: %d of %d integer sums inexact; smallest inexact |sum| %d units "
                    "(budget %d), largest exact %d" % (
                        K, _label(linear_kernel(520, 288, F32, _sms(), two, bn)), bad.sum(), bad.numel(),
                        U.abs()[bad].min().item(), op.budget.cuda()[bad].min().item(),
                        U.abs()[~bad].max().item()))


# --------------------------------------------------------------------------------------------
# linear cases
# --------------------------------------------------------------------------------------------
def _lin(name, M, N, K, kind, label, **opt):
    return (name, (M, N, K, kind, opt), label)


# the frame-sharded K,V scatter: B = 2 entries of T_loc = 2 local frames of V = 3 views of S = 50
# tokens, rank 1 of frame shards T = 6 (crossview_temporal.sharded_temporal_qkv_attend)
SCATTER = dict(rows_per_item=300, out_item_stride=900, out_row_offset=300)

LINEAR_CASES = [
    # STORE: every activation, M / N / K edges (K = 16, 48, 80: one half-filled k32 MMA)
    _lin("store_M1_N32_K16", 1, 32, 16, STORE, "NT128_CL1"),
    _lin("store_gelu_tanh_M127_N96_K48", 127, 96, 48, STORE, "NT128_CL1", act=GELU_TANH, bias=True),
    _lin("store_gelu_erf_M129_N288_K1552", 129, 288, 1552, STORE, "NT128_CL1", act=GELU_ERF, bias=True),
    _lin("store_silu_M511_N6144_K80", 511, 6144, 80, STORE, "NT256_CL1", act=SILU, bias=True),
    _lin("store_relu_M512_N288_K6144", 512, 288, 6144, STORE, "NT128_CL2", act=RELU, bias=True),
    _lin("store_M513_N6144_K144", 513, 6144, 144, STORE, "NT128_CL2", bias=True),   # odd blocks
    _lin("store_remap_M300_N288_K144", 300, 288, 144, STORE, "NT128_CL1", bias=True,
         rows_per_item=100, out_item_stride=130, out_row_offset=7),
    # F32: rows_per_item / offsets must not remap fp32 outputs
    _lin("f32_gelu_tanh_M513_N288_K1552", 513, 288, 1552, F32, "NT128_CL2", act=GELU_TANH, bias=True),
    _lin("f32_items_M129_N96_K16", 129, 96, 16, F32, "NT128_CL1", bias=True, rows_per_item=50,
         out_row_offset=5),
    # RESID
    _lin("resid_M513_N288_K1552", 513, 288, 1552, RESID, "NT128_CL2", bias=True, resid="full"),
    # the patch embedding's positional rows (resid_row_mod = S = 100) with a gate per item
    _lin("resid_mod_gate_M300_N96_K48", 300, 96, 48, RESID, "NT128_CL1", bias=True, resid="mod",
         resid_mod=100, gate=True, rows_per_item=100),
    _lin("resid_item_M129_N6144_K144", 129, 6144, 144, RESID, "NT128_CL1", bias=True,
         resid="item", rows_per_item=43),
    _lin("resid_blend_gate_M513_N288_K1552", 513, 288, 1552, RESID, "NT128_CL2", bias=True,
         resid="full", gate=True, rows_per_item=57, blend=(0.0, 0.3, 1.0)),
    _lin("resid_inplace_gate_M512_N96_K6144", 512, 96, 6144, RESID, "NT128_CL2", bias=True,
         resid="full", gate=True, rows_per_item=128, inplace="resid"),
    _lin("resid_inplace_blend_M127_N288_K80", 127, 288, 80, RESID, "NT128_CL1", bias=True,
         resid="full", blend=(0.3, 1.0), inplace="blend"),
    _lin("resid_nobias_M1_N32_K16", 1, 32, 16, RESID, "NT128_CL1", resid="full"),
    # GEGLU (always 256 wide)
    _lin("geglu_M513_N512_K1552", 513, 512, 1552, GEGLU, "NT256_CL2", bias=True),
    _lin("geglu_remap_M300_N768_K48", 300, 768, 48, GEGLU, "NT256_CL1", bias=True,
         rows_per_item=100, out_item_stride=110, out_row_offset=3),
    # QKNORM, D = 320: region boundaries inside 256-wide tiles
    _lin("qknorm2_M513_N960_K1552", 513, 960, 1552, QKNORM, "NT128_CL2", bias=True, qk_region=320,
         regions=2),
    _lin("qknorm1_M129_N960_K80", 129, 960, 80, QKNORM, "NT128_CL1", qk_region=320, regions=1),
    # the frame-sharded K,V scatter into out and two peers (D = 192: K normalised, V not)
    _lin("scatter_store_M600_N384_K144", 600, 384, 144, STORE, "NT128_CL2", bias=True, **SCATTER),
    _lin("scatter_qknorm_M600_N384_K80", 600, 384, 80, QKNORM, "NT128_CL2", bias=True,
         qk_region=192, regions=1, **SCATTER),
]


def _linear_case(M, N, K, kind, opt, dtype, seed=None, qk_seed=0):
    """(operands, Epi with CUDA operands) of one case.  Residual, gate and blend rows are scaled
    like the result rows, so that a small row's error does not vanish under a large residual."""
    out16 = kind in (STORE, GEGLU, QKNORM)
    big = big_scale(dtype, out16)
    op = LinearOperands(M, N, K, big, seed=M + N + K if seed is None else seed)
    g = torch.Generator().manual_seed(M + 3 * N + K + qk_seed)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    ra, rw = row_scales(M, big)[:, None], row_scales(N, big)[None, :]
    rpi = opt.get("rows_per_item", 0)
    items = cdiv(M, rpi) if rpi else 1
    e = Epi(kind, act=opt.get("act", NONE), rows_per_item=rpi,
            out_item_stride=opt.get("out_item_stride", 0), out_row_offset=opt.get("out_row_offset", 0))
    if opt.get("bias"):
        e.bias = padded_vec(rn(N) * 0.1 * rw[0])
    if kind == RESID:
        mode = opt.get("resid")
        if mode == "mod":
            e.resid_row_mod = opt["resid_mod"]
            e.resid = pitched(rn(e.resid_row_mod, N) * 0.1 * rw)
        elif mode == "item":
            e.resid_row_mod = -1
            e.resid = pitched(rn(items, N) * 0.1 * rw)
        elif mode == "full":
            e.resid = pitched(rn(M, N) * 0.1 * ra * rw)
        if opt.get("gate"):
            e.gate = pitched(rn(items, N))
        if opt.get("blend"):
            e.blend_x = pitched(rn(M, N) * 0.1 * ra * rw)
            e.alpha = torch.tensor(opt["blend"], dtype=torch.float32).cuda()
            e.rows_per_batch = cdiv(M, len(opt["blend"]))
    if kind == QKNORM:
        e.qw, e.kw = (rn(64) * 0.2 + 1).cuda(), (rn(64) * 0.2 + 1).cuda()
        e.qk_region, e.regions = opt["qk_region"], opt["regions"]
    return op, e


def _reference(op, e, out_dtype):
    return epilogue_reference(op.z.cuda(), op.P.cuda(), op.K, e, out_dtype, acc_err=op.acc_err.cuda())


def _launch_linear(calls, rows, cols, out_dtype, gemm_2cta=1, gemm_bn=0, resid_tma=1):
    """Runs each call (device operands, Epi, opt) into views of the same fresh sentinel buffers;
    returns [out buffer, peer buffers...] (peers for 16-bit outputs)."""
    from opendwm_b200 import ops
    out16 = calls[0][1].out16
    odt = out_dtype if out16 else torch.float32
    bufs = [sentinel_buffer(rows, cols, odt) for _ in range(3 if out16 else 1)]
    view = lambda b: b[GUARD:GUARD + rows, :cols]  # noqa: E731
    out = view(bufs[0])
    with _Options(gemm_2cta=gemm_2cta, gemm_bn=gemm_bn, resid_tma=resid_tma):
        for (A, W, sa, sw), e, opt in calls:
            M, N = A.shape[0], W.shape[0]
            resid, blend_x = e.resid, e.blend_x
            if opt.get("inplace") == "resid":
                out[:M, :N] = resid
                resid = out
            elif opt.get("inplace") == "blend":
                out[:M, :N] = blend_x
                blend_x = out
            ops.linear(A, W, e.bias, epilogue=e.kind, act=e.act, out=out, a_scale=sa, w_scale=sw,
                       out_dtype=out_dtype, rows_per_item=e.rows_per_item,
                       out_item_stride=e.out_item_stride, out_row_offset=e.out_row_offset,
                       q_norm_weight=e.qw, k_norm_weight=e.kw, qk_region=e.qk_region, eps=e.eps,
                       qk_norm_regions=e.regions if e.kind == QKNORM else 0,
                       peer_out=[view(b).data_ptr() for b in bufs[1:]] or None,
                       resid=resid, resid_row_mod=e.resid_row_mod, gate=e.gate, blend_x=blend_x,
                       alpha=e.alpha, rows_per_batch=e.rows_per_batch)
        torch.cuda.synchronize()
    return bufs


def _run_variants(calls, rows, cols, dtype, kinds, what):
    """The default call, checked for peers and repeatability, then every other (gemm_2cta,
    gemm_bn) the options reach (and resid_tma = 0 for RESID): all must give the same bits.
    `kinds` are the (M, N, kind) of the calls.  Returns the default call's buffers."""
    sms = _sms()
    b0 = _launch_linear(calls, rows, cols, dtype)
    for i, p in enumerate(b0[1:]):
        assert torch.equal(_bits(p), _bits(b0[0])), "%s: peer_out[%d] differs from out" % (what, i)
    same = lambda bufs: all(torch.equal(_bits(x), _bits(y)) for x, y in zip(bufs, b0))  # noqa: E731
    assert same(_launch_linear(calls, rows, cols, dtype)), "%s: the repeated call gave other bits" % what
    key = lambda two, bn: tuple(linear_kernel(M, N, k, sms, two, bn) for M, N, k in kinds)  # noqa: E731
    seen = {key(1, 0)}
    for two in (1, 0):
        for bn in (128, 256):
            k = key(two, bn)
            if k not in seen:
                seen.add(k)
                assert same(_launch_linear(calls, rows, cols, dtype, two, bn)), \
                    "%s: %s gave other bits than the default" % (what, [_label(x) for x in k])
    if kinds[0][2] == RESID:
        assert same(_launch_linear(calls, rows, cols, dtype, resid_tma=0)), \
            "%s: resid_tma = 0 gave other bits" % what
    return b0


DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,shape,label", LINEAR_CASES,
                         ids=["%s_%s" % (c[0], c[2]) for c in LINEAR_CASES])
def test_fp8_linear_conforms(name, shape, label, dtype):
    """`label` is the kernel (tile width, CTAs per cluster) the default options reach on an H100;
    `dtype` is out_dtype, the type of the 16-bit outputs."""
    M, N, K, kind, opt = shape
    sms = _sms()
    if sms == H100_SMS:
        assert _label(linear_kernel(M, N, kind, sms)) == label
    op, e = _linear_case(M, N, K, kind, opt, dtype)
    odt = dtype if e.out16 else torch.float32
    ref, tol = _reference(op, e, odt)
    rows = int(e.out_rows(M).max()) + 1
    b0 = _run_variants([(op.cuda(), e, opt)], rows, e.out_cols(N), dtype, [(M, N, kind)], name)
    worst = check_output(b0[0], e.out_rows(M), e.out_cols(N), ref, tol, name)
    _record("fp8_linear_resid" if kind == RESID else "fp8_linear", "%s_%s" % (name, dtype), worst)


@pytest.mark.gpu
@DTYPES
def test_fp8_qknorm_joint_buffer(dtype):
    """The DiT's joint q|k|v buffer: the sample projection (items of S = 100 rows) and the
    context projection (L = 30 rows) write one 390-row buffer with out_item_stride = 130, each
    with its own weights and norm weights; the two calls are checked as one write set."""
    D, K = 320, 80
    parts = []
    for M, rpi, off in ((300, 100, 0), (90, 30, 100)):
        opt = dict(bias=True, qk_region=D, regions=2, rows_per_item=rpi, out_item_stride=130,
                   out_row_offset=off)
        op, e = _linear_case(M, 3 * D, K, QKNORM, opt, dtype, seed=M + 1, qk_seed=M)
        parts.append((op, e, opt))
    refs = [_reference(op, e, dtype) for op, e, _ in parts]
    b0 = _run_variants([(op.cuda(), e, opt) for op, e, opt in parts], 390, 3 * D, dtype,
                       [(op.M, 3 * D, QKNORM) for op, _, _ in parts], "joint q|k|v")
    worst = check_output(b0[0], torch.cat([e.out_rows(op.M) for op, e, _ in parts]), 3 * D,
                         torch.cat([r for r, _ in refs]), torch.cat([t for _, t in refs]), "joint q|k|v")
    _record("fp8_linear", "qknorm_joint_%s" % dtype, worst)


# --------------------------------------------------------------------------------------------
# convolution cases (RESID only in E4M3)
# --------------------------------------------------------------------------------------------
def _cv(name, nb, t_out, h, w, c_in, c_out, kernel, resid, label):
    return (name, (nb, t_out, h, w, c_in, c_out, kernel, resid), label)


CONV_CASES = [
    _cv("w14_h9_k133_cin16_cout32_full", 3, 1, 9, 14, 16, 32, (1, 3, 3), "full", "NT32_CL1"),
    _cv("w56_h5_k311_cin48_cout320_item", 4, 2, 5, 56, 48, 320, (3, 1, 1), "item", "NT64_CL1"),
    _cv("w3_h5_k333_cin144_cout96_blend", 3, 2, 5, 3, 144, 96, (3, 3, 3), "blend", "NT32_CL1"),
    _cv("w128_h48_k133_cin48_cout384_none_halo", 1, 1, 48, 128, 48, 384, (1, 3, 3), "none",
        "NT128_CL1_HALO"),
    _cv("w129_h40_k133_cin16_cout320_full_halo", 1, 1, 40, 129, 16, 320, (1, 3, 3), "full",
        "NT64_CL1_HALO"),
    _cv("w200_h14_k133_cin144_cout128_blend_self_halo", 2, 3, 14, 200, 144, 128, (1, 3, 3),
        "blend_self", "NT128_CL1_HALO"),
    _cv("w448_h3_k133_cin320_cout32_item_halo", 3, 4, 3, 448, 320, 32, (1, 3, 3), "item",
        "NT32_CL1_HALO"),
    _cv("w56_h5_k311_cin48_cout512_blend_self_pair_odd", 5, 9, 5, 56, 48, 512, (3, 1, 1),
        "blend_self", "NT256_CL2"),
    _cv("w56_h5_k311_cin1280_cout96_full", 3, 1, 5, 56, 1280, 96, (3, 1, 1), "full", "NT32_CL1"),
    _cv("w40_h8_k133_cin320_cout320_item", 3, 1, 8, 40, 320, 320, (1, 3, 3), "item", "NT64_CL1"),
]


def _conv_case(shape):
    """(operands, Epi with CUDA operands): residual and blend rows scaled like their volume's
    results, a bias at the smallest volume's magnitude."""
    nb, t_out, h, w, c_in, c_out, kernel, mode = shape
    op = ConvOperands(nb, t_out + kernel[0] - 1, h, w, c_in, c_out, kernel, seed=h * w + c_in)
    rows = op.U.shape[0]
    g = torch.Generator().manual_seed(rows + c_out)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    vol = torch.exp2(torch.tensor(VOL_EXP[:nb], dtype=torch.float32))
    rw = row_scales(c_out, 1e3)[None, :] * 0.1
    e = Epi(RESID, bias=padded_vec(rn(c_out) * rw[0] * vol.min()))
    if mode == "item":
        e.resid_row_mod, e.rows_per_item = -1, h * w
        e.resid = pitched(rn(nb * t_out, c_out) * rw * vol.repeat_interleave(t_out)[:, None])
    elif mode != "none":
        e.resid = pitched(rn(rows, c_out) * rw * vol[op.vol][:, None])
        if mode.startswith("blend"):
            e.blend_x = e.resid if mode == "blend_self" else pitched(rn(rows, c_out) * rw * vol[op.vol][:, None])
            e.alpha = torch.tensor([0.3, 0.0, 1.0][:nb * t_out]).cuda()
            e.rows_per_batch = cdiv(rows, e.alpha.numel())
    return op, e


def _launch_conv(op, dev, e, conv_2cta=1, conv_halo=1):
    from opendwm_b200 import ops
    x, wt, sa, sw = dev
    rows = op.U.shape[0]
    buf = sentinel_buffer(rows, op.c_out, torch.float32)
    with _Options(conv_2cta=conv_2cta, conv_halo=conv_halo):
        ops.conv(x, wt, e.bias, kernel=op.kernel, epilogue=RESID, out=buf[GUARD:GUARD + rows, :op.c_out],
                 resid=e.resid, resid_rows_per_item=e.rows_per_item if e.resid_row_mod < 0 else 0,
                 blend_x=e.blend_x, alpha=e.alpha, rows_per_batch=e.rows_per_batch, a_scale=sa, w_scale=sw)
        torch.cuda.synchronize()
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,label", CONV_CASES,
                         ids=["%s_%s" % (c[0], c[2]) for c in CONV_CASES])
def test_fp8_conv_conforms(name, shape, label):
    """`label` is the kernel (C_out tile, CTAs per cluster, halo rows) the default options reach
    on an H100.  Every variant the options reach (1-CTA, pair, halo-row, per-tap) must give the
    same bits: every partial sum is exact in any order."""
    nb, t_out, h, w, c_in, c_out, kernel, _ = shape
    sms = _sms()
    k0 = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms)
    if sms == H100_SMS:
        assert _label(k0) == label
    op, e = _conv_case(shape)
    ref, tol = epilogue_reference(op.z.cuda(), op.P.cuda(), kernel[0] * kernel[1] * kernel[2] * c_in,
                                  e, torch.float32, acc_err=op.acc_err.cuda())
    dev = (in_nan_block(op.x8), in_nan_block(op.w8), padded_vec(op.sa), padded_vec(op.sw))
    outs = {}
    for two in (1, 0):
        for halo in (1, 0):
            k = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms, two, halo)
            if k not in outs:
                outs[k] = _launch_conv(op, dev, e, two, halo)
    assert torch.equal(_bits(_launch_conv(op, dev, e)), _bits(outs[k0])), "the repeated call gave other bits"
    for k, b in outs.items():
        assert torch.equal(_bits(b), _bits(outs[k0])), "%s gave other bits than %s" % (_label(k), label)
    worst = check_output(outs[k0], torch.arange(op.U.shape[0]), c_out, ref, tol, name)
    _record("fp8_conv", "%s_%s" % (name, "+".join(_label(k) for k in outs)), worst)


# --------------------------------------------------------------------------------------------
# which kernel ran
# --------------------------------------------------------------------------------------------
E4M3_T = "__nv_fp8_e4m3"


@pytest.mark.gpu
def test_fp8_kernel_selection():
    """check_fp8_kernel_selection, in a process of its own (run_isolated)."""
    run_isolated("test_fp8_conformance_gpu", "check_fp8_kernel_selection")


def check_fp8_kernel_selection():
    """With E4M3 operands the launched kernel is the one linear_kernel / conv_kernel predict, on
    both sides of each threshold, and its instantiation is the E4M3 one: TA = __nv_fp8_e4m3,
    T = __half for fp16 STORE / GEGLU / QKNORM, __nv_bfloat16 for RESID and F32 whatever the
    out_dtype (one shared instantiation) and for the convolution.  Every kernel named in a case
    label is among them."""
    from opendwm_b200 import ops
    sms = _sms()
    lin, conv, _ = _selection_shapes(sms)   # the text epilogues refuse E4M3 operands
    seen = set()
    for M, N, kind in lin:
        a = torch.randn(M, 64, device="cuda").to(F8)
        w = torch.randn(N, 64, device="cuda").to(F8)
        sc = dict(a_scale=torch.ones(M, device="cuda"), w_scale=torch.ones(N, device="cuda"))
        if kind == RESID:
            sc.update(resid=torch.zeros(M, N, device="cuda"))
        elif kind == QKNORM:
            sc.update(q_norm_weight=torch.ones(64, device="cuda"), qk_region=N, qk_norm_regions=1)
        for od in (torch.bfloat16, torch.float16):
            t = "__half" if od == torch.float16 and kind in (STORE, GEGLU, QKNORM) else "__nv_bfloat16"
            for two in (1, 0):
                for bn in (0, 128, 256):
                    k = linear_kernel(M, N, kind, sms, two, bn)
                    with _Options(gemm_2cta=two, gemm_bn=bn):
                        got = _launched(lambda: ops.linear(a, w, epilogue=kind, out_dtype=od, **sc), types=True)
                    assert got == [k + (E4M3_T, t)], ((M, N, kind, od, two, bn), got, k)
                    seen.add(_label(k))
    for nb, t_out, h, w_, c_out, kernel in conv:
        x = torch.randn(nb, t_out + kernel[0] - 1, h, w_, 64, device="cuda").to(F8)
        wt = torch.randn(kernel[0] * kernel[1] * kernel[2], c_out, 64, device="cuda").to(F8)
        sc = dict(a_scale=torch.ones(nb, device="cuda"), w_scale=torch.ones(c_out, device="cuda"))
        for two in (1, 0):
            for halo in (1, 0):
                k = conv_kernel(nb, t_out, h, w_, c_out, kernel[2], sms, two, halo)
                with _Options(conv_2cta=two, conv_halo=halo):
                    got = _launched(lambda: ops.conv(x, wt, kernel=kernel, epilogue=RESID, **sc), types=True)
                assert got == [k + (E4M3_T, "__nv_bfloat16")], ((nb, t_out, h, w_, c_out, kernel, two, halo), got, k)
                seen.add(_label(k))
    if sms == H100_SMS:
        named = {c[2] for c in LINEAR_CASES + CONV_CASES}
        assert named <= seen, named - seen
