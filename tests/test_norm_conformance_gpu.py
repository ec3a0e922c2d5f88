"""Element-wise conformance of the GroupNorm / SpatialNorm kernels (vae.cu), the LayerNorm / AdaLN
kernels, the RMSNorm of the T5 encoder and the E4M3 row quantizer (rowops.cu) against float64.

Every GPU case writes into a sentinel-filled allocation (guard elements before and after, a row
pitch or frames the call must not touch) and reads inputs whose padding holds NaN / +-Inf.  The
reference is float64 with a two-pass variance; the bound on |out - ref| is derived from the
kernel's arithmetic, each fp32 step rounding by at most U32 = 2^-24 of its result:

  * GroupNorm statistics (`groupnorm_stats`): every float is widened to double before it is
    added or squared (the square of an fp32 value is exact in double), so |sum - ref| <=
    n_g 2^-53 sum|x| and |sumsq - ref| <= n_g 2^-53 sum x^2 for the n_g values of a group (each
    of them takes part in a chain of at most n_g additions).  The three kernels are chosen as
    `stats_kernel` restates from dwm_b200_groupnorm_stats.  The sums use atomics, so their bits
    may change from call to call; no repeat check.
  * GroupNorm apply (`gn_reference`): the kernel finalises mean_d = s / n and var_d =
    max(ss / n - mean_d^2, 0) in double (error E_var <= 3 (n_g + 2) 2^-53 (var + mean^2)), then
    rstd = rsqrtf(float(var_d) + eps) (relative error e_r: the exact effect of E_var on
    (var + eps)^-1/2 plus 5 U32 for the two conversions, the addition and rsqrtf's 2 ulps) and
    mu = float(mean_d) (|mu - mean| <= U32 |mean| + n_g 2^-52 mean|x|).  Per element
    d = x - mu (E_d = |mu - mean| + U32 |d|), y = d * rstd * gamma + beta with two roundings
    of products and one of the sum (fast path: fmaf(d, rstd * gamma, beta); general path:
    ((d * rstd) * gamma) + beta): E_y = |gamma| rstd (E_d + |x - mean| (e_r + 2 U32)) +
    U32 |y|.  SpatialNorm: z = y * zy + zb, E_z = |zy| E_y + U32 (|y zy| + |z|).  SiLU: 1.1 E +
    the error of silu's __expf formula (`act_reference` of the GEMM suite).  A 16-bit output
    adds u |ref| (u = 2^-8 bf16, 2^-11 fp16) and, for fp16, 2^-25 for its subnormals.
  * LayerNorm (`ln_reference`): v = x (+ add_item) (+ add_full) in fp32 is `sum_out`, bit for
    bit; the reference normalises that fp32 row.  mean: fp32 sums of D / 32 values per lane and
    a 5-level shuffle tree, E_mean <= (4 ceil(D / 128) + 7) U32 mean|v|; d = v - mean:
    E_d = E_mean + U32 |d|; var = sum d^2 / D (the mean's error only adds E_mean^2, the cross
    term sums to zero): relative error (4 ceil(D / 128) + 10) U32 + E_mean^2 / var; rstd as
    above.  Each later step (x weight, + bias, x (1 + scale), + shift) adds |factor| E plus
    U32 of its result (and of 1 + scale's rounding).
  * RMSNorm (`rms_reference`): the sum of squares is fp32, per-thread float4 partials over the
    row's D / 4 vectors in steps of 256 threads, a 5-level warp shuffle tree and a sequential
    sum of the 8 warps' partials.  Every term is non-negative, so the sum's relative error is at
    most L U32 with L = 4 + ceil(D / 1024) + 5 + 7 the longest chain of roundings a square takes
    part in; / D and + eps add 2 U32, rsqrtf 2 ulps (4 U32) and halves the rest:
    e_r = (L + 2) U32 / 2 + 4 U32.  out = w (x r), two rounded products: E = (e_r + 2 U32) |ref|.
    An all-zero row must give 0; fp16 results past 65504 must be +-Inf where the bound puts the
    exact value beyond fp16's rounding threshold 65520 (and +-65504 or +-Inf within it).
  * E4M3 outputs (GroupNorm: one scale per volume, LayerNorm: per row): amax is the max of the
    kernel's fp32 values, so |448 scale - amax_ref| <= max E + 2^-23 amax_ref.  Each byte's
    fp32 pre-image v * fl(448 / amax) lies within E_p = 448 (E + |ref| E_max / amax_lo) /
    amax_lo + 3 U32 |p| of p_ref = 448 ref / amax_ref (amax_lo = amax_ref - E_max); rounding
    is monotone, so the byte must lie between e4m3(p_ref - E_p) and e4m3(p_ref + E_p): the
    neighbouring code is accepted exactly where the pre-image may sit across a midpoint.  An
    all-zero volume or row must give scale 1 and zero bytes.
  * `quantize_rows` is bit-exact against tests/fp8_emulation.quantize_rows.

The CPU self-test runs fp32 emulations of the kernels through the same checks and rejects nine
wrong kernels: a one-pass fp32 LayerNorm variance, a GroupNorm group index one channel off for
10-channel groups, t * Tz / T as the frame map for odd T, eps added outside the square root, the
modulation of item + 1, an inverted E4M3 scale, fp32 GroupNorm statistics whose negative
variance is not clamped, and an RMSNorm whose mean runs over D - 4 columns or whose eps sits
outside the rsqrt.

Worst ratio |out - ref| / tol over this file's cases, measured on an H100 80GB HBM3 at a 700 W
power limit (bf16 / fp16): groupnorm_stats 0.078; spatialnorm_silu 0.995 / 0.996;
groupnorm_silu_halo 0.986 / 0.976; layernorm 0.996 / 0.997.  E4M3 scales: groupnorm_silu_e4m3
0.001, the halo variant 0.020, layernorm 0.136 (every byte within its allowed codes).  rmsnorm
(bf16 / fp16 / fp32) 0.996 / 0.997 / 0.268, same card and limit.  The
16-bit maxima sit in the output rounding, which is exact; the statistics use 8 % of a bound that
assumes every rounding of a double chain as long as the group is adds up.  At the parent
revision (fp32 statistics) every groupnorm_stats case missed its bound by 3e2 to 4e7 times, and
every GroupNorm apply case failed on its large-mean groups (NaN on the constant ones).
"""
import math

import pytest
import torch

import fp8_emulation as fe
from test_gemm_conformance_gpu import SILU, U32, act_reference, bound_violations, unit_roundoff

SENT16 = -21555                  # int16 bits of every 16-bit element a call must not write
SENT8 = 0x5A                     # byte of every E4M3 element a call must not write
GUARD = 4096                     # sentinel elements before and after each output
U64 = 2.0 ** -53
FP8 = torch.float8_e4m3fn


# --------------------------------------------------------------------------------------------
# bound helpers
# --------------------------------------------------------------------------------------------
def rstd_rel_error(var, eps, e_var):
    """Relative error of fp32 rsqrtf(float(var_k) + eps) when |var_k - var| <= e_var (var_k >= 0)."""
    v = var + eps
    hi = torch.rsqrt(torch.clamp(v - e_var, min=eps) / v) - 1
    lo = 1 - torch.rsqrt((v + e_var) / v)
    return torch.maximum(hi, lo) + 5 * U32


def out16_tol(err, ref, dtype):
    u = unit_roundoff(dtype)
    sub = 2.0 ** -25 if dtype == torch.float16 else 0.0
    return (1 + u) * err + u * ref.abs() + sub


def e4m3_check(q, scale, ref, err, what):
    """q [R, N] E4M3, scale [R], ref / err float64 [R, N] (fp32 value before quantization and its
    bound).  Returns the worst scale ratio."""
    q, scale, ref, err = q.cpu(), scale.cpu().double(), ref.cpu(), err.cpu()
    amax = ref.abs().amax(1)
    emax = err.amax(1)
    zero = amax == 0
    assert torch.equal(scale[zero], torch.ones_like(scale[zero])), "%s: zero rows need scale 1" % what
    assert not q[zero].view(torch.uint8).any(), "%s: zero rows need zero bytes" % what
    nz = ~zero
    bad, worst = bound_violations(448 * scale[nz], amax[nz], emax[nz] + 2.0 ** -23 * amax[nz])
    assert not bad.any(), "%s: scale outside its bound (worst %.3g)" % (what, worst)
    amax_lo = (amax - emax).clamp_min(1e-30)[:, None]
    p = 448 * ref / amax.clamp_min(1e-30)[:, None]
    e_p = 448 * (err + ref.abs() * emax[:, None] / amax_lo) / amax_lo + 3 * U32 * p.abs()
    lo, hi = fe.e4m3_round(p - e_p), fe.e4m3_round(p + e_p)
    got = q.float().double()
    ok = (got >= lo) & (got <= hi) | zero[:, None]
    if not ok.all():
        r, c = (int(i) for i in (~ok).nonzero()[0])
        raise AssertionError("%s: %d byte(s) outside the bound; first at [%d, %d]: got %r, allowed "
                             "[%r, %r]" % (what, (~ok).sum(), r, c, got[r, c].item(), lo[r, c].item(),
                                           hi[r, c].item()))
    return worst


def check16(out, ref, tol, what):
    bad, worst = bound_violations(out, ref, tol)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d of %d outside the float64 bound (worst %.3g); first at %s: got %r "
                             "ref %r tol %r" % (what, bad.sum(), bad.numel(), worst, i,
                                                out[tuple(i)].item(), ref[tuple(i)].item(),
                                                tol[tuple(i)].item()))
    return worst


def _record(family, name, worst):
    print("BOUND_RATIO %s %s %.4g" % (family, name, worst))


# --------------------------------------------------------------------------------------------
# GroupNorm: reference, bound, emulation
# --------------------------------------------------------------------------------------------
def stats_kernel(C, G):
    """The statistics kernel dwm_b200_groupnorm_stats launches."""
    vec = C // 4
    if (C // G) % 4 == 0 and vec <= 256 and 256 % vec == 0:
        return "fast"
    return "wide" if vec <= 1024 else "generic"


def apply_path(C, T):
    """spatialnorm_kernel's path: blockDim is a multiple of C / 4 up to C / 4 = 1024."""
    return "fast" if C // 4 <= 1024 and T <= 64 else "general"


def frame_map(T, Tz, bug=None):
    t = torch.arange(T)
    if T > 1 and T % 2 == 1 and bug != "t*Tz/T for odd T":
        return torch.where(t == 0, 0, 1 + (t - 1) * (Tz - 1) // (T - 1))
    return t * Tz // T


def group_sums(x, G):
    """float64 (sum, sum sq) [nb, G, 2] and sum |x| [nb, G] of x [nb, T, H, W, C]."""
    nb, C = x.shape[0], x.shape[-1]
    g = x.double().reshape(nb, -1, G, C // G).transpose(1, 2).reshape(nb, G, -1)
    return torch.stack([g.sum(-1), (g * g).sum(-1)], -1), g.abs().sum(-1)


def gn_reference(x, G, gamma, beta, eps, zy=None, zb=None, silu=True, stat_x=None):
    """float64 (ref, err) of GroupNorm(+SpatialNorm)(+SiLU) of x fp32 [nb, T, H, W, C] before the
    output rounding; statistics over stat_x (default x), err as the module docstring states."""
    sx = (x if stat_x is None else stat_x).double()
    nb, T, H, W, C = x.shape
    cg = C // G
    grp = sx.reshape(nb, -1, G, cg).transpose(1, 2).reshape(nb, G, -1)
    n_g = grp.shape[-1]
    mean = grp.mean(-1)
    var = ((grp - mean[..., None]) ** 2).mean(-1)
    mabs = grp.abs().mean(-1)
    e_var = 3 * (n_g + 2) * U64 * (var + mean ** 2)
    e_r = rstd_rel_error(var, eps, e_var)
    e_mu = U32 * mean.abs() + n_g * 2 * U64 * mabs
    per_c = lambda t: t.repeat_interleave(cg, -1)[:, None, None, None, :]  # noqa: E731
    mean_c, rstd_c, e_mu_c, e_r_c = per_c(mean), per_c(torch.rsqrt(var + eps)), per_c(e_mu), per_c(e_r)
    x64 = x.double()
    ga, be = gamma.double()[:C], beta.double()[:C]
    d = x64 - mean_c
    y = d * rstd_c * ga + be
    e_d = e_mu_c + U32 * (d.abs() + e_mu_c)
    err = ga.abs() * rstd_c * (e_d + d.abs() * (e_r_c + 2 * U32)) + U32 * y.abs()
    if zy is not None:
        Tz, hz, wz = zy.shape[1:4]
        tz = frame_map(T, Tz).to(x.device)
        hq = (torch.arange(H) * hz // H).to(x.device)
        wq = (torch.arange(W) * wz // W).to(x.device)
        zyy = zy.double()[:, tz][:, :, hq][:, :, :, wq]
        zbb = zb.double()[:, tz][:, :, hq][:, :, :, wq]
        prod = y * zyy
        y = prod + zbb
        err = zyy.abs() * err + U32 * (prod.abs() + y.abs())
    if silu:
        s, e_act = act_reference(y, SILU)
        y, err = s, 1.1 * err + e_act
    return y, err


def gn_emulate(x, G, gamma, beta, eps, zy=None, zb=None, silu=True, bug=None):
    """fp32 emulation of groupnorm_stats + the fast apply path; `bug` makes it a wrong kernel."""
    nb, T, H, W, C = x.shape
    cg = C // G
    if bug == "fp32 stats, no clamp":
        g = x.reshape(nb, -1, G, cg).transpose(1, 2).reshape(nb, G, -1).float()
        s = g.cumsum(-1)[..., -1].double()
        ss = (g * g).cumsum(-1)[..., -1].double()
        n = g.shape[-1]
        mean_d = s / n
        var_d = ss / n - mean_d * mean_d
    else:
        sums, _ = group_sums(x, G)
        n = x[0].numel() // G
        mean_d = sums[..., 0] / n
        var_d = (sums[..., 1] / n - mean_d * mean_d).clamp_min(0)
    var_f = var_d.float()
    rstd = 1 / (var_f.sqrt() + eps) if bug == "eps outside the sqrt" else torch.rsqrt(var_f + eps)
    mu = mean_d.float()
    gi = torch.arange(C)
    gi = (gi + 1) // cg % G if bug == "group index + 1 channel" else gi // cg
    mu_c, a_c = mu[:, gi], rstd[:, gi] * gamma[:C]
    y = ((x - mu_c[:, None, None, None]).double() * a_c[:, None, None, None].double() + beta[:C].double()).float()
    if zy is not None:
        Tz, hz, wz = zy.shape[1:4]
        tz = frame_map(T, Tz, bug)
        hq, wq = torch.arange(H) * hz // H, torch.arange(W) * wz // W
        zyy, zbb = zy[:, tz][:, :, hq][:, :, :, wq], zb[:, tz][:, :, hq][:, :, :, wq]
        y = (y.double() * zyy.double() + zbb.double()).float()
    if silu:
        y = torch.nn.functional.silu(y)
    return y


def gn_data(nb, T, H, W, C, G, seed, kinds=None):
    """x [nb, T, H, W, C] whose groups cycle through: benign (mean 0.5, std 2); |mean| / std of
    1e2, 1e3 and 1e4 (std 0.05 to 1, mean of either sign); a constant non-zero group; an all-zero
    group; a group of std 1e-3 (variance comparable to eps).  The kinds rotate with the volume
    index, so one volume holds groups of different offsets."""
    g = torch.Generator().manual_seed(seed)
    cg = C // G
    x = torch.empty(nb, T, H, W, G, cg)
    kinds = kinds or ["benign", "r1e2", "r1e3", "r1e4", "const", "zero", "tiny"]
    for n in range(nb):
        for gi in range(G):
            k = kinds[(gi + n) % len(kinds)]
            r = torch.randn(T, H, W, cg, generator=g)
            sign = 1 if (gi // len(kinds)) % 2 == 0 else -1
            if k == "benign":
                v = 0.5 + 2 * r
            elif k.startswith("r1e"):
                std = {"r1e2": 1.0, "r1e3": 0.2, "r1e4": 0.05}[k]
                v = sign * float(k[1:]) * std + std * r
            elif k == "const":
                v = torch.full_like(r, 123.4 * sign)
            elif k == "zero":
                v = torch.zeros_like(r)
            else:
                v = 1e-3 * r + 0.3
            x[n, :, :, :, gi] = v
    return x.reshape(nb, T, H, W, C)


def gn_params(C, seed, zero_beta=False):
    g = torch.Generator().manual_seed(seed + 1)
    gamma = 1 + 0.3 * torch.randn(C, generator=g)
    gamma[::7] *= -1
    beta = torch.zeros(C) if zero_beta else 0.2 * torch.randn(C, generator=g)
    return gamma, beta


def z_data(nb, Tz, hz, wz, C, seed):
    g = torch.Generator().manual_seed(seed + 2)
    return 1 + 0.5 * torch.randn(nb, Tz, hz, wz, C, generator=g), 0.5 * torch.randn(nb, Tz, hz, wz, C, generator=g)


# --------------------------------------------------------------------------------------------
# LayerNorm: reference, bound, emulation
# --------------------------------------------------------------------------------------------
class Ln:
    """One layernorm call's logical operands (fp32, [M, D] / [items, D] / [D])."""

    def __init__(self, x, rows_per_item=0, add_item=None, add_full=None, weight=None, bias=None,
                 shift=None, scale=None, shift2=None, scale2=None, eps=1e-6):
        self.x, self.rpi, self.add_item, self.add_full = x, rows_per_item, add_item, add_full
        self.weight, self.bias, self.eps = weight, bias, eps
        self.shift, self.scale, self.shift2, self.scale2 = shift, scale, shift2, scale2

    @property
    def dual(self):
        return self.shift2 is not None or self.scale2 is not None

    def items(self, bug=None):
        m = torch.arange(self.x.shape[0], device=self.x.device)
        it = m // self.rpi if self.rpi > 0 else torch.zeros_like(m)
        if bug == "modulation of item + 1":
            n_items = self.shift.shape[0] if self.shift is not None else 1
            it = (it + 1).clamp_max(n_items - 1)
        return it

    def row_sum(self):
        """fp32 v = x (+ add_item[item]) (+ add_full), in the kernel's order."""
        v = self.x.clone()
        if self.add_item is not None:
            v = v + self.add_item[self.items()]
        if self.add_full is not None:
            v = v + self.add_full
        return v


def _mod_steps(e, second):
    sc, sh = (e.scale2, e.shift2) if second else (e.scale, e.shift)
    return sc, sh


def ln_reference(e):
    """float64 [(ref, err)] of out (and out2) before the output rounding."""
    v32 = e.row_sum()
    M, D = v32.shape
    v = v32.double()
    mean = v.mean(-1, keepdim=True)
    d = v - mean
    var = (d * d).mean(-1, keepdim=True)
    L = 4 * math.ceil(D / 128) + 7
    e_mean = L * U32 * v.abs().mean(-1, keepdim=True)
    e_var = ((L + 3) * U32 * var + e_mean ** 2)
    e_r = rstd_rel_error(var, e.eps, e_var)
    rstd = torch.rsqrt(var + e.eps)
    y = d * rstd
    err = rstd * (e_mean + U32 * d.abs() + d.abs() * (e_r + U32))
    if e.weight is not None:
        w = e.weight.double()
        y, err = y * w, w.abs() * err + U32 * (y * w).abs()
    if e.bias is not None:
        y = y + e.bias.double()
        err = err + U32 * y.abs()
    it = e.items()
    outs = []
    for second in ([False, True] if e.dual else [False]):
        z, ez = y.clone(), err.clone()
        sc, sh = _mod_steps(e, second)
        if sc is not None:
            f = 1 + sc.double()[it]
            z, ez = z * f, f.abs() * ez + U32 * (z * f).abs() + U32 * z.abs() * (1 + sc.double()[it].abs())
        if sh is not None:
            z = z + sh.double()[it]
            ez = ez + U32 * z.abs()
        outs.append((z, ez))
    return outs


def ln_emulate(e, bug=None):
    """fp32 kernel: [out (fp32 values before the output rounding), (out2)]."""
    v = e.row_sum()
    D = v.shape[1]
    mean = v.sum(-1, keepdim=True) / D
    if bug == "one-pass fp32 variance":
        var = (v * v).sum(-1, keepdim=True) / D - mean * mean
    else:
        var = ((v - mean) ** 2).sum(-1, keepdim=True) / D
    y = (v - mean) * torch.rsqrt(var + e.eps)
    if e.weight is not None:
        y = y * e.weight
    if e.bias is not None:
        y = y + e.bias
    it = e.items(bug)
    outs = []
    for second in ([False, True] if e.dual else [False]):
        z = y.clone()
        sc, sh = _mod_steps(e, second)
        if sc is not None:
            z = z * (1 + sc[it])
        if sh is not None:
            z = z + sh[it]
        outs.append(z)
    return outs


def e4m3_emulate(v, bug=None):
    """Row-wise E4M3 of fp32 v [R, N] with the kernel's recipe -> (q, scale)."""
    q, s = fe.quantize_rows(v)
    if bug == "E4M3 scale inverted":
        amax = v.abs().amax(-1)
        s = torch.where(amax > 0, 448 / amax, torch.ones_like(amax))
    return q, s


def ln_rows(M, D, seed):
    """[M, D] rows cycling through mean / std = 0 (std 1), 1e2, 1e3, 1e4 (std 1, 0.1, 1) and a
    row of std 1e-3 (variance comparable to eps)."""
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(M, D, generator=g)
    mean = torch.tensor([0.5, 100.0, -1e2, 1e4, 0.3])[torch.arange(M) % 5][:, None]
    std = torch.tensor([1.0, 1.0, 0.1, 1.0, 1e-3])[torch.arange(M) % 5][:, None]
    return mean + std * r


def ln_case(M, D, seed, rpi=37, add_item=True, add_full=False, affine=True, mod="single",
            zero_item=None):
    g = torch.Generator().manual_seed(seed + 11)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    items = -(-M // rpi) if rpi else 1
    e = Ln(ln_rows(M, D, seed), rows_per_item=rpi)
    if add_item:
        e.add_item = 1e-3 * rn(items, D)
    if add_full:
        e.add_full = 1e-3 * rn(M, D)
    if affine:
        e.weight, e.bias = 1 + 0.2 * rn(D), 0.1 * rn(D)
    if mod in ("single", "dual"):
        e.shift, e.scale = 0.3 * rn(items, D), 0.3 * rn(items, D)
        if zero_item is not None:
            e.scale[zero_item] = -1.0
            e.shift[zero_item] = 0.0
    if mod == "dual":
        e.shift2, e.scale2 = 0.3 * rn(items, D), 0.3 * rn(items, D)
    return e


# --------------------------------------------------------------------------------------------
# CPU self-test
# --------------------------------------------------------------------------------------------
def _gn_selftest(bug, dtype=torch.bfloat16, zy=False):
    nb, T, H, W, C, G = 2, 3, 4, 6, 320, 32
    x = gn_data(nb, T, H, W, C, G, seed=3)
    gamma, beta = gn_params(C, 3)
    z = z_data(nb, 2, 2, 3, C, 3) if zy else (None, None)
    ref, err = gn_reference(x, G, gamma, beta, 1e-6, *z)
    out = gn_emulate(x, G, gamma, beta, 1e-6, *z, bug=bug).to(dtype)
    return bound_violations(out, ref, out16_tol(err, ref, dtype))


def _ln_selftest(bug, e4m3=False, dtype=torch.bfloat16):
    e = ln_case(96, 320, seed=5, rpi=20, mod="dual", zero_item=2)
    refs = ln_reference(e)
    outs = ln_emulate(e, bug if bug != "E4M3 scale inverted" else None)
    bad = False
    for v, (ref, err) in zip(outs, refs):
        if e4m3:
            q, s = e4m3_emulate(v, bug)
            try:
                e4m3_check(q, s, ref, err, "selftest")
            except AssertionError:
                bad = True
        else:
            b, _ = bound_violations(v.to(dtype), ref, out16_tol(err, ref, dtype))
            bad = bad or bool(b.any())
    return bad


def test_bounds_accept_emulated_kernels_and_reject_wrong_ones():
    """The fp32 emulations pass every bound (bf16 and fp16, 16-bit and E4M3 outputs); each
    wrong kernel fails."""
    for dtype in (torch.bfloat16, torch.float16):
        for zy in (False, True):
            bad, worst = _gn_selftest(None, dtype, zy)
            assert not bad.any(), ("groupnorm", dtype, zy, worst)
        assert not _ln_selftest(None, dtype=dtype)
    assert not _ln_selftest(None, e4m3=True)
    for bug in ("group index + 1 channel", "eps outside the sqrt", "fp32 stats, no clamp"):
        bad, _ = _gn_selftest(bug)
        assert bad.any(), bug
    # t * Tz / T differs from the odd-T map (Tz = 2, T = 3: frame 1 -> latent frame 0, not 1)
    bad, _ = _gn_selftest("t*Tz/T for odd T", zy=True)
    assert bad.any()
    for bug in ("one-pass fp32 variance", "modulation of item + 1"):
        assert _ln_selftest(bug), bug
    assert _ln_selftest("E4M3 scale inverted", e4m3=True)


def test_e4m3_check_rejects_a_code_off_by_one():
    """Moving one byte of an exact quantization to its neighbouring code is caught (the check does
    not accept every neighbour, only those whose pre-image may cross a midpoint)."""
    g = torch.Generator().manual_seed(0)
    v = torch.randn(8, 64, generator=g)
    q, s = fe.quantize_rows(v)
    e4m3_check(q, s, v.double(), torch.zeros_like(v, dtype=torch.float64), "exact")
    b = q.view(torch.uint8).clone()
    b[3, 5] += 1
    with pytest.raises(AssertionError):
        e4m3_check(b.view(FP8), s, v.double(), torch.zeros_like(v, dtype=torch.float64), "moved")


# --------------------------------------------------------------------------------------------
# GPU buffers
# --------------------------------------------------------------------------------------------
def in_poison(t, pad=64):
    """Contiguous CUDA copy of t inside an allocation whose other elements are NaN / +-Inf."""
    n = t.numel()
    x = torch.tensor([float("nan"), float("inf"), float("-inf")]).repeat((n + 2 * pad) // 3 + 1)[:n + 2 * pad]
    x = x.to(t.dtype)
    x[pad:pad + n] = t.reshape(-1)
    return x.cuda()[pad:pad + n].view(t.shape)


def sentinel_out(shape, dtype):
    """(flat sentinel allocation, contiguous view of `shape` GUARD elements into it)."""
    n = math.prod(shape)
    if dtype == FP8:
        buf = torch.full((n + 2 * GUARD,), SENT8, dtype=torch.uint8, device="cuda")
        return buf, buf[GUARD:GUARD + n].view(FP8).view(shape)
    buf = torch.full((n + 2 * GUARD,), SENT16, dtype=torch.int16, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(dtype).view(shape)


def _bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int16)


def check_untouched(buf, shape, written, what):
    """Every element of buf outside the frames [nb, written, ...] of the view keeps its sentinel."""
    sent = SENT8 if buf.dtype == torch.uint8 else SENT16
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    view = mask[GUARD:GUARD + math.prod(shape)].view(shape)
    view[:, written] = False
    stray = (buf != sent) & mask
    assert not stray.any(), "%s: %d element(s) written outside the frame window" % (what, stray.sum())


# --------------------------------------------------------------------------------------------
# GroupNorm statistics
# --------------------------------------------------------------------------------------------
STATS_CASES = [
    # (nb, T, H, W, C, G, kernel)
    (3, 2, 5, 7, 128, 32, "fast"),         # 70 pixels, 8 rows per iteration: ragged
    (2, 1, 3, 5, 64, 16, "fast"),
    (2, 1, 1, 1, 512, 32, "fast"),         # a single pixel
    (1, 1, 256, 448, 128, 32, "fast"),     # one large frame: long per-thread sums
    (2, 1, 3, 7, 64, 32, "wide"),          # 2 channels per group
    (2, 1, 5, 9, 320, 32, "wide"),         # 10
    (3, 1, 4, 7, 640, 32, "wide"),         # 20
    (2, 1, 3, 5, 960, 32, "wide"),         # 30
    (2, 1, 2, 3, 1280, 32, "wide"),        # 40
    (1, 1, 1, 1, 2560, 32, "wide"),        # 80, one pixel
    (2, 1, 3, 5, 4608, 32, "generic"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("nb,T,H,W,C,G,kernel", STATS_CASES,
                         ids=["%dx%dx%dx%dx%d_g%d_%s" % c for c in STATS_CASES])
def test_groupnorm_stats_conforms(nb, T, H, W, C, G, kernel):
    from opendwm_b200 import ops
    assert stats_kernel(C, G) == kernel
    x = gn_data(nb, T, H, W, C, G, seed=C + H)
    xd = in_poison(x)
    buf = torch.full((nb * G * 2 + 16,), float("nan"), dtype=torch.float64, device="cuda")
    sums = buf[8:8 + nb * G * 2].view(nb, G, 2)
    ops.groupnorm_stats(xd, G, sums)
    assert torch.isnan(buf[:8]).all() and torch.isnan(buf[-8:]).all(), "wrote outside sums"
    ref, sabs = group_sums(x, G)
    n_g = x[0].numel() // G
    # the kernel's chains and the float64 reference's own summation: 2 n_g 2^-53 each
    tol = torch.stack([2 * n_g * U64 * sabs, 2 * n_g * U64 * ref[..., 1]], -1)
    worst = check16(sums.cpu(), ref, tol, "groupnorm_stats")
    _record("groupnorm_stats", "%s_C%d" % (kernel, C), worst)


# --------------------------------------------------------------------------------------------
# GroupNorm / SpatialNorm apply
# --------------------------------------------------------------------------------------------
APPLY_CASES = [
    # (name, nb, T, H, W, C, G, silu, zy (Tz, hz, wz) or None, out_T, out_t0)
    ("fast_C128_plain", 2, 3, 4, 6, 128, 32, False, None, 5, 2),
    ("fast_C320_silu", 2, 2, 5, 7, 320, 32, True, None, 4, 1),
    ("fast_C64_g32_silu", 3, 1, 4, 5, 64, 32, True, None, 1, 0),
    ("fast_zy_T1_shift", 2, 1, 8, 12, 128, 32, True, (1, 4, 6), 3, 2),
    ("fast_zy_T4_shift", 1, 4, 8, 8, 128, 32, True, (2, 2, 4), 6, 1),
    ("fast_zy_T5_div", 2, 5, 6, 9, 64, 16, True, (3, 2, 3), 7, 2),
    ("fast_zy_T3_div_nosilu", 1, 3, 6, 10, 320, 32, False, (2, 3, 5), 4, 1),
    ("general_C4608_silu", 2, 1, 2, 3, 4608, 32, True, None, 2, 1),
    ("general_C4608_zy_T3", 1, 3, 2, 2, 4608, 32, True, (2, 1, 1), 5, 2),
    ("general_T65_zy_div", 1, 65, 2, 3, 64, 32, True, (17, 1, 1), 66, 1),
    ("general_T65_plain", 2, 65, 1, 2, 320, 32, False, None, 65, 0),
]


def _gn_inputs(case):
    name, nb, T, H, W, C, G, silu, z, out_T, out_t0 = case
    seed = C + T + H
    x = gn_data(nb, T, H, W, C, G, seed)
    gamma, beta = gn_params(C, seed)
    zy = zb = None
    if z is not None:
        zy, zb = z_data(nb, *z, C, seed)
    return x, gamma, beta, zy, zb


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", APPLY_CASES, ids=[c[0] for c in APPLY_CASES])
def test_spatialnorm_silu_conforms(case, dtype):
    from opendwm_b200 import ops
    name, nb, T, H, W, C, G, silu, z, out_T, out_t0 = case
    assert apply_path(C, T) == name.split("_")[0]
    x, gamma, beta, zy, zb = _gn_inputs(case)
    ref, err = gn_reference(x, G, gamma, beta, 1e-6, zy, zb, silu)
    xd = in_poison(x)
    sums = ops.groupnorm_stats(xd, G)
    args = dict(zy=in_poison(zy), zb=in_poison(zb)) if zy is not None else {}

    def run():
        buf, out = sentinel_out((nb, out_T, H, W, C), dtype)
        ops.spatialnorm_silu(xd, sums, in_poison(gamma), in_poison(beta), out, groups=G, eps=1e-6,
                             out_t0=out_t0, silu=silu, **args)
        torch.cuda.synchronize()
        return buf, out

    buf, out = run()
    check_untouched(buf, out.shape, slice(out_t0, out_t0 + T), name)
    got = out[:, out_t0:out_t0 + T].cpu()
    worst = check16(got, ref, out16_tol(err, ref, dtype), name)
    assert torch.equal(run()[0], buf), "the repeated call gave other bits"
    _record("spatialnorm", "%s_%s" % (name, dtype), worst)


E4M3_CASES = [
    # (name, nb, T, H, W, C, G, silu, out_T, out_t0)
    ("fast_C320_silu", 2, 3, 4, 6, 320, 32, True, 5, 1),
    ("fast_C128_plain", 3, 2, 5, 5, 128, 32, False, 2, 0),
    ("general_C4608", 1, 2, 2, 2, 4608, 32, True, 4, 2),
    ("general_T65_C64", 1, 65, 1, 2, 64, 16, True, 67, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", E4M3_CASES, ids=[c[0] for c in E4M3_CASES])
def test_groupnorm_silu_e4m3_conforms(case):
    """One volume of the batch is all zero with beta = 0 (its amax is 0: scale 1, zero bytes)."""
    from opendwm_b200 import ops
    name, nb, T, H, W, C, G, silu, out_T, out_t0 = case
    x = gn_data(nb, T, H, W, C, G, seed=C + T)
    gamma, beta = gn_params(C, C + T, zero_beta=True)
    x[-1] = 0
    ref, err = gn_reference(x, G, gamma, beta, 1e-6, silu=silu)
    xd = in_poison(x)
    sums = ops.groupnorm_stats(xd, G)

    def run():
        buf, out = sentinel_out((nb, out_T, H, W, C), FP8)
        scale = torch.full((nb,), -7.0, device="cuda")
        ops.groupnorm_silu_e4m3(xd, sums, in_poison(gamma), in_poison(beta), out, scale, groups=G,
                                eps=1e-6, out_t0=out_t0, silu=silu)
        torch.cuda.synchronize()
        return buf, out, scale

    buf, out, scale = run()
    check_untouched(buf, out.shape, slice(out_t0, out_t0 + T), name)
    q = out[:, out_t0:out_t0 + T].reshape(nb, -1)
    worst = e4m3_check(q, scale, ref.reshape(nb, -1), err.reshape(nb, -1), name)
    b2, _, s2 = run()
    assert torch.equal(b2, buf) and torch.equal(s2, scale), "the repeated call gave other bits"
    _record("groupnorm_e4m3_scale", name, worst)


HALO_CASES = [("fast_C320", 320, 6, 2, 3), ("fast_C64", 64, 5, 0, 2), ("fast_C128_last", 128, 5, 3, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, FP8], ids=["bf16", "fp16", "e4m3"])
@pytest.mark.parametrize("name,C,Tw,t0,T", HALO_CASES, ids=[c[0] for c in HALO_CASES])
def test_groupnorm_halo_conforms(name, C, Tw, t0, T, dtype):
    """A frame shard [t0, t0 + T) of a Tw-frame window, statistics over the window: its frames
    against float64, its boundary frames in the neighbours' operands (missing neighbours at the
    window's ends: a zero halo frame of its own), every other element at its sentinel."""
    from opendwm_b200 import ops
    nb, H, W, G = 2, 3, 5, 32
    xw = gn_data(nb, Tw, H, W, C, G, seed=C + Tw)
    gamma, beta = gn_params(C, C)
    ref, err = gn_reference(xw[:, t0:t0 + T], G, gamma, beta, 1e-6, stat_x=xw)
    xd = in_poison(xw[:, t0:t0 + T].contiguous())
    sums = ops.groupnorm_stats(in_poison(xw), G)
    has_prev, has_next = t0 > 0, t0 + T < Tw
    P, N = 4, 3                                      # neighbours' operand frames
    own_buf, out = sentinel_out((nb, T + 2, H, W, C), dtype)
    prev_buf, prev = sentinel_out((nb, P, H, W, C), dtype) if has_prev else (None, None)
    next_buf, nxt = sentinel_out((nb, N, H, W, C), dtype) if has_next else (None, None)
    g, b = in_poison(gamma), in_poison(beta)
    if dtype == FP8:
        amax = ops.groupnorm_silu_e4m3_amax(xd, sums, g, b, torch.empty(nb, device="cuda"), groups=G,
                                            stat_frames=Tw, eps=1e-6)
        torch.cuda.synchronize()
        amax_ref = ref.reshape(nb, -1).abs().amax(1)
        bad, _ = bound_violations(amax.cpu(), amax_ref, err.reshape(nb, -1).amax(1) + U32 * amax_ref)
        assert not bad.any(), "amax outside its bound"
        scale = torch.empty(nb, device="cuda")
        ops.groupnorm_silu_e4m3_halo(xd, sums, g, b, amax, out, scale, groups=G, stat_frames=Tw,
                                     prev_out=prev, next_out=nxt, eps=1e-6)
    else:
        ops.groupnorm_silu_halo(xd, sums, g, b, out, groups=G, stat_frames=Tw, prev_out=prev,
                                next_out=nxt, eps=1e-6)
    torch.cuda.synchronize()
    own = torch.zeros(T + 2, dtype=torch.bool)
    own[1:T + 1] = True
    own[0], own[T + 1] = not has_prev, not has_next
    check_untouched(own_buf, out.shape, own, name)
    if has_prev:
        check_untouched(prev_buf, prev.shape, slice(P - 1, P), name + " prev")
    if has_next:
        check_untouched(next_buf, nxt.shape, slice(0, 1), name + " next")
    for t in (0, T + 1):
        if own[t]:
            assert not _bits(out[:, t]).any(), "missing neighbour: the halo frame must be zero"
    frames = [out[:, 1:T + 1]]
    # the neighbours hold this shard's first / last frame
    first = prev[:, P - 1] if has_prev else out[:, 1]
    last = nxt[:, 0] if has_next else out[:, T]
    assert torch.equal(_bits(first), _bits(out[:, 1])) and torch.equal(_bits(last), _bits(out[:, T]))
    if dtype == FP8:
        q = frames[0].reshape(nb, -1)
        worst = e4m3_check(q, scale, ref.reshape(nb, -1), err.reshape(nb, -1), name)
    else:
        worst = check16(frames[0].cpu(), ref, out16_tol(err, ref, dtype), name)
    _record("groupnorm_halo", "%s_%s" % (name, dtype), worst)


# --------------------------------------------------------------------------------------------
# LayerNorm
# --------------------------------------------------------------------------------------------
LN_RESIDENT = [4, 320, 384, 388, 768, 772, 1280, 1536, 1540, 2048]
LN_STAGED = [320, 384, 388, 1536]
LD_PAD = 8


def _pitched(t, pad=LD_PAD):
    """CUDA [R, C] view of t with `pad` NaN / +-Inf columns after each row (pitch C + pad)."""
    R, C = t.shape
    x = torch.tensor([float("nan"), float("inf"), float("-inf")]).repeat(R * (C + pad) // 3 + 1)
    x = x[:R * (C + pad)].view(R, C + pad).to(t.dtype)
    x[:, :C] = t
    return x.cuda()[:, :C]


def _ln_launch(e, dtype, sum_out=True):
    """One call into fresh sentinel buffers: (out buffers [(buf, view)], scales, sum_out)."""
    from opendwm_b200 import ops
    M, D = e.x.shape
    P = LD_PAD * 2
    outs = []
    for _ in range(2 if e.dual else 1):
        n = M * (D + P)
        if dtype == FP8:
            buf = torch.full((n + 2 * GUARD,), SENT8, dtype=torch.uint8, device="cuda")
            view = buf[GUARD:GUARD + n].view(FP8).view(M, D + P)[:, :D]
        else:
            buf = torch.full((n + 2 * GUARD,), SENT16, dtype=torch.int16, device="cuda")
            view = buf[GUARD:GUARD + n].view(dtype).view(M, D + P)[:, :D]
        outs.append((buf, view))
    scales = [torch.full((M,), -7.0, device="cuda") for _ in outs] if dtype == FP8 else [None, None]
    so = _pitched(torch.full((M, D), float("nan")), 4) if sum_out else None
    mods = {}
    if e.shift is not None:
        # the four modulation vectors of an item share one row pitch (one [items, 4 D + 8] block)
        blk = torch.cat([t if t is not None else torch.zeros_like(e.shift)
                         for t in (e.shift, e.scale, e.shift2, e.scale2)], 1)
        blk = _pitched(blk)
        for i, k in enumerate(("shift", "scale", "shift2", "scale2")):
            if getattr(e, k) is not None:
                mods[k] = blk[:, i * D:(i + 1) * D]
    opt = lambda t: None if t is None else in_poison(t)  # noqa: E731
    ops.layernorm(_pitched(e.x), outs[0][1], weight=opt(e.weight), bias=opt(e.bias), eps=e.eps,
                  add_item=None if e.add_item is None else _pitched(e.add_item),
                  add_full=None if e.add_full is None else _pitched(e.add_full, 4),
                  rows_per_item=e.rpi, sum_out=so, out2=outs[1][1] if e.dual else None,
                  out_scale=scales[0], out2_scale=scales[1] if e.dual else None, **mods)
    torch.cuda.synchronize()
    return outs, scales, so


def _ln_check(e, dtype, what):
    outs, scales, so = _ln_launch(e, dtype)
    M, D = e.x.shape
    assert torch.equal(so.cpu().view(torch.int32), e.row_sum().view(torch.int32)), \
        "%s: sum_out is not the fp32 sum" % what
    worst = 0.0
    for (buf, view), s, (ref, err) in zip(outs, scales, ln_reference(e)):
        sent = SENT8 if dtype == FP8 else SENT16
        mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
        mask[GUARD:GUARD + M * (D + 2 * LD_PAD)].view(M, -1)[:, :D] = False
        assert not ((buf != sent) & mask).any(), "%s: wrote outside the rows" % what
        if dtype == FP8:
            worst = max(worst, e4m3_check(view.contiguous(), s, ref, err, what))
        else:
            worst = max(worst, check16(view.cpu(), ref, out16_tol(err, ref, dtype), what))
    outs2, scales2, _ = _ln_launch(e, dtype)
    for (b1, _), (b2, _) in zip(outs, outs2):
        assert torch.equal(b1, b2), "%s: the repeated call gave other bits" % what
    if dtype == FP8:
        for s1, s2 in zip(scales, scales2):
            assert s1 is None or torch.equal(s1, s2), "%s: the repeated call gave other scales" % what
    return worst


def _ln_dtype_ids():
    return pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, FP8],
                                   ids=["bf16", "fp16", "e4m3"])


@pytest.mark.gpu
@_ln_dtype_ids()
@pytest.mark.parametrize("D", LN_RESIDENT)
def test_layernorm_resident_conforms(D, dtype):
    """M = 150 rows (ragged against 4 rows per block), items of 37 rows, add_item + add_full +
    sum_out + weight / bias + DUAL modulation, one item with scale -1 / shift 0 (all-zero rows);
    the resident kernel (add_full keeps the staged one away)."""
    e = ln_case(150, D, seed=D, rpi=37, add_full=True, mod="dual", zero_item=1)
    worst = _ln_check(e, dtype, "resident_D%d" % D)
    _record("layernorm", "resident_D%d_%s" % (D, dtype), worst)


@pytest.mark.gpu
@_ln_dtype_ids()
@pytest.mark.parametrize("staged", [1, 0])
@pytest.mark.parametrize("D", LN_STAGED)
def test_layernorm_large_m_conforms(D, staged, dtype):
    """M = 4103 rows (a ragged last 16-row group), items of 37 rows (item boundaries inside the
    staged kernel's row groups), add_item + sum_out + single modulation (no affine), with the
    staged kernel (ln_staged = 1) and the resident one (0)."""
    from opendwm_b200 import lib
    e = ln_case(4103, D, seed=D + 1, rpi=37, affine=False, mod="single", zero_item=3)
    lib.set_option("ln_staged", staged)
    try:
        worst = _ln_check(e, dtype, "M4103_D%d_staged%d" % (D, staged))
    finally:
        lib.set_option("ln_staged", 1)
    _record("layernorm", "M4103_D%d_staged%d_%s" % (D, staged, dtype), worst)


@pytest.mark.gpu
def test_layernorm_plain_no_items():
    """No items, no affine, no modulation: plain LayerNorm of ill-conditioned rows."""
    e = ln_case(33, 1536, seed=9, rpi=0, add_item=False, affine=False, mod=None)
    _ln_check(e, torch.bfloat16, "plain")


# --------------------------------------------------------------------------------------------
# E4M3 row quantization
# --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("K", [16, 272, 4096 + 16])
def test_quantize_rows_bit_exact(K, dtype):
    """ld > K (poisoned), ldo > K (bytes [K, ldo) keep their sentinel); a zero row, a row with one
    non-zero, a row in E4M3's subnormal range after scaling, rows of mixed magnitude.  K = 272:
    34 chunks of 8, not a multiple of 32 lanes."""
    from opendwm_b200 import ops
    g = torch.Generator().manual_seed(K)
    M = 13
    x = torch.randn(M, K, generator=g) * torch.logspace(-3, 3, M)[:, None]
    x[0] = 0
    x[1] = 0
    x[1, K // 3] = -2.5
    x[2] = torch.randn(K, generator=g) * 1e-5
    x[2, 0] = 1.0                                   # the rest scales below 2^-6: subnormal codes
    x = x.to(dtype)
    xd = _pitched(x, 8)
    ldo = K + 32
    buf = torch.full((M * ldo + 2 * GUARD,), SENT8, dtype=torch.uint8, device="cuda")
    out = buf[GUARD:GUARD + M * ldo].view(M, ldo)[:, :K].view(FP8)
    scale = torch.full((M,), -7.0, device="cuda")
    ops.quantize_rows(xd, out, scale)
    torch.cuda.synchronize()
    q_ref, s_ref = fe.quantize_rows(x)
    assert torch.equal(out.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert torch.equal(scale.cpu(), s_ref)
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    mask[GUARD:GUARD + M * ldo].view(M, ldo)[:, :K] = False
    assert not ((buf != SENT8) & mask).any(), "wrote outside [M, K]"
    assert (q_ref[2].float().abs() < 2.0 ** -6).sum() > K // 2


# --------------------------------------------------------------------------------------------
# RMSNorm (T5LayerNorm)
# --------------------------------------------------------------------------------------------
SENT32 = 0x7FABCDEF              # int32 bits of every fp32 element a call must not write (a NaN)
RMS_THREADS = 256
FP16_MAX, FP16_OVERFLOW = 65504.0, 65520.0   # fp16's largest finite value; RN rounds >= 65520 to Inf


def rms_rows(M, D, seed):
    """[M, D] rows cycling through: benign (0.5 + 2 N(0, 1)); all zero; N(0, 1) scaled by 1e-4
    (mean square far below eps) and by 1e4; and rows sized like T5-v1.1's residual stream
    (std 30 with every 331st column 300 times larger)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=g)
    kind = torch.arange(M) % 5
    x[kind == 0] = 0.5 + 2 * x[kind == 0]
    x[kind == 1] = 0
    x[kind == 2] *= 1e-4
    x[kind == 3] *= 1e4
    t5 = x[kind == 4] * 30
    t5[:, ::331] *= 300
    x[kind == 4] = t5
    return x


def rms_weight(D, seed, big=True):
    """1 + 0.2 N(0, 1); with `big`, every 97th entry +-3e5 (fp16 overflows there)."""
    g = torch.Generator().manual_seed(seed + 1)
    w = 1 + 0.2 * torch.randn(D, generator=g)
    if big:
        w[::97] = 3e5 * (torch.randint(0, 2, w[::97].shape, generator=g) * 2 - 1)
    return w


def rms_reference(x, w, eps):
    """float64 (ref, err) of w x rsqrt(mean(x^2) + eps), err as the module docstring states."""
    D = x.shape[1]
    eps = torch.tensor(eps, dtype=torch.float32).item()
    xd = x.double()
    ref = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    L = 4 + math.ceil(D / (4 * RMS_THREADS)) + 5 + 7
    return ref, ((L + 2) * U32 / 2 + 6 * U32) * ref.abs()


def rms_emulate(x, w, eps, bug=None):
    """fp32 kernel; `bug` makes it a wrong one."""
    D = x.shape[1]
    n = D - 4 if bug == "mean over D - 4 columns" else D
    ms = (x[:, :n] * x[:, :n]).sum(-1, keepdim=True) / n
    r = 1 / (ms.sqrt() + eps) if bug == "eps outside the rsqrt" else torch.rsqrt(ms + eps)
    return w * (x * r)


def rms_check(out, ref, err, dtype, what):
    """out (any device) against (ref, err): the bound, and fp16's overflow to +-Inf."""
    out = out.cpu().double()
    tol = out16_tol(err, ref, dtype)
    if dtype == torch.float16:
        inf = ref.abs() - tol >= FP16_OVERFLOW           # rounds to Inf whatever the kernel's error
        edge = ~inf & (ref.abs() + tol >= FP16_OVERFLOW)  # may round either way
        sign = torch.sign(ref)
        assert torch.equal(out[inf], sign[inf] * math.inf), "%s: fp16 overflow is not +-Inf" % what
        ok_edge = (out[edge] == sign[edge] * math.inf) | (out[edge] == sign[edge] * FP16_MAX)
        assert ok_edge.all(), "%s: fp16 result at the overflow threshold is neither +-65504 nor +-Inf" % what
        fin = ~(inf | edge)
        return check16(out[fin], ref[fin], tol[fin], what)
    return check16(out, ref, tol, what)


def test_rmsnorm_bound_accepts_emulated_kernel_and_rejects_wrong_ones():
    """The fp32 emulation passes the bound in every output type (fp16 overflow included); the
    mean over D - 4 columns and eps outside the rsqrt fail it, at D = 68 in every type and at
    D = 1028 in fp32."""
    for D, dtypes in ((68, (torch.bfloat16, torch.float16, torch.float32)), (1028, (torch.float32,))):
        x, w = rms_rows(40, D, seed=D), rms_weight(D, seed=D)
        ref, err = rms_reference(x, w, 1e-6)
        for dtype in dtypes:
            rms_check(rms_emulate(x, w, 1e-6).to(dtype), ref, err, dtype, "emulated")
            if dtype == torch.float16:
                assert (ref.abs() > FP16_OVERFLOW).any(), "the case must overflow fp16"
            for bug in ("mean over D - 4 columns", "eps outside the rsqrt"):
                with pytest.raises(AssertionError):
                    rms_check(rms_emulate(x, w, 1e-6, bug).to(dtype), ref, err, dtype, bug)


RMS_CASES = [(1, 4), (77, 1020), (300, 1024), (5, 1028), (77, 1284), (2053, 4096), (300, 4100),
             (3001, 1024)]
RMS_LDO_PAD = 12


def _rms_launch(xd, wd, dtype):
    """One call into a fresh sentinel allocation: (flat buffer, [M, D] view of pitch D + 12)."""
    from opendwm_b200 import ops
    M, D = xd.shape
    n = M * (D + RMS_LDO_PAD)
    if dtype == torch.float32:
        buf = torch.full((n + 2 * GUARD,), SENT32, dtype=torch.int32, device="cuda")
    else:
        buf = torch.full((n + 2 * GUARD,), SENT16, dtype=torch.int16, device="cuda")
    view = buf[GUARD:GUARD + n].view(dtype).view(M, D + RMS_LDO_PAD)[:, :D]
    ops.rmsnorm(xd, wd, view, eps=1e-6)
    torch.cuda.synchronize()
    return buf, view


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("M,D", RMS_CASES, ids=["M%d_D%d" % c for c in RMS_CASES])
def test_rmsnorm_conforms(M, D, dtype):
    """x with a NaN / +-Inf row pitch, the weight inside a NaN / +-Inf allocation, the output in
    a sentinel allocation with a pitch and guard elements.  D = 1020 / 1024 / 1028: both sides
    of one pass of 256 threads x float4; 4096 / 4100: four passes and a ragged fifth."""
    x, w = rms_rows(M, D, seed=M + D), rms_weight(D, seed=D)
    ref, err = rms_reference(x, w, 1e-6)
    xd, wd = _pitched(x), in_poison(w)
    buf, out = _rms_launch(xd, wd, dtype)
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    mask[GUARD:GUARD + M * (D + RMS_LDO_PAD)].view(M, -1)[:, :D] = False
    sent = SENT32 if dtype == torch.float32 else SENT16
    assert not ((buf != sent) & mask).any(), "wrote outside the [M, D] rows"
    assert (out[(torch.arange(M) % 5 == 1).cuda()] == 0).all(), "an all-zero row must give 0"
    worst = rms_check(out, ref, err, dtype, "rmsnorm_M%d_D%d" % (M, D))
    assert torch.equal(_rms_launch(xd, wd, dtype)[0], buf), "the repeated call gave other bits"
    _record("rmsnorm", "M%d_D%d_%s" % (M, D, dtype), worst)
