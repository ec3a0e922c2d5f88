"""Element-wise conformance of both attention kernels against a float64 softmax(QK^T s) V of
the same 16-bit q|k|v, at the tile, mask and layout edges where they can go wrong.

attention.cu (mma.sync, cp.async gathers) and attention_wgmma.cu (warpgroup MMA with TMA
loads: a contiguous 2-D tensor-map path and a gathered 5-D one with a unit mask) must agree
with the reference everywhere, and `dwm_b200_attention` picks between them silently from the
layout.  Every GPU case therefore:

  * writes into views of sentinel-filled buffers with guard rows before and after and a
    row pitch `ldo > D`: every element outside the expected write set must keep the
    sentinel's bits, every element inside must be finite and within `bound_violations`;
  * reads a q|k|v buffer whose rows that no sequence position maps to (padding between
    groups, rows after the last group) and whose columns past 3D hold NaN / +-Inf;
  * runs under attn_tc = 0 (mma.sync only) and attn_tc = 2 (wgmma where eligible), with
    `kernel_path` (a restatement of attn_tc_eligible / attn_tcg_eligible) saying which kernel
    attn_tc = 2 must reach: the same bits as attn_tc = 0 when it says mma.sync, other bits when
    it says wgmma (so a case meant for the wgmma kernel cannot quietly test mma.sync twice);
  * repeats the attn_tc = 2 call, which must give identical bits.

Causal (CLIP) and biased (T5) attention, `dwm_b200_attention_text`, runs one kernel,
attn_wgmma_kernel<T, false, false, CAUSAL, BIAS>, under every attn_tc setting: its cases run
under attn_tc = 0 and 2 and must give the same bits, and `check_text_attention_selection` checks
with torch.profiler that the kernel launched carries the expected flags.

The CPU self-test checks the bound itself against an emulated kernel and seven wrong ones.
"""
import re
import math

import pytest
import torch

from test_gemm_conformance_gpu import run_isolated

SENTINEL = -21555     # int16 0xABCD: the bits of every output element the call must not write
GUARD = 3             # sentinel rows before and after each output buffer
LDO_PAD = 24          # sentinel columns after D in each output row (ldo = D + 24)
LD_PAD = 8            # poisoned columns after 3D in each q|k|v row (ld = 3D + 8)
POISON = (float("nan"), float("inf"), float("-inf"))


def unit_roundoff(dtype):
    return {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dtype]


# --------------------------------------------------------------------------------------------
# layouts
# --------------------------------------------------------------------------------------------
class Layout:
    """One attention call's addressing, as dwm_attention_args (include/dwm_b200.h) defines
    it: position j of group (g0, g1, g2) reads q|k|v row
        g0*gs0 + g1*gs1 + g2*gs2 + (j // inner)*stride_outer + (j % inner)*stride_inner
    and writes the same formula over the out_* strides; with split > 0, positions j >= split
    write out2 row g*(seq - split) + (j - split), g the flat group index."""

    def __init__(self, heads, group_dims, group_strides, seq, inner=None, stride_outer=0,
                 stride_inner=1, out_group_strides=None, out_stride_outer=None,
                 out_stride_inner=None, split=0, mask=None, mask_div=1, tail=5, scale=0.125,
                 causal=False, bias=None):
        pad = lambda v, fill: list(v) + [fill] * (3 - len(v))  # noqa: E731
        self.heads, self.seq, self.split = heads, seq, split
        self.scale, self.causal, self.bias = scale, causal, bias
        self.gd, self.gs = pad(group_dims, 1), pad(group_strides, 0)
        self.inner = seq if inner is None else inner
        self.so, self.si = stride_outer, stride_inner
        self.ogs = self.gs if out_group_strides is None else pad(out_group_strides, 0)
        self.oso = stride_outer if out_stride_outer is None else out_stride_outer
        self.osi = stride_inner if out_stride_inner is None else out_stride_inner
        self.mask, self.mask_div = mask, mask_div
        self.G = self.gd[0] * self.gd[1] * self.gd[2]
        self.in_rows = self._rows(self.gs, self.so, self.si)
        self.n_rows = int(self.in_rows.max()) + 1 + tail     # `tail` unused rows at the end
        n_main = split if split else seq
        self.out_rows = self._rows(self.ogs, self.oso, self.osi)[:, :n_main]
        assert self.out_rows.unique().numel() == self.out_rows.numel(), "output rows overlap"
        if split:
            g = torch.arange(self.G).view(-1, 1)
            self.out2_rows = g * (seq - split) + torch.arange(seq - split).view(1, -1)

    def _rows(self, gs, so, si):
        g0, g1, g2, j = torch.meshgrid(torch.arange(self.gd[0]), torch.arange(self.gd[1]),
                                       torch.arange(self.gd[2]), torch.arange(self.seq),
                                       indexing="ij")
        r = g0 * gs[0] + g1 * gs[1] + g2 * gs[2] + (j // self.inner) * so + (j % self.inner) * si
        return r.reshape(self.G, self.seq)

    def mask_bool(self):
        """bool [G, seq(query), seq(key)] or None: mask[g0 // mask_div, jq // inner, jk // inner]."""
        if self.mask is None:
            return None
        g0 = torch.arange(self.G) // (self.gd[1] * self.gd[2])
        u = torch.arange(self.seq) // self.inner
        m = self.mask.cpu().bool()[g0 // self.mask_div]
        return m[:, u][:, :, u]

    def kwargs(self):
        kw = dict(heads=self.heads, group_dims=self.gd, group_strides=self.gs, seq=self.seq,
                  inner=self.inner, stride_outer=self.so, stride_inner=self.si,
                  out_group_strides=self.ogs, out_stride_outer=self.oso,
                  out_stride_inner=self.osi, split=self.split, mask_div=self.mask_div)
        if self.mask is not None:
            kw["mask"] = self.mask.to(torch.uint8).cuda().contiguous()
        if self.text:
            kw.update(scale=self.scale, causal=self.causal,
                      bias=None if self.bias is None else self.bias.float().cuda().contiguous())
        return kw

    @property
    def text(self):
        return self.causal or self.bias is not None

    def kernel_path(self):
        """Which kernel attn_tc >= 1 selects: "tc" (wgmma, 2-D tensor map), "tcg" (wgmma, 5-D
        gathered tensor map) or "mma" (attention.cu).  Restates attn_tc_eligible and
        attn_tcg_eligible of attention_wgmma.cu for calls without a separate kv.  Causal or
        biased calls ("text") run attn_wgmma_kernel<T, false, false, CAUSAL, BIAS> whatever
        attn_tc says."""
        if self.text:
            return "text"
        gd, gs, ogs = self.gd, self.gs, self.ogs
        if (self.mask is None and gd[1] == 1 and gd[2] == 1 and self.inner == self.seq and
                self.si == 1 and self.osi == 1 and self.seq > 64 and gs[0] == self.seq and
                gd[0] * gs[0] < 2 ** 31):
            return "tc"
        if self.split > 0 or self.seq <= 64 or not 0 < self.inner <= 128:
            return "mma"
        if self.inner == self.seq and self.mask is None:
            return "mma"
        if self.seq % self.inner or self.si != 1 or self.osi != 1:
            return "mma"
        n_out = self.seq // self.inner
        if n_out > 32 or (self.mask is not None and self.mask.shape[-1] != n_out):
            return "mma"
        if gd[2] > 1 and (gs[1] != gd[2] * gs[2] or ogs[1] != gd[2] * ogs[2]):
            return "mma"
        if self.so <= 0 or gs[0] <= 0 or self.G * self.heads * 8 >= 2 ** 31:
            return "mma"
        return "tcg"


def contiguous(heads, N, seq, pad=0, out_pad=None, split=0, **text):
    """N contiguous sequences `pad` rows apart (joint / dual / UNet spatial attention; with
    `text` = scale / causal / bias, the text encoders' attention)."""
    ogs = None if out_pad is None else [seq + out_pad]
    return Layout(heads, [N], [seq + pad], seq, out_group_strides=ogs, split=split, **text)


def crossview(heads, BT, H, V, W, *, unit_pad=0, group_pad=0, out="same", mask=None,
              mask_div=1):
    """(bt v) (h w) -> (bt h) (v w): view v of frame bt is a block of S = H*W + unit_pad
    rows; sequence (bt, h) is V units of W tokens.  out="seq" writes each sequence
    contiguously instead of back in the input layout."""
    S = H * W + unit_pad
    kw = {}
    if out == "seq":
        kw = dict(out_group_strides=[H * V * W, V * W], out_stride_outer=W)
    return Layout(heads, [BT, H], [V * S + group_pad, W], V * W, inner=W, stride_outer=S,
                  mask=mask, mask_div=mask_div, **kw)


def temporal_rowwise(heads, B, T, V, H, W, *, group_pad=0, out="same", mask=None, mask_div=1):
    """(b t v) (h w) -> (b v h) (t w): three group dims, merged by the gathered wgmma kernel
    (group_strides[1] == group_dims[2] * group_strides[2])."""
    S = H * W
    kw = {}
    if out == "seq":
        kw = dict(out_group_strides=[V * H * T * W, H * T * W, T * W], out_stride_outer=W)
    return Layout(heads, [B, V, H], [T * V * S + group_pad, S, W], T * W, inner=W,
                  stride_outer=V * S, mask=mask, mask_div=mask_div, **kw)


def pointwise(heads, B, R, T, group_pad=0):
    """(b t r) -> (b r) t: sequences of single-token units (temporal point-wise)."""
    return Layout(heads, [B, R], [T * R + group_pad, 1], T, inner=1, stride_outer=R,
                  stride_inner=0)


def unit_mask(kind, batches, n, seed):
    """uint8 [batches, n, n] unit mask: "ones"; "diag" = random with the self unit always set;
    "empty" = "diag" with whole rows cleared (queries that may attend to nothing)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "ones":
        return torch.ones(batches, n, n, dtype=torch.uint8)
    m = torch.rand(batches, n, n, generator=g) < 0.5
    m |= torch.eye(n, dtype=torch.bool)
    if kind == "empty":
        rows = torch.rand(batches, n, generator=g) < 0.3
        rows[:, n // 2] = True
        m &= ~rows[:, :, None]
    return m.to(torch.uint8)


# --------------------------------------------------------------------------------------------
# reference, bound and emulated kernel
# --------------------------------------------------------------------------------------------
def gather_qkv(qkv, rows, heads):
    """q, k, v as [G, heads, seq, 64] from the rows of a [*, >= 3*heads*64] buffer."""
    G, S = rows.shape
    x = qkv[rows.reshape(-1).to(qkv.device), :3 * heads * 64].view(G, S, 3, heads, 64)
    return x.permute(2, 0, 3, 1, 4)


def causal_mask(S, shift=0):
    """bool [S, S]: query i attends keys j <= i + shift (CLIP's causal mask at shift 0)."""
    return torch.ones(S, S, dtype=torch.bool).tril(shift)


def reference(q, k, v, scale, mask=None, causal=False, bias=None):
    """float64 (softmax(q k^T scale + bias) v, the same softmax applied to |v|, the sum of |v|
    over each query's attended keys) for q, k, v [G, H, S, 64], mask bool [G, S, S] (True =
    attend), `causal` (key j > query i dropped) and bias [H, S, S] (added after the scale, as
    the kernel does).  A query whose every key is masked gives 0 in all three (the kernels'
    contract, include/dwm_b200.h)."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.transpose(-1, -2) * scale
    if bias is not None:
        s = s + bias.double().to(s.device)[None]
    if mask is not None:
        s = s.masked_fill(~mask[:, None].to(s.device), float("-inf"))
    if causal:
        s = s.masked_fill(~causal_mask(s.shape[-1]).to(s.device), float("-inf"))
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - torch.where(torch.isfinite(m), m, torch.zeros_like(m)))
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    return p @ v, p @ v.abs(), torch.isfinite(s).double() @ v.abs()


def bound_violations(out, ref, pv_abs, u, v_sum=None):
    """Elements of `out` outside |out - ref| <= u |ref| + 2u (P|V|) + 1e-6 (P|V|) (+ 2^-24 sum|v|
    in fp16), and the worst ratio |out - ref| / bound.  P|V| is the float64 softmax applied to
    |V|: the weighted mean of the attended |v| for that query, head and column; sum|v| (`v_sum`)
    the plain sum of the attended |v|.

    The bound follows from where a kernel rounds (u = unit roundoff: 2^-8 bf16, 2^-11 fp16):
      * P is rounded to 16 bits for the P.V MMA: each p_j moves by at most u p_j, so the
        numerator sum_j p_j v_j moves by at most u sum_j p_j |v_j|.  The normaliser l is summed
        from the unrounded p, so nothing cancels this: at most u (P|V|) after dividing by l;
      * the second u (P|V|) is slack for the same rounding seen through a running max that
        differs from the final one by a rescale (corr) and for the ex2.approx / fp32 MMA
        accumulation, whose relative errors (~2^-22) are far smaller;
      * the output is rounded to 16 bits once: at most u |ref| (plus u times the errors above);
      * 1e-6 (P|V|) covers fp16 P values below 2^-14 that round to subnormals, whose absolute
        error 2^-25 is not relative to p.  That holds while the keys with such p carry |v| like
        the winners'.  With `v_sum`, fp16 also gets 2^-24 sum|v|: every unnormalised p_j <=
        2^(1/16) (see below) moves by at most 2^-25 absolutely and l >= 2^(-1/16), so this
        bounds them whatever their |v|.  The unscaled T5 logits (std ~10 and more) put most
        keys there.
    A query whose every key is masked has ref = P|V| = 0, so it must come out exactly 0.

    Worst ratio over this file's cases, measured on an H100 80GB HBM3 (bf16 / fp16):
    mma.sync 0.43 / 0.46; wgmma 0.63 / 0.65, both in the case where one key wins by 2^20.
    The text kernel (causal / biased, on an H100 80GB HBM3 at a 700 W power limit): 0.60 / 0.62
    on the random-data cases, 0.63 / 0.64 on the logit extremes.
    There the wgmma kernel's running max is the fp32 product max*scale while p is
    ex2(fma(s, scale, -max)), so the winner's p is 2^(+-1/16), not 1: its 16-bit rounding then
    costs the full u (P|V|) above, on top of the output's u |ref|."""
    out = out.double()
    tol = u * ref.abs() + (2 * u + 1e-6) * pv_abs
    if v_sum is not None and u == 2.0 ** -11:
        tol = tol + 2.0 ** -24 * v_sum
    err = (out - ref).abs()
    bad = ~(err <= tol)                         # NaN / Inf in out count as violations
    ratio = torch.where(err == 0, 0.0, err / tol)
    ratio = torch.where(torch.isnan(ratio), math.inf, ratio)   # a NaN in out
    return bad, ratio.max().item() if ratio.numel() else 0.0


def emulate(q, k, v, scale, dtype, mask=None, block=128, drop_last_block=False, causal=False,
            bias=None):
    """fp32 online softmax over key blocks as both kernels compute it: running max, P rounded
    to `dtype` before P.V, l summed from the unrounded p, the output rounded to `dtype` once;
    `causal` / `bias` [H, S, S] as `reference` takes them."""
    q, k, v = q.float(), k.float(), v.float()
    G, H, S, _ = q.shape
    if causal:
        cm = causal_mask(S).expand(G, S, S)
        mask = cm if mask is None else mask & cm
    m = torch.full((G, H, S, 1), float("-inf"))
    l = torch.zeros(G, H, S, 1)
    o = torch.zeros(G, H, S, 64)
    n_blocks = (S + block - 1) // block - (1 if drop_last_block else 0)
    for b in range(n_blocks):
        sl = slice(b * block, (b + 1) * block)
        s = q @ k[:, :, sl].transpose(-1, -2) * scale
        if bias is not None:
            s = s + bias.float()[None, :, :, sl]
        if mask is not None:
            s = s.masked_fill(~mask[:, None, :, sl], float("-inf"))
        m_new = torch.maximum(m, s.amax(-1, keepdim=True))
        ref = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
        corr = torch.exp(m - ref)
        p = torch.exp(s - ref)
        l = l * corr + p.sum(-1, keepdim=True)
        o = o * corr + p.to(dtype).float() @ v[:, :, sl]
        m = m_new
    return (o * torch.where(l > 0, 1.0 / l, torch.zeros_like(l))).to(dtype)


# --------------------------------------------------------------------------------------------
# CPU self-test of the bound
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bound_accepts_emulated_kernel_and_rejects_wrong_ones(dtype):
    """The bound passes an emulated kernel and fails each of three plausible kernel bugs:
    a dropped last key block, the scale 1/sqrt(65) for 1/sqrt(64), and keys / values read one
    row off in a gathered layout.  Cross-view layout, seq 4 x 48 = 192 (two key blocks), a
    mask with fully masked rows, queries of std 2 (logits of std ~2).

    Then the text path, 3 contiguous sequences of 150 tokens (two key blocks), 2 heads: the
    emulated causal and biased kernels pass, and four wrong ones fail: the causal mask
    shifted by one key, the bias transposed ([h, j, i]), the bias of head h + 1, and the bias
    multiplied by the scale (0.125 here: at T5's scale 1 that bug is invisible)."""
    lay = crossview(2, BT=2, H=2, V=4, W=48, unit_pad=3,
                    mask=unit_mask("empty", 2, 4, seed=1), mask_div=1)
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(lay.n_rows, 3 * 128, generator=g)
    qkv[:, :128] *= 2.0
    qkv = qkv.to(dtype)
    u = unit_roundoff(dtype)
    mask = lay.mask_bool()
    q, k, v = gather_qkv(qkv, lay.in_rows, 2)
    ref, pv, _ = reference(q, k, v, 0.125, mask)
    assert (~mask).all(-1).any(), "the case must have fully masked queries"

    bad, worst = bound_violations(emulate(q, k, v, 0.125, dtype, mask), ref, pv, u)
    assert not bad.any(), worst
    assert worst > 0.05, worst          # the bound is not vacuous for the correct kernel either

    wrong = {
        "drop last key block": emulate(q, k, v, 0.125, dtype, mask, drop_last_block=True),
        "scale 1/sqrt(65)": emulate(q, k, v, 65 ** -0.5, dtype, mask),
    }
    _, k1, v1 = gather_qkv(qkv, lay.in_rows + 1, 2)
    wrong["k, v one row off"] = emulate(q, k1, v1, 0.125, dtype, mask)
    for name, out in wrong.items():
        bad, worst = bound_violations(out, ref, pv, u)
        assert bad.any(), (name, worst)

    lay = contiguous(2, 3, 150)
    q, k, v = gather_qkv(torch.randn(lay.n_rows, 3 * 128, generator=g).to(dtype), lay.in_rows, 2)
    bias = torch.randn(2, 150, 150, generator=g) * 3
    S = lay.seq
    for causal, b, wrong in [
            (True, None, {"causal mask shifted by one key":
                          dict(mask=causal_mask(S, 1).expand(lay.G, S, S))}),
            (False, bias, {"bias transposed": dict(bias=bias.transpose(1, 2)),
                           "bias of head h + 1": dict(bias=bias.roll(-1, 0)),
                           "bias multiplied by the scale": dict(bias=bias * 0.125)})]:
        ref, pv, vs = reference(q, k, v, 0.125, causal=causal, bias=b)
        bad, worst = bound_violations(emulate(q, k, v, 0.125, dtype, causal=causal, bias=b), ref, pv, u, vs)
        assert not bad.any(), ("causal" if causal else "bias", worst)
        assert worst > 0.05, worst
        for name, kw in wrong.items():
            kw = dict(dict(causal=causal, bias=b), **kw)
            if "mask" in kw:
                kw["causal"] = False
            bad, worst = bound_violations(emulate(q, k, v, 0.125, dtype, **kw), ref, pv, u, vs)
            assert bad.any(), (name, worst)


# --------------------------------------------------------------------------------------------
# GPU cases
# --------------------------------------------------------------------------------------------
def _contiguous_cases():
    # (seq, heads, N): items = N * heads * ceil(seq / 128) against 132 SMs
    shapes = [(65, 1, 3),       # 3 items: far below one wave
              (127, 5, 2),
              (128, 24, 12),    # 288 items: more than two waves
              (129, 1, 140),    # 280 items, 1 head, a 1-row last tile
              (255, 5, 3),
              (256, 24, 3),     # 144 items: just over one wave
              (257, 1, 2),
              (602, 5, 12),     # 300 items: the joint attention's length
              (1792, 24, 1)]    # 336 items, 14 key blocks
    cases = []
    for seq, heads, N in shapes:
        # pad37: 37 poisoned rows between input sequences; both outputs have their own stride
        cases.append(("contig_s%d_h%d_n%d" % (seq, heads, N), "tc",
                      lambda s=seq, h=heads, n=N: contiguous(h, n, s, out_pad=9)))
        cases.append(("contig_s%d_h%d_n%d_pad37" % (seq, heads, N), "mma",
                      lambda s=seq, h=heads, n=N: contiguous(h, n, s, pad=37, out_pad=0)))
    for split in (448, 1, 601):     # mid-tile, first token, last token
        cases.append(("joint_split%d" % split, "tc",
                      lambda sp=split: contiguous(3, 3, 602, out_pad=5, split=sp)))
    return cases


def _gathered_cases():
    cases = []
    # (inner, n_out): units per 128-row tile upt = min(128 // inner, n_out)
    shapes = [(12, 6),     # upt 6: 72 rows in the tile
              (12, 11),    # tiles of 10 + 1 units
              (12, 32),    # 32-bit unit masks full; tiles 10 + 10 + 10 + 2
              (20, 4),     # 80 rows
              (20, 7),     # tiles of 6 + 1
              (28, 3),     # 84 rows
              (28, 6),     # the CTSD cross-view sequence: tiles of 4 + 2
              (48, 2),
              (48, 5),     # tiles of 2 + 2 + 1
              (100, 3),    # one unit per tile, 28 empty rows
              (128, 2)]    # one full unit per tile
    masks = ["none", "ones", "diag", "empty"]
    for i, (inner, n_out) in enumerate(shapes):
        mk = masks[i % 4]
        mdiv = 1 if i % 2 else 2     # mask batch = g0 / mask_div (T = 2 frames per batch)

        def cv(inner=inner, n_out=n_out, mk=mk, mdiv=mdiv, i=i):
            BT = 4
            m = None if mk == "none" else unit_mask(mk, BT // mdiv, n_out, seed=i)
            return crossview(2, BT, 3, n_out, inner, unit_pad=5 * (i % 2), group_pad=3,
                             out="seq" if i % 3 == 0 else "same", mask=m, mask_div=mdiv)
        cases.append(("cv_w%d_v%d_%s_div%d" % (inner, n_out, mk, mdiv), "tcg", cv))
    # three group dims (merged), and a unit middle dim, with every mask kind
    for j, (T, W, V, mk) in enumerate([(6, 28, 2, "none"), (5, 20, 3, "empty"),
                                       (4, 48, 1, "diag"), (3, 100, 2, "ones")]):
        def tr(T=T, W=W, V=V, mk=mk, j=j):
            m = None if mk == "none" else unit_mask(mk, 1, T, seed=10 + j)
            return temporal_rowwise(2, 2, T, V, 2, W, group_pad=7, mask=m, mask_div=2,
                                    out="seq" if j % 2 else "same")
        cases.append(("tr_t%d_w%d_v%d_%s" % (T, W, V, mk), "tcg", tr))
    # 33 units: the 32-bit unit masks no longer fit, so this falls back to mma.sync
    cases.append(("cv_w12_v33_empty", "mma",
                  lambda: crossview(2, 2, 2, 33, 12, unit_pad=4,
                                    mask=unit_mask("empty", 2, 33, seed=3))))
    cases.append(("cv_w12_v33_nomask", "mma", lambda: crossview(2, 2, 2, 33, 12)))
    # 4 x 8 sequences x 10 heads x 2 unit tiles = 640 items > 4 x 132: several items per CTA
    cases.append(("cv_w28_v6_persistent", "tcg",
                  lambda: crossview(10, 4, 8, 6, 28, mask=unit_mask("empty", 2, 6, seed=4),
                                    mask_div=2)))
    return cases


def _short_cases():
    cases = []
    for seq in (1, 2, 15, 16, 17, 31, 32, 33, 63, 64):
        cases.append(("short_contig_s%d" % seq, "mma", lambda s=seq: contiguous(2, 3, s, pad=2)))
        cases.append(("short_point_t%d" % seq, "mma",
                      lambda s=seq: pointwise(2, 2, 5, s, group_pad=3)))
    return cases


CASES = _contiguous_cases() + _gathered_cases() + _short_cases()
DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


def _make_qkv(lay, dtype, seed):
    """[n_rows, 3D] view (ld = 3D + LD_PAD) of random q|k|v; rows no position maps to and
    the columns past 3D hold NaN / +-Inf."""
    D = lay.heads * 64
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(lay.n_rows, 3 * D + LD_PAD, generator=g)
    used = torch.zeros(lay.n_rows, dtype=torch.bool)
    used[lay.in_rows.reshape(-1)] = True
    poison = torch.tensor(POISON).repeat(x.shape[1] // 3 + 1)[:x.shape[1]]
    x[~used] = poison
    x[:, 3 * D:] = poison[:LD_PAD]
    return x.to(dtype).cuda()[:, :3 * D]


def _launch(lay, qkv, dtype, tc):
    """One call into sentinel-filled buffers; returns (buf, buf2) including the guard bands.
    Text layouts pass scale / causal / bias through lay.kwargs()."""
    from opendwm_b200 import lib, ops
    D = lay.heads * 64

    def buffer(rows):
        return torch.full((rows + 2 * GUARD, D + LDO_PAD), SENTINEL, dtype=torch.int16,
                          device="cuda").view(dtype)
    buf = buffer(int(lay.out_rows.max()) + 1)
    buf2 = buffer(lay.G * (lay.seq - lay.split)) if lay.split else None
    lib.set_option("attn_tc", tc)
    try:
        ops.attention(qkv, buf[GUARD:-GUARD, :D], D=D,
                      out2=None if buf2 is None else buf2[GUARD:-GUARD, :D], **lay.kwargs())
        torch.cuda.synchronize()
    finally:
        lib.set_option("attn_tc", -1)
    return buf, buf2


def _written(buf, rows, D):
    w = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    w[(rows.reshape(-1) + GUARD).to(buf.device), :D] = True
    return w


def _check(lay, bufs, ref, pv, u, what, vs=None):
    """Sentinel bits outside the write set; finite values within the bound inside it."""
    D = lay.heads * 64
    buf, buf2 = bufs
    n_main = lay.split if lay.split else lay.seq
    got = torch.empty(lay.G, lay.seq, D, dtype=buf.dtype, device=buf.device)
    pairs = [(buf, lay.out_rows, slice(0, n_main))]
    if lay.split:
        pairs.append((buf2, lay.out2_rows, slice(lay.split, lay.seq)))
    for b, rows, js in pairs:
        w = _written(b, rows, D)
        stray = b.view(torch.int16)[~w] != SENTINEL
        assert not stray.any(), "%s: %d element(s) written outside the output" % (what, stray.sum())
        got[:, js] = b[(rows + GUARD).to(b.device)][..., :D]
    bad, worst = bound_violations(got, ref, pv, u, vs)
    if bad.any():
        g, j, d = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(
            "%s: %d of %d outside the float64 bound (worst ratio %.3g, non-finite %d); first at "
            "group %d position %d col %d: got %r ref %r" % (
                what, bad.sum(), bad.numel(), worst, (~torch.isfinite(got)).sum(), g, j, d,
                got[g, j, d].item(), ref[g, j, d].item()))
    return worst


def _reference(lay, qkv):
    """float64 (ref, P|V|, sum|v|) as [G, seq, D], computed a few groups at a time."""
    mask = lay.mask_bool()
    step = max(1, (1 << 25) // (lay.heads * lay.seq * lay.seq))
    outs = []
    for g0 in range(0, lay.G, step):
        q, k, v = gather_qkv(qkv, lay.in_rows[g0:g0 + step], lay.heads)
        outs.append(reference(q, k, v, lay.scale, None if mask is None else mask[g0:g0 + step],
                              lay.causal, lay.bias))
    flat = lambda t: torch.cat(t).transpose(1, 2).reshape(lay.G, lay.seq, -1)  # noqa: E731
    return tuple(flat([o[i] for o in outs]) for i in range(3))


def _conform(lay, qkv, dtype, distinct=True):
    """Both kernels against float64, the dispatch check and the repeat; returns the worst
    bound ratio of each run."""
    u = unit_roundoff(dtype)
    ref, pv, vs = _reference(lay, qkv)
    # the text kernel's fp16 P underflows for most keys (see bound_violations); elsewhere the
    # bound stays as it was measured
    vs = vs if lay.text else None
    path = lay.kernel_path()
    b0 = _launch(lay, qkv, dtype, 0)
    b2 = _launch(lay, qkv, dtype, 2)
    b2r = _launch(lay, qkv, dtype, 2)
    r0 = _check(lay, b0, ref, pv, u, "attn_tc=0 (%s)" % ("text" if lay.text else "mma.sync"), vs)
    r2 = _check(lay, b2, ref, pv, u, "attn_tc=2 (%s)" % path, vs)
    bits = lambda b: [x.view(torch.int16) for x in b if x is not None]  # noqa: E731
    assert all(torch.equal(x, y) for x, y in zip(bits(b2), bits(b2r))), "not repeatable"
    same = all(torch.equal(x, y) for x, y in zip(bits(b0), bits(b2)))
    if path == "text":
        assert same, "causal / biased attention gave other bits under attn_tc=0 and attn_tc=2"
    elif path == "mma":
        assert same, "the layout is not wgmma-eligible, yet attn_tc=2 ran another kernel"
    elif distinct and lay.G * lay.seq * lay.heads * 64 >= 64 * 64:
        assert not same, ("the layout is %s-eligible, yet attn_tc=2 gave the mma.sync kernel's "
                          "bits: the wgmma kernel never ran" % path)
    return r0, r2


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,path,make", CASES, ids=[c[0] for c in CASES])
def test_attention_conforms(name, path, make, dtype):
    """`path` is the kernel the case is meant to exercise under attn_tc >= 1."""
    lay = make()
    assert lay.kernel_path() == path
    _conform(lay, _make_qkv(lay, dtype, seed=lay.seq), dtype)


EXTREMES = ["uniform", "dominant", "zero_q", "pm80"]


def _extreme(qkv, lay, kind):
    """Rewrites the q / k columns of the rows the layout reads:
    uniform: every key equal (uniform P); dominant: one key per sequence wins by 2^20 in the
    logit; zero_q: all queries 0 (uniform P); pm80: scaled logits near +80 or -80, so exp of
    the losers underflows even in fp32."""
    D = lay.heads * 64
    rows = lay.in_rows.to(qkv.device)
    g = torch.Generator(device=qkv.device).manual_seed(5)
    if kind == "uniform":
        qkv[rows.reshape(-1), D:2 * D] = qkv[rows[0, 0], D:2 * D]
    elif kind == "dominant":
        c = torch.arange(lay.heads, device=qkv.device) * 64
        qkv[rows.reshape(-1)[:, None], c] = 2.0 ** 12
        qkv[rows.reshape(-1)[:, None], D + c] = 0.0
        qkv[rows[:, (2 * lay.seq) // 3][:, None], D + c] = 2.0 ** 11     # 2^23 / 8 = 2^20
    elif kind == "zero_q":
        qkv[rows.reshape(-1), :D] = 0.0
    else:
        a = math.sqrt(80 / 0.125)
        n = rows.numel()
        for cols in (slice(0, D), slice(D, 2 * D)):
            x = 0.05 * torch.randn(n, D, generator=g, device=qkv.device)
            sign = torch.randint(0, 2, (n, lay.heads), generator=g, device=qkv.device) * 2 - 1
            x.view(n, lay.heads, 64)[:, :, 0] = a * sign
            qkv[rows.reshape(-1), cols] = x.to(qkv.dtype)
    return qkv


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("kind", EXTREMES)
@pytest.mark.parametrize("layout", ["contig", "gathered"])
def test_attention_logit_extremes(layout, kind, dtype):
    """Both kernels on each wgmma path.  One-hot and near-uniform P can give the same bits on
    every kernel, so the bits are not required to differ here: the random-data cases of
    test_attention_conforms show that both paths reach the wgmma kernel."""
    if layout == "contig":
        lay = contiguous(2, 2, 257)
    else:
        lay = crossview(2, 2, 2, 6, 28, mask=unit_mask("diag", 2, 6, seed=6))
    assert lay.kernel_path() == ("tc" if layout == "contig" else "tcg")
    qkv = _extreme(_make_qkv(lay, dtype, seed=9), lay, kind)
    _conform(lay, qkv, dtype, distinct=False)


# --------------------------------------------------------------------------------------------
# text encoders: causal (CLIP) and biased (T5) attention on contiguous sequences
# --------------------------------------------------------------------------------------------
TEXT_SEQS = [1, 63, 64, 65, 77, 127, 128, 129, 300]
TEXT_HEADS = [12, 20, 64]


def _text_bias(heads, seq, seed, std=3.0):
    return torch.randn(heads, seq, seq, generator=torch.Generator().manual_seed(seed)) * std


def _text_layout(mode, seq, heads, G, seed, out_pad=None):
    """`mode` "causal" (CLIP, scale 1/8) or "bias" (T5: unscaled, but scale 1/8 at 20 heads so
    that a kernel scaling the bias too is caught)."""
    if mode == "causal":
        return contiguous(heads, G, seq, out_pad=out_pad, causal=True)
    return contiguous(heads, G, seq, out_pad=out_pad, scale=0.125 if heads == 20 else 1.0,
                      bias=_text_bias(heads, seq, seed))


def _text_cases():
    cases = []
    for mode in ("causal", "bias"):
        for seq in TEXT_SEQS:
            for heads in TEXT_HEADS:
                cases.append(("%s_s%d_h%d_g3" % (mode, seq, heads), mode, seq, heads, 3))
        # a CFG window's prompt batch: 192 prompts of 77 tokens, several waves of 128-row
        # tiles that straddle the sequences
        for heads in (12, 20):
            cases.append(("%s_s77_h%d_g192" % (mode, heads), mode, 77, heads, 192))
    return cases


TEXT_CASES = _text_cases()


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,mode,seq,heads,G", TEXT_CASES, ids=[c[0] for c in TEXT_CASES])
def test_text_attention_conforms(name, mode, seq, heads, G, dtype):
    """q|k|v with ld = 3D + 8 poisoned columns and poisoned rows after the last sequence; the
    cases with an odd seq + heads write their sequences 3 rows apart (sentinel rows between)."""
    lay = _text_layout(mode, seq, heads, G, seed=seq * 131 + heads,
                       out_pad=3 if (seq + heads) % 2 else None)
    assert lay.kernel_path() == "text"
    r0, r2 = _conform(lay, _make_qkv(lay, dtype, seed=seq + heads), dtype)
    print("BOUND_RATIO attention_text %s_%s %.4g" % (name, dtype, max(r0, r2)))


def _text_extreme(lay, qkv, kind):
    """The EXTREMES on the text path.  Causal: as `_extreme` makes them.  Bias (unscaled, as in
    T5): the bias carries the extreme where it can: "dominant" adds 2^20 to one key of every
    row, "pm80" makes every logit bias +-80 (the losers' exp underflows fp32), "uniform" and
    "zero_q" keep a bias that is constant along each row (uniform P) or only the bias (zero q).
    "pad_mask" adds -1e9, as a padding mask does, to every fifth key and the last 7 keys of each
    row: their P must be exactly 0.  A row whose every key is so masked would be a uniform
    softmax in float64 and is out of scope."""
    H, S = lay.heads, lay.seq
    g = torch.Generator().manual_seed(17)
    if lay.causal:
        return lay, _extreme(qkv, lay, kind)
    b = _text_bias(H, S, seed=S)
    if kind in ("uniform", "zero_q"):
        qkv = _extreme(qkv, lay, kind)
        b = b[:, :, :1].expand(H, S, S).contiguous() if kind == "uniform" else b
    elif kind == "dominant":
        b[:, :, (2 * S) // 3] = 2.0 ** 20
    elif kind == "pm80":
        b = 80.0 * (torch.randint(0, 2, (H, S, S), generator=g) * 2 - 1) + 0.5 * torch.randn(H, S, S, generator=g)
    else:
        j = torch.arange(S)
        b[:, :, (j % 5 == 0) | (j >= S - 7)] = -1e9
    lay.bias = b
    return lay, qkv


TEXT_EXTREMES = [("causal", k) for k in EXTREMES] + [("bias", k) for k in EXTREMES + ["pad_mask"]]


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("mode,kind", TEXT_EXTREMES, ids=["%s_%s" % c for c in TEXT_EXTREMES])
def test_text_attention_logit_extremes(mode, kind, dtype):
    """3 sequences of 129 tokens (a 1-row second tile), 4 heads, T5's scale 1 for the bias; the
    padding mask is a bias, so it has no causal case."""
    lay = contiguous(4, 3, 129, causal=mode == "causal", scale=0.125 if mode == "causal" else 1.0,
                     bias=None if mode == "causal" else torch.zeros(4, 129, 129))
    lay, qkv = _text_extreme(lay, _make_qkv(lay, dtype, seed=21), kind)
    r0, r2 = _conform(lay, qkv, dtype, distinct=False)
    print("BOUND_RATIO attention_text_extremes %s_%s_%s %.4g" % (mode, kind, dtype, max(r0, r2)))


def _attn_launched(fn):
    """(T, G, SKV, CAUSAL, BIAS) of every attn_wgmma_kernel `fn` launches, in order."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    found = []
    for ev in prof.events():
        m = re.search(r"attn_wgmma_kernel<(.*)>", ev.name)
        if m:
            args = [re.sub(r"^\((int|bool)\)", "", a.strip()) for a in m.group(1).split(",")]
            found.append((args[0].split("::")[-1],) + tuple(a in ("true", "1") for a in args[1:5]))
    return found


@pytest.mark.gpu
def test_text_attention_selection():
    """check_text_attention_selection, in a process of its own (run_isolated)."""
    run_isolated("test_attention_conformance_gpu", "check_text_attention_selection")


def check_text_attention_selection():
    """Causal and biased calls launch attn_wgmma_kernel<T, false, false, CAUSAL, BIAS> with the
    flags of the call, in both dtypes, under every attn_tc setting, at a short sequence (which
    the plain path would send to mma.sync) and a long one."""
    from opendwm_b200 import lib, ops
    for dtype, tname in ((torch.bfloat16, "__nv_bfloat16"), (torch.float16, "__half")):
        for seq in (63, 129):
            qkv = torch.randn(2 * seq, 3 * 128, device="cuda").to(dtype)
            out = torch.empty(2 * seq, 128, device="cuda", dtype=dtype)
            kw = dict(D=128, heads=2, group_dims=[2], group_strides=[seq], seq=seq)
            for causal in (True, False):
                bias = None if causal else torch.zeros(2, seq, seq, device="cuda")
                for tc in (-1, 0, 2):
                    lib.set_option("attn_tc", tc)
                    try:
                        got = _attn_launched(lambda: ops.attention(qkv, out, causal=causal, bias=bias, **kw))
                    finally:
                        lib.set_option("attn_tc", -1)
                    want = [(tname, False, False, causal, not causal)]
                    assert got == want, ((dtype, seq, causal, tc), got, want)


@pytest.mark.gpu
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
