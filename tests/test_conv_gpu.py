"""Parity of the im2col-free wgmma convolution against torch conv3d (fp32) on the same
16-bit inputs: CogVideoX causal 3x3x3, per-frame 1x3x3, 3x3 adapter conv, ragged tiles."""
import pytest
import torch

pytestmark = pytest.mark.gpu
_LAST = [None]      # output of the most recent _case (kernel-variant comparisons)


def _case(nb, t_out, h, w, cin, cout, kernel, dtype, epilogue="f32", seed=0):
    from opendwm_b200 import ops, lib
    kt, kh, kw = kernel
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(nb, cin, t_out + kt - 1, h, w, generator=g).to(dtype).cuda()   # NCTHW, time-padded
    wt = (torch.randn(cout, cin, kt, kh, kw, generator=g) * (cin * kt * kh * kw) ** -0.5).to(dtype).cuda()
    b = torch.randn(cout, generator=g).cuda()
    ref = torch.nn.functional.conv3d(x.float(), wt.float(), b, padding=(0, kh // 2, kw // 2))
    ref = ref.permute(0, 2, 3, 4, 1).reshape(-1, cout)                              # channels-last rows
    cin_p = (cin + 7) // 8 * 8
    cout_p = (cout + 31) // 32 * 32
    xcl = torch.zeros(nb, t_out + kt - 1, h, w, cin_p, dtype=dtype, device="cuda")
    xcl[..., :cin] = x.permute(0, 2, 3, 4, 1)
    wp = ops.pack_conv_weight(wt, dtype, pad_out_to=cout_p, pad_in_to=cin_p)
    bp = torch.zeros(cout_p, device="cuda")
    bp[:cout] = b
    if epilogue == "f32":
        y = ops.conv(xcl, wp, bp, kernel=kernel, epilogue=lib.EPI_F32)[:, :cout]
    elif epilogue == "resid":
        r = torch.randn(ref.shape[0], cout_p, generator=g).cuda()
        y = ops.conv(xcl, wp, bp, kernel=kernel, epilogue=lib.EPI_RESID, resid=r)[:, :cout]
        ref = ref + r[:, :cout]
    else:
        y = ops.conv(xcl, wp, bp, kernel=kernel, epilogue=lib.EPI_STORE, act=lib.ACT_SILU)[:, :cout].float()
        ref = torch.nn.functional.silu(ref)
    _LAST[0] = y
    return ((y - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_causal_conv3d_3x3x3(dtype):
    assert _case(2, 3, 8, 14, 64, 256, (3, 3, 3), dtype) < 2e-5 * 50


@pytest.mark.parametrize("shape", [
    (1, 2, 32, 56, 128, 128, (3, 3, 3)),    # bw 56, bh 2
    (1, 1, 16, 112, 64, 128, (1, 3, 3)),    # bw 112
    (1, 1, 6, 224, 64, 256, (1, 3, 3)),     # W > 128: ragged second tile
    (2, 1, 16, 28, 192, 512, (1, 3, 3)),    # adapter-like, 2 N tiles
    (1, 2, 5, 9, 16, 32, (3, 3, 3)),        # tiny ragged, C_in padded... c_out 32
    (1, 1, 7, 130, 72, 3, (1, 3, 3)),       # conv_out-like: C_out 3 padded to 32
    (3, 1, 4, 4, 64, 128, (1, 1, 1)),       # 1x1x1
    (2, 1, 8, 14, 64, 320, (1, 3, 3)),      # UNet widths: 5 tiles of 64
    (1, 1, 8, 14, 320, 640, (1, 3, 3)),     # 5 tiles of 128, C_in 320 = 5 k-blocks
    (1, 1, 4, 7, 128, 1280, (1, 3, 3)),     # 5 tiles of 256
    (2, 4, 1, 112, 64, 128, (3, 1, 1)),     # temporal ResBlock conv: 3 frame taps, no padding
])
def test_shapes(shape):
    err = _case(*shape, torch.bfloat16)
    assert err < 1e-3, err


def test_epilogues():
    assert _case(1, 2, 16, 56, 128, 256, (3, 3, 3), torch.bfloat16, "resid") < 1e-3
    assert _case(1, 2, 16, 56, 128, 128, (3, 3, 3), torch.bfloat16, "store") < 8e-3


def test_per_item_residual():
    """conv + bias + one residual row per item (ResnetBlock2D temb add)."""
    from opendwm_b200 import ops, lib
    nb, h, w, cin, cout = 3, 8, 14, 64, 128
    g = torch.Generator().manual_seed(0)
    x = torch.randn(nb, 1, h, w, cin, generator=g).bfloat16().cuda()
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).bfloat16().cuda()
    b = torch.randn(cout, generator=g).cuda()
    temb = torch.randn(nb, cout, generator=g).cuda()
    y = ops.conv(x, ops.pack_conv_weight(wt, torch.bfloat16), b, kernel=(1, 3, 3),
                 epilogue=lib.EPI_RESID, resid=temb, resid_rows_per_item=h * w)
    ref = torch.nn.functional.conv2d(x[:, 0].permute(0, 3, 1, 2).float(), wt.float(), b, padding=1)
    ref = ref + temb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(-1, cout)
    assert ((y - ref).abs().max() / ref.abs().max()).item() < 1e-3


@pytest.mark.parametrize("epilogue", ["f32", "resid", "store"])
@pytest.mark.parametrize("shape", [
    (2, 3, 64, 96, 64, 128, (3, 3, 3)),     # 384 pixel tiles: C_out 128 (the smem-bound width)
    (1, 2, 150, 128, 64, 256, (1, 3, 3)),   # 300 tiles, C_out 256
    (3, 1, 101, 120, 72, 64, (1, 3, 3)),    # 303 tiles (odd: dummy last tile), C_out 64
    (1, 1, 299, 130, 128, 320, (1, 3, 3)),  # ragged W tiles, 5 N tiles of 64
])
def test_two_cta_conv_equals_one_cta(shape, epilogue):
    """Enough pixel tiles (>= 2 x SMs) route the convolution to the kernel for clusters of two
    CTAs (two pixel tiles sharing each weight slice, half of it loaded by each CTA and
    multicast); it must agree with the 1-CTA kernel bit for bit (same accumulation order) and
    with torch."""
    from opendwm_b200 import lib
    lib.set_option("conv_2cta", 1)
    lib.set_option("conv_halo", 0)       # the per-tap pair kernel, not the halo-row one
    try:
        e2 = _case(*shape, torch.float16, epilogue, seed=3)
        y2 = _LAST[0].clone()
        lib.set_option("conv_2cta", 0)
        e1 = _case(*shape, torch.float16, epilogue, seed=3)
        y1 = _LAST[0]
    finally:
        lib.set_option("conv_2cta", 1)
        lib.set_option("conv_halo", 1)
    assert e2 < (8e-3 if epilogue == "store" else 1e-3), e2
    assert e1 < (8e-3 if epilogue == "store" else 1e-3), e1
    assert torch.equal(y1, y2)


@pytest.mark.parametrize("epilogue", ["f32", "resid", "store"])
@pytest.mark.parametrize("shape", [
    (2, 1, 160, 200, 64, 128, (1, 3, 3)),    # W = 200: one full + one ragged 72-pixel segment
    (1, 3, 64, 130, 128, 128, (3, 3, 3)),    # causal 3x3x3, second segment holds 2 pixels
    (1, 1, 300, 128, 72, 64, (1, 3, 3)),     # C_out 64, partial second C_in block
    (3, 1, 101, 448, 128, 128, (1, 3, 3)),   # VAE width 448 (3.5 segments), odd tile count
])
def test_halo_row_conv_equals_shifted_patch_kernels(shape, epilogue):
    """kw = 3, W >= 128, C_out tiles <= 128: the halo-row kernel loads each 130-pixel row
    segment once and feeds the three dw taps through row-shifted wgmma descriptors; it must
    match torch and the per-tap kernels (different tap order: agreement to rounding)."""
    from opendwm_b200 import lib
    tol = 8e-3 if epilogue == "store" else 1e-3
    lib.set_option("conv_halo", 1)
    try:
        eh = _case(*shape, torch.float16, epilogue, seed=11)
        yh = _LAST[0].float().clone()
        lib.set_option("conv_halo", 0)
        e2 = _case(*shape, torch.float16, epilogue, seed=11)
        y2 = _LAST[0].float()
    finally:
        lib.set_option("conv_halo", 1)
    assert eh < tol and e2 < tol, (eh, e2)
    assert ((yh - y2).abs().max() / y2.abs().max()).item() < (2e-3 if epilogue == "store" else 2e-5)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C", [320, 640])
@pytest.mark.parametrize("S", [112, 1792])
def test_temporal_resblock_convs(S, C, dtype):
    """The two (3,1,1) convolutions of the UNet TemporalResnetBlock on `(b v)` volumes
    [B*V, T+2, 1, S, C] with a zero frame at both ends: (i) + one temb row per (b, v, t) item;
    (ii) + the block input as residual, then the AlphaBlender against that same tensor,
    out = alpha[b] * x + (1 - alpha[b]) * (conv + bias + x).  S = 1792 (SD-2.1 level 0 at
    256 x 448) has enough pixel tiles for the 2-CTA kernel, which must give the bits of the
    1-CTA kernel."""
    from opendwm_b200 import ops, lib
    B, V, T = 2, 3, 8
    g = torch.Generator().manual_seed(S + C)
    x = torch.zeros(B * V, T + 2, 1, S, C, dtype=dtype, device="cuda")
    x[:, 1:T + 1] = torch.randn(B * V, T, 1, S, C, generator=g).to(dtype).cuda()
    wt = (torch.randn(C, C, 3, 1, 1, generator=g) * (3 * C) ** -0.5).to(dtype).cuda()
    b = torch.randn(C, generator=g).cuda()
    temb = torch.randn(B * V * T, C, generator=g).cuda()
    xr = torch.randn(B * V * T * S, C, generator=g).cuda()
    alpha = torch.tensor([0.3, 0.8], device="cuda")
    conv = torch.nn.functional.conv3d(x.float().permute(0, 4, 1, 2, 3), wt.float(), b)
    conv = conv.permute(0, 2, 3, 4, 1).reshape(-1, C)               # rows (b v, t, s)
    ref1 = conv + temb.repeat_interleave(S, 0)
    a = alpha.repeat_interleave(V * T * S)[:, None]
    ref2 = a * xr + (1 - a) * (conv + xr)
    wp = ops.pack_conv_weight(wt, dtype)
    outs = {}
    try:
        for two in (1, 0):
            lib.set_option("conv_2cta", two)
            y1 = ops.conv(x, wp, b, kernel=(3, 1, 1), epilogue=lib.EPI_RESID, resid=temb,
                          resid_rows_per_item=S)
            y2 = ops.conv(x, wp, b, kernel=(3, 1, 1), epilogue=lib.EPI_RESID, resid=xr,
                          blend_x=xr, alpha=alpha, rows_per_batch=V * T * S)
            outs[two] = (y1, y2)
    finally:
        lib.set_option("conv_2cta", 1)
    for name, y, ref in zip(("temb", "blend"), outs[1], (ref1, ref2)):
        err = ((y - ref).abs().max() / ref.abs().max()).item()
        assert err < 1e-3, (name, err)
    for y2, y1 in zip(outs[1], outs[0]):
        assert torch.equal(y2, y1)
