"""The opt-in FP8 (E4M3) path of the CTSD-2.1 UNet on the GPU: the implicit-GEMM convolution
with per-volume activation scales against float64 on the dequantized operands, its kernel
variants, the E4M3 GroupNorm+SiLU against float64, the loud errors, and the UNet with
gemm_dtype=torch.float8_e4m3fn against the fake-quant oracle, under CUDA graphs and through a
pipeline config."""
import ctypes

import pytest
import torch

import fp8_emulation as fe
import fp8_unet_emulation as fue

pytestmark = pytest.mark.gpu
F8 = torch.float8_e4m3fn


def acc_tol(K):
    """DESIGN §7's bound on the Hopper FP8 accumulation error (max|d| / max|ref| against
    float64 on the dequantized operands), K = taps * C_in."""
    return 2e-4 + 2e-6 * K


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _vol_scaled(shape, seed):
    """fp32 [nb, ...] with volume n scaled by 10^n (a wrong volume scale fails)."""
    x = torch.randn(shape, generator=_gen(seed))
    x *= torch.pow(10.0, torch.arange(shape[0], dtype=torch.float32)).view(-1, *[1] * (len(shape) - 1))
    return x.cuda()


def _quant_volumes(x):
    q, s = fe.quantize_rows(x.reshape(x.shape[0], -1))
    return q.view(x.shape).contiguous(), s.contiguous()


def _conv_ref(q8, sa, w8, sw, kernel):
    """float64 convolution of the dequantized operands -> rows [nb*t_out*h*w, c_out]."""
    kt, kh, kw = kernel
    nb, tp, h, w, c_in = q8.shape
    taps, c_out, _ = w8.shape
    x = q8.double() * sa.double().view(-1, 1, 1, 1, 1)
    wt = (w8.double() * sw.double().view(1, -1, 1)).view(kt, kh, kw, c_out, c_in)\
        .permute(3, 4, 0, 1, 2)
    y = torch.nn.functional.conv3d(x.permute(0, 4, 1, 2, 3), wt, padding=(0, kh // 2, kw // 2))
    return y.permute(0, 2, 3, 4, 1).reshape(-1, c_out)


def _per_volume_err(y, ref, nb):
    y, ref = y.double().view(nb, -1), ref.view(nb, -1)
    return max(((y[n] - ref[n]).abs().max() / ref[n].abs().max()).item() for n in range(nb))


# kernel, C_in, C_out (tile 64 / 256 / 128 / 32), nb, frames (T, or tp = T + 2 for (3,1,1)),
# H, W (>= 128: halo-row kernel, < 128: pixel patches), residual mode
CONV_CASES = [
    ((1, 3, 3), 320, 320, 3, 1, 8, 160, "none"),
    ((1, 3, 3), 640, 512, 3, 1, 16, 40, "item"),
    ((1, 3, 3), 960, 384, 3, 1, 8, 136, "none"),
    ((1, 3, 3), 1280, 96, 4, 1, 6, 10, "item"),
    ((1, 3, 3), 320, 320, 12, 1, 32, 56, "item"),
    ((3, 1, 1), 320, 320, 3, 6, 1, 112, "item"),
    ((3, 1, 1), 640, 640, 4, 5, 1, 56, "blend"),
    ((3, 1, 1), 1280, 1280, 4, 4, 1, 24, "blend"),
]


def _conv_case(kernel, c_in, c_out, nb, tp, h, w, mode, seed=0):
    from opendwm_b200 import ops
    kt, kh, kw = kernel
    q8, sa = _quant_volumes(_vol_scaled((nb, tp, h, w, c_in), seed))
    wt = torch.randn(c_out, c_in, kt, kh, kw, generator=_gen(seed + 1)) * (kt * kh * kw * c_in) ** -0.5
    w8, sw = ops.pack_conv_weight_fp8(wt.cuda())
    bias = (0.1 * torch.randn(c_out, generator=_gen(seed + 2))).cuda()
    t_out = tp - kt + 1
    rows = nb * t_out * h * w
    vol = torch.pow(10.0, torch.arange(nb, dtype=torch.float64)).cuda()
    kw_args, extra = {}, None
    if mode == "item":      # one residual row per item (frame) of h*w pixels
        r = torch.randn(nb * t_out, c_out, generator=_gen(seed + 3)).cuda() * \
            vol.float().repeat_interleave(t_out)[:, None]
        kw_args = dict(resid=r, resid_rows_per_item=h * w)
        extra = r.double().repeat_interleave(h * w, 0)
    elif mode == "blend":   # AlphaBlender with blend_x the residual, two batches
        r = torch.randn(rows, c_out, generator=_gen(seed + 3)).cuda() * \
            vol.float().repeat_interleave(rows // nb)[:, None]
        alpha = torch.tensor([0.3, 0.8]).cuda()
        kw_args = dict(resid=r, blend_x=r, alpha=alpha, rows_per_batch=rows // 2)
        extra = (r.double(), alpha.double().repeat_interleave(rows // 2)[:, None])
    return q8, sa, w8, sw, bias, kw_args, extra


def _run_conv(q8, sa, w8, sw, bias, kernel, kw_args):
    from opendwm_b200 import lib, ops
    return ops.conv(q8, w8, bias, kernel=kernel, epilogue=lib.EPI_RESID, a_scale=sa, w_scale=sw,
                    **kw_args)


@pytest.mark.parametrize("kernel,c_in,c_out,nb,tp,h,w,mode", CONV_CASES)
def test_fp8_conv_against_float64(kernel, c_in, c_out, nb, tp, h, w, mode):
    q8, sa, w8, sw, bias, kw_args, extra = _conv_case(kernel, c_in, c_out, nb, tp, h, w, mode)
    ref = _conv_ref(q8, sa, w8, sw, kernel) + bias.double()
    if mode == "item":
        ref = ref + extra
    elif mode == "blend":
        r, al = extra
        ref = al * r + (1 - al) * (ref + r)
    y = _run_conv(q8, sa, w8, sw, bias, kernel, kw_args)
    K = kernel[0] * kernel[1] * kernel[2] * c_in
    err = _per_volume_err(y, ref, nb)
    print("fp8 conv", kernel, c_in, c_out, nb, tp, h, w, mode, "worst per-volume rel err", err)
    assert err < acc_tol(K), (err, acc_tol(K))


# halo-row kernel (64 / 128 columns), 2-CTA pairs at 64 / 256 / 128 columns (the last one a
# temporal (3,1,1) conv with the AlphaBlender)
VARIANT_CASES = [CONV_CASES[0], CONV_CASES[2], CONV_CASES[4],
                 ((1, 3, 3), 640, 512, 12, 1, 32, 56, "item"),
                 ((3, 1, 1), 640, 640, 4, 10, 1, 512, "blend")]


@pytest.mark.parametrize("kernel,c_in,c_out,nb,tp,h,w,mode", VARIANT_CASES)
def test_fp8_conv_kernel_variants(kernel, c_in, c_out, nb, tp, h, w, mode):
    """conv_2cta 0 / 1 give identical bits (same accumulation order).  The halo-row kernel
    accumulates the dw taps in another order (inside each C_in block), so conv_halo 0 / 1
    agree to the FP8 accumulation bound, as they agree to rounding in 16 bit
    (test_conv_gpu.py)."""
    from opendwm_b200 import lib
    q8, sa, w8, sw, bias, kw_args, _ = _conv_case(kernel, c_in, c_out, nb, tp, h, w, mode)
    outs = {}
    try:
        for pair in (0, 1):
            for halo in (0, 1):
                lib.set_option("conv_2cta", pair)
                lib.set_option("conv_halo", halo)
                args = dict(kw_args)
                if mode == "blend":   # in place over a copy, as the model does
                    r = kw_args["resid"].clone()
                    args.update(resid=r, blend_x=r)
                outs[pair, halo] = _run_conv(q8, sa, w8, sw, bias, kernel, args).clone()
    finally:
        lib.set_option("conv_2cta", -1)
        lib.set_option("conv_halo", -1)
    for halo in (0, 1):
        assert torch.equal(outs[1, halo], outs[0, halo]), halo
    K = kernel[0] * kernel[1] * kernel[2] * c_in
    ref = outs[0, 0].double()
    assert _per_volume_err(outs[0, 1], ref, nb) < acc_tol(K)


# ------------------------------------------------------------------ E4M3 GroupNorm + SiLU
def _gn_ref(x, gamma, beta, groups, eps, silu):
    nb, T, H, W, C = x.shape
    xd = x.double()
    g = xd.view(nb, T * H * W, groups, C // groups)
    mean = g.mean(dim=(1, 3), keepdim=True)
    var = g.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((g - mean) / torch.sqrt(var + eps)).view(nb, T, H, W, C) * gamma.double() + beta.double()
    return torch.nn.functional.silu(y) if silu else y


@pytest.mark.parametrize("silu", [True, False])
@pytest.mark.parametrize("C,T,H,W,out_t0,extra", [(320, 1, 16, 24, 0, 0), (640, 4, 1, 112, 1, 2),
                                                   (1280, 3, 4, 6, 1, 2), (96, 2, 8, 8, 0, 1)])
def test_groupnorm_silu_e4m3(C, T, H, W, out_t0, extra, silu):
    from opendwm_b200 import ops
    nb, eps = 4, 1e-5
    x = _vol_scaled((nb, T, H, W, C), C) + 0.5
    x[2] = 0.0                                  # an all-zero volume (beta = 0 below for it)
    gamma = (1 + 0.1 * torch.randn(C, generator=_gen(1))).cuda()
    beta = (0.05 * torch.randn(C, generator=_gen(2))).cuda()
    ref = _gn_ref(x, gamma, beta, 32, eps, silu)
    out_T = T + extra
    out = torch.full((nb, out_T, H, W, C), 0x7E, dtype=torch.uint8).cuda().view(F8)   # sentinels
    scale = torch.full((nb,), -1.0).cuda()
    sums = ops.groupnorm_stats(x, 32)
    ops.groupnorm_silu_e4m3(x, sums, gamma, beta, out, scale, groups=32, eps=eps, out_t0=out_t0,
                            silu=silu)
    bytes_ = out.view(torch.uint8)
    keep = torch.ones(out_T, dtype=torch.bool)
    keep[out_t0:out_t0 + T] = False
    assert (bytes_[:, keep] == 0x7E).all(), "frames outside the window were written"
    q = out[:, out_t0:out_t0 + T]
    amax = ref.abs().reshape(nb, -1).amax(dim=1)
    for n in range(nb):
        if amax[n] == 0:
            continue
        s = scale[n].double()
        assert abs(s / (amax[n] / 448) - 1) < 1e-6, (n, s.item(), amax[n].item())
        xh = q[n].double() * s
        bound = 2.0 ** -4 * ref[n].abs() + 2.0 ** -10 * s + 1e-6 * amax[n]
        assert ((xh - ref[n]).abs() <= bound).all(), n
    # all-zero volume: GroupNorm of zeros is beta, so with beta = 0 and silu(0) = 0 it is zero
    z = torch.zeros(nb, T, H, W, C).cuda()
    sz = ops.groupnorm_stats(z, 32)
    out.view(torch.uint8).fill_(0x7E)
    ops.groupnorm_silu_e4m3(z, sz, gamma, torch.zeros_like(beta), out, scale, groups=32, eps=eps,
                            out_t0=out_t0, silu=silu)
    assert (scale == 1).all()
    assert (out.view(torch.uint8)[:, out_t0:out_t0 + T] == 0).all()


# ------------------------------------------------------------------ loud errors
def test_errors_are_loud():
    from opendwm_b200 import lib, ops
    q8, sa, w8, sw, bias, _, _ = _conv_case((1, 3, 3), 320, 64, 2, 1, 4, 8, "none")
    with pytest.raises(ValueError, match="a_scale and w_scale"):
        ops.conv(q8, w8, bias, kernel=(1, 3, 3), epilogue=lib.EPI_RESID, a_scale=sa)
    with pytest.raises(ValueError, match="RESID"):
        ops.conv(q8, w8, bias, kernel=(1, 3, 3), epilogue=lib.EPI_F32, a_scale=sa, w_scale=sw)
    with pytest.raises(ValueError, match="a_scale"):
        ops.conv(q8, w8, bias, kernel=(1, 3, 3), epilogue=lib.EPI_RESID, a_scale=sa[:1], w_scale=sw)
    # C_in % 16 != 0 reaches the C layer
    x24 = torch.zeros(2, 1, 4, 8, 24, device="cuda", dtype=F8)
    w24 = torch.zeros(9, 64, 24, device="cuda", dtype=F8)
    with pytest.raises(RuntimeError, match="C_in % 16"):
        ops.conv(x24, w24, bias, kernel=(1, 3, 3), epilogue=lib.EPI_RESID, a_scale=sa, w_scale=sw)

    # the C ABI checks on its own: missing scales, a non-RESID epilogue
    def raw(epilogue, a_scale, w_scale):
        a = lib.ConvArgs()
        a.x, a.nb, a.tp, a.h, a.w, a.c_in = q8.data_ptr(), 2, 1, 4, 8, 320
        a.weight, a.kt, a.kh, a.kw, a.c_out = w8.data_ptr(), 1, 3, 3, 64
        out = torch.empty(64, 64, device="cuda")
        a.dtype, a.epilogue, a.out, a.ldo = lib.DWM_E4M3, epilogue, out.data_ptr(), 64
        a.a_scale, a.w_scale = a_scale, w_scale
        rc = lib.load().dwm_b200_conv(ctypes.byref(a), torch.cuda.current_stream().cuda_stream)
        lib.check(rc, "dwm_b200_conv")
    with pytest.raises(RuntimeError, match="a_scale"):
        raw(lib.EPI_RESID, None, sw.data_ptr())
    with pytest.raises(RuntimeError, match="DWM_EPI_RESID"):
        raw(lib.EPI_STORE, sa.data_ptr(), sw.data_ptr())
    # E4M3 GroupNorm: C % 16
    x = torch.randn(2, 1, 4, 4, 40).cuda()
    o = torch.empty(2, 1, 4, 4, 40, device="cuda", dtype=F8)
    with pytest.raises(RuntimeError, match="C % 16"):
        ops.groupnorm_silu_e4m3(x, ops.groupnorm_stats(x, 8), torch.ones(40).cuda(),
                                torch.zeros(40).cuda(), o, torch.empty(2).cuda(), groups=8)


# ------------------------------------------------------------------ the model
def _unet(cfg, sd, dtype=torch.float16, fp8=True):
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    m = U(**cfg, compute_dtype=dtype, gemm_dtype=F8 if fp8 else None)
    m.load_state_dict(sd)
    return m.cuda()


def _cuda(c):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}


@pytest.mark.parametrize("case", ["image", "video", "pointwise", "full_width"])
def test_model_accuracy_against_fake_quant_oracle(case):
    from test_unet import UNET_CASES, _inputs, _oracle, unet_case
    if case == "full_width":
        cfg = fue.FULL_WIDTH
        x, t, c = _inputs(1, 2, 2, H=16, W=24)
        c["condition_image_tensor"] = None
    else:
        B, T, V, _ = next(u for u in UNET_CASES if u[3] == case)
        cfg, x, t, c = unet_case(B, T, V, case)
    o = _oracle(cfg).cuda()
    x, t, c = x.cuda(), t.cuda(), _cuda(c)
    emu, ref = fue.emulated_error(o, x, t, c)
    m = _unet(cfg, o.state_dict())
    y = m(x, t, **c)[0][0].clone()
    err = fe.rel_err(y, ref)
    # the spread of the model's own answer: GroupNorm statistics are summed with atomics, and
    # a last-bit change of a GroupNorm output moves an E4M3 rounding by 2^-4 (2^-10 in 16 bit),
    # which these small random UNets amplify (two 16-bit calls differ by ~2e-3, two FP8 calls
    # by ~8e-2 on the `image` case)
    spread = fe.rel_err(m(x, t, **c)[0][0], y)
    print("fp8 unet error", case, err, "fake-quant oracle", emu, "run-to-run spread", spread)
    # measured on an H100: emulator 0.155 / 0.101 / 0.125 / 0.114 (image / video / pointwise /
    # full_width), the FP8 model 0.113 / 0.086 / 0.141 / 0.108
    assert err <= 1.5 * emu + spread and err < 0.25, (err, emu, spread)
    # the packed conv weights are the emulator's: same quantizer on the same fp32 parameters
    conv = o.down_blocks[0].resnets[0].spatial_res_block.conv1
    q_ref, s_ref = fe.quantize_rows(conv.weight.detach().float().reshape(conv.out_channels, -1).cpu())
    w8, s = m._pk["down"][0]["res"][0]["c1"].w, m._pk["down"][0]["res"][0]["c1"].scale
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(w8.permute(1, 0, 2).reshape(conv.out_channels, -1).cpu().view(torch.uint8),
                       q_ref.view(conv.out_channels, conv.in_channels, 9).transpose(1, 2)
                       .reshape(conv.out_channels, -1).view(torch.uint8))


def test_model_repeatable_and_graph_equals_eager():
    """Two eager calls, and a CUDA-graph replay against eager (DDIM).  The GroupNorm statistics
    are summed with atomics in either precision, so as for the 16-bit UNet
    (test_pipeline_gpu.py) the step is not bit-reproducible: the graphed run may differ from
    an eager one by no more than two eager runs differ from each other."""
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from test_unet import UCFG, _inputs, _oracle
    m = _unet(UCFG, _oracle(UCFG).state_dict())
    x, t, c = _inputs(2, 2, 2)
    x, t, c = x.cuda(), t.cuda(), _cuda(c)
    y1 = m(x, t, **c)[0][0].clone()
    y2 = m(x, t, **c)[0][0].clone()
    assert torch.isfinite(y1).all() and torch.isfinite(y2).all()
    print("fp8 unet two eager calls, max rel diff", fe.rel_err(y2, y1))
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda",
                               {"frame_prediction_style": "ctsd"}, {},
                               {"guidance_scale": 3.0, "inference_steps": 4}, None, m,
                               model_dtype=torch.float32)
    pipe.test_scheduler.set_timesteps(4, "cuda")
    a, a2, b = (x[:1].clone() for _ in range(3))
    for ts_ in pipe.test_scheduler.timesteps.tolist():
        ts = torch.full((1, 2, 2), ts_, dtype=torch.int32, device="cuda")
        pipe.denoise_step(a, c, None, ts, None)
        pipe.denoise_step(a2, c, None, ts, None)
        pipe.denoise_step_graphed(b, c, None, ts, None)
    assert len(pipe._graphs) == 1
    assert torch.isfinite(a).all() and not torch.equal(a, x[:1])
    noise = (a - a2).abs().max().item()
    assert (a - b).abs().max().item() <= max(4 * noise, 2e-2 * a.abs().max().item()), noise


def test_pipeline_with_gemm_dtype_from_config():
    from dwm.common import create_instance_from_config
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from test_pipeline_gpu import COMMON, _batch
    from test_unet import UCFG, _oracle
    o = _oracle(UCFG)
    m = create_instance_from_config(
        {"_class_name": "dwm.models.crossview_temporal_unet.UNetCrossviewTemporalConditionModel",
         **UCFG, "compute_dtype": {"_class_name": "get_class", "class_name": "torch.float16"},
         "gemm_dtype": {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}})
    m.load_state_dict(o.state_dict())
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda",
                               dict(COMMON, frame_prediction_style="ctsd"), {},
                               {"guidance_scale": 3.0, "inference_steps": 3}, None, m,
                               model_dtype=torch.float32)
    batch = _batch(2, 3, dict(joint_attention_dim=96, pooled_projection_dim=8), hw=(128, 192))
    r = pipe.inference_pipeline((1, 2, 3, 4, 16, 24), batch, "pt")
    assert m._pk["fp8"]
    assert torch.isfinite(r["latents"]).all()
