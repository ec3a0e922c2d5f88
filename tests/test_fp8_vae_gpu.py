"""The opt-in FP8 (E4M3) path of the VAE decoders on the GPU: the E4M3 SpatialNorm3D + SiLU with
its causal-conv cache tail against float64, the E4M3 x F32 convolution element by element on
exactly-accumulating operands, the CogVideoX and AutoencoderKL decodes against the fake-quant
oracle, gemm_dtype=None against a model built without it, and the loud errors."""
import ctypes

import pytest
import torch

import fp8_emulation as fe
import fp8_vae_emulation as fve
from test_fp8_conformance_gpu import ConvOperands
from test_gemm_conformance_gpu import (
    F32, GUARD, H100_SMS, Epi, _bits, _label, _Options, _sms, check_output, conv_kernel,
    epilogue_reference, in_nan_block, padded_vec, row_scales, sentinel_buffer)
from test_norm_conformance_gpu import (
    SENT8, check16, e4m3_check, gn_data, gn_params, gn_reference, out16_tol, z_data)

pytestmark = pytest.mark.gpu
F8 = torch.float8_e4m3fn


# ------------------------------------------------------------------ E4M3 SpatialNorm + SiLU
# C, T, (Tz, hz, wz) of zy / zb (None: plain GroupNorm), cache: "none" (no tails), "first"
# (tail_out only: a first chunk), "in_place" (tail_in is tail_out), "separate"; tail dtype
SN_CASES = [
    (128, 5, (3, 4, 6), "first", torch.bfloat16),      # odd T, the first chunk's frame map
    (256, 4, (2, 2, 4), "in_place", torch.float16),    # even T after a chunk
    (128, 1, (1, 8, 6), "separate", torch.bfloat16),   # T = 1 with a cached tail
    (512, 1, (1, 4, 3), "first", torch.float16),       # T = 1, the tail replicates frame 0
    (128, 3, None, "none", torch.bfloat16),            # no modulation, no cache, out_t0 = 1
]


@pytest.mark.parametrize("C,T,zdims,cache,dtype", SN_CASES)
def test_spatialnorm_silu_e4m3(C, T, zdims, cache, dtype):
    """Bytes and scales against a float64 restatement, within the E4M3 bound of
    test_norm_conformance_gpu (e4m3_check); groups of large mean and constant groups from its
    gn_data.  The volume's amax covers the 16-bit cached tail, which lands in the operand's
    frames out_t0 - 2, out_t0 - 1; tail_out holds the operand's last two frames in 16 bit."""
    from opendwm_b200 import ops
    nb, H, W, G, eps = 3, 8, 12, 32, 1e-6
    x = gn_data(nb, T, H, W, C, G, seed=C + T)
    gamma, beta = gn_params(C, C)
    zy = zb = None
    if zdims is not None:
        zy, zb = z_data(nb, *zdims, C, seed=C)
    ref, err = gn_reference(x, G, gamma, beta, eps, zy, zb, silu=True)
    tail_in = None
    if cache in ("in_place", "separate"):
        g = torch.Generator().manual_seed(7)
        # volume 1's tail holds its largest values: the tail sets that volume's scale
        mag = ref.abs().reshape(nb, -1).amax(1) * torch.tensor([0.5, 3.0, 1.0], dtype=torch.float64)
        tail_in = (torch.randn(nb, 2, H, W, C, generator=g, dtype=torch.float64) / 3 *
                   mag.view(-1, 1, 1, 1, 1)).to(dtype)
    out_t0 = 2 if cache != "none" else 1
    out_T = out_t0 + T + 1
    out = torch.full((nb, out_T, H, W, C), SENT8, dtype=torch.uint8).cuda().view(F8)
    scale = torch.full((nb,), -1.0).cuda()
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    tin = dev(tail_in)
    tout = None
    if cache == "in_place":
        tout = tin.clone()
        tin = tout
    elif cache in ("first", "separate"):
        tout = torch.full((nb, 2, H, W, C), float("nan"), dtype=dtype).cuda()
    keep = tin.clone() if tin is not None else None
    ops.spatialnorm_silu_e4m3(dev(x), ops.groupnorm_stats(dev(x), G), dev(gamma), dev(beta), out,
                              scale, groups=G, eps=eps, zy=dev(zy), zb=dev(zb), out_t0=out_t0,
                              silu=True, tail_in=tin, tail_out=tout)
    torch.cuda.synchronize()
    lo = out_t0 - (2 if tail_in is not None else 0)
    written = torch.zeros(out_T, dtype=torch.bool)
    written[lo:out_t0 + T] = True
    assert (out.view(torch.uint8)[:, ~written.cuda()] == SENT8).all(), "frames outside the window were written"
    q = out[:, lo:out_t0 + T].cpu()
    if tail_in is not None:
        ref_v = torch.cat([keep.cpu().double(), ref], 1)
        err_v = torch.cat([torch.zeros(nb, 2, H, W, C, dtype=torch.float64), err], 1)
    else:
        ref_v, err_v = ref, err
    e4m3_check(q.reshape(nb, -1), scale, ref_v.reshape(nb, -1), err_v.reshape(nb, -1),
               "spatialnorm_silu_e4m3 C=%d T=%d %s" % (C, T, cache))
    if tout is None:
        return
    tout = tout.cpu()
    if T >= 2:
        r, e = ref[:, T - 2:], err[:, T - 2:]
        check16(tout.double(), r, out16_tol(e, r, dtype), "tail_out")
    else:
        check16(tout[:, 1:].double(), ref, out16_tol(err, ref, dtype), "tail_out frame 1")
        want0 = keep[:, 1:].cpu() if tail_in is not None else tout[:, 1:]
        assert torch.equal(tout[:, :1].view(torch.int16), want0.view(torch.int16)), "tail_out frame 0"


# ------------------------------------------------------------------ E4M3 x F32 convolution
# name, (nb, t_out, h, w, c_in, c_out, kernel), the kernel the default options reach on an H100
F32_CONV_CASES = [
    ("k333_cin128_cout128", (2, 3, 8, 40, 128, 128, (3, 3, 3)), "NT128_CL1"),
    ("k333_cin512_cout128", (2, 2, 8, 40, 512, 128, (3, 3, 3)), "NT128_CL1"),
    ("k333_cin256_cout512", (2, 2, 6, 24, 256, 512, (3, 3, 3)), "NT256_CL1"),
    ("k133_cin128_cout256_pair", (6, 1, 44, 128, 128, 256, (1, 3, 3)), "NT256_CL2"),
    ("k133_cin256_cout128_halo", (2, 1, 66, 128, 256, 128, (1, 3, 3)), "NT128_CL1_HALO"),
    ("k333_cin128_cout128_halo", (1, 2, 66, 128, 128, 128, (3, 3, 3)), "NT128_CL1_HALO"),
    ("k133_cin128_cout128_halo_pair", (2, 1, 132, 128, 128, 128, (1, 3, 3)), "NT128_CL1_HALO"),
]


def _launch_f32(op, dev, bias, conv_2cta=1, conv_halo=1):
    from opendwm_b200 import ops
    x, wt, sa, sw = dev
    rows = op.U.shape[0]
    buf = sentinel_buffer(rows, op.c_out, torch.float32)
    with _Options(conv_2cta=conv_2cta, conv_halo=conv_halo):
        ops.conv(x, wt, bias, kernel=op.kernel, epilogue=F32, out=buf[GUARD:GUARD + rows, :op.c_out],
                 a_scale=sa, w_scale=sw)
        torch.cuda.synchronize()
    return buf


@pytest.mark.parametrize("name,shape,label", F32_CONV_CASES, ids=[c[0] for c in F32_CONV_CASES])
def test_fp8_conv_f32_conforms(name, shape, label):
    """The operands of test_fp8_conformance_gpu accumulate exactly in any order, so the 1-CTA,
    pair, halo-row and per-tap kernels the options reach must give identical bits, within the
    fp32 epilogue's bound of float64 (bias only: out = acc sa sw + bias)."""
    nb, t_out, h, w, c_in, c_out, kernel = shape
    sms = _sms()
    k0 = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms)
    if sms == H100_SMS:
        assert _label(k0) == label
    op = ConvOperands(nb, t_out + kernel[0] - 1, h, w, c_in, c_out, kernel, seed=h * w + c_in)
    g = torch.Generator().manual_seed(c_out)
    bias = padded_vec(torch.randn(c_out, generator=g) * row_scales(c_out, 1e3) * 0.1 * 2.0 ** -20)
    e = Epi(F32, bias=bias)
    ref, tol = epilogue_reference(op.z.cuda(), op.P.cuda(), kernel[0] * kernel[1] * kernel[2] * c_in,
                                  e, torch.float32, acc_err=op.acc_err.cuda())
    dev = (in_nan_block(op.x8), in_nan_block(op.w8), padded_vec(op.sa), padded_vec(op.sw))
    outs = {}
    for two in (1, 0):
        for halo in (1, 0):
            k = conv_kernel(nb, t_out, h, w, c_out, kernel[2], sms, two, halo)
            if k not in outs:
                outs[k] = _launch_f32(op, dev, bias, two, halo)
    for k, b in outs.items():
        assert torch.equal(_bits(b), _bits(outs[k0])), "%s gave other bits than %s" % (_label(k), label)
    worst = check_output(outs[k0], torch.arange(op.U.shape[0]), c_out, ref, tol, name)
    print("BOUND_RATIO fp8_conv_f32 %s_%s %.4g" % (name, "+".join(_label(k) for k in outs), worst))


# ------------------------------------------------------------------ the decoders
def _cogvideox(o, dtype, fp8=True):
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    m = AutoencoderKLCogVideoX(**fve.COGVIDEOX, compute_dtype=dtype, gemm_dtype=F8 if fp8 else None)
    m.load_state_dict(o.state_dict())
    return m.cuda()


def _check_model(y, y2, out, what):
    emu = fe.rel_err(out["fq"], out["ref"])
    err = fe.rel_err(y, out["ref"])
    spread = fe.rel_err(y2, y)
    print("fp8 vae", what, "error", err, "fake-quant oracle", emu, "run-to-run spread", spread)
    assert torch.isfinite(y).all()
    assert spread <= fve.SPREAD_CAP, spread
    assert err <= 1.5 * emu + spread, (err, emu, spread)


@pytest.mark.parametrize("views,frames,dtype", [(2, 5, torch.bfloat16), (6, 2, torch.float16),
                                                (2, 1, torch.float16), (2, 3, torch.float16)],
                         ids=["multi_chunk", "df_frame_and_zero_frame", "one_frame",
                              "one_odd_chunk"])
def test_cogvideox_decode_against_fake_quant_oracle(views, frames, dtype):
    """5 latent frames decode in chunks 3 + 2, so every FP8 conv of the second chunk starts from
    the first chunk's 16-bit tail.  The diffusion-forcing decode of the pipeline is one even
    chunk: the emitted latent frame and a zero frame (ctsd.py's DF branch).  One latent frame
    alone is the T = 1 operand at every level; 3 frames one odd chunk."""
    o = fve.cogvideox_oracle().cuda()
    z = fve.cogvideox_latents(views, frames, 4, 6)
    if frames == 2:
        z[:, :, 1] = 0
    z = z.cuda()
    out = fve.cogvideox_outputs(o, z, dtype)
    m = _cogvideox(o, dtype)
    y = m.decode(z, return_dict=False)[0].clone()
    y2 = m.decode(z, return_dict=False)[0]
    assert y.shape == out["ref"].shape
    _check_model(y, y2, out, "cogvideox %d views %d frames" % (views, frames))
    # the packed weights are the emulator's: same quantizer on the same fp32 parameters
    c = o.decoder.mid_block.resnets[0].conv1.conv
    q_ref, s_ref = fe.quantize_rows(c.weight.detach().float().reshape(c.out_channels, -1).cpu())
    pk = m._pk["mid"][0]["c1"]
    assert torch.equal(pk.scale.cpu(), s_ref)
    assert torch.equal(pk.w.permute(1, 0, 2).reshape(c.out_channels, -1).cpu().view(torch.uint8),
                       q_ref.view(c.out_channels, c.in_channels, 27).transpose(1, 2)
                       .reshape(c.out_channels, -1).view(torch.uint8))


def test_autoencoder_kl_decode_against_fake_quant_oracle():
    from dwm.models.autoencoder_kl import AutoencoderKL
    o = fve.autoencoder_kl_oracle().cuda()
    g = torch.Generator().manual_seed(3)
    z = (torch.randn(3, 16, 8, 12, generator=g) *
         torch.tensor([1.0, 4.0, 0.25]).view(-1, 1, 1, 1)).to(torch.float16)
    out = fve.autoencoder_kl_outputs(o, z.float().cuda())
    m = AutoencoderKL(**fve.SD_KL, compute_dtype=torch.float16, gemm_dtype=F8)
    m.load_state_dict(o.state_dict())
    m.cuda()
    y = m.decode(z.cuda(), return_dict=False)[0].clone()
    y2 = m.decode(z.cuda(), return_dict=False)[0]
    _check_model(y, y2, out, "autoencoder_kl")
    assert m._pk["mid"][0]["c1"].scale is not None and m._pk["conv_in"].scale is None


# The 16-bit decode methods the FP8 path touched, as they read before it (verbatim, commit
# 9eb0e97): gemm_dtype=None must launch what they launch, in their order, and give their bits.
def _pre_fp8_cogvideox_causal_conv(self, name, x_pad, c, cache, new_cache, **kw):
    from dwm.models.packing import conv
    prev = cache.get(name)
    if prev is not None:
        x_pad[:, :2].copy_(prev)
    else:
        x_pad[:, :2].copy_(x_pad[:, 2:3].expand(-1, 2, -1, -1, -1))
    new_cache[name] = x_pad[:, -2:]
    return conv(x_pad, c, kernel=(3, 3, 3), **kw)


def _pre_fp8_cogvideox_norm_act(self, h, shape, p, zq16, zshape, groups):
    from dwm.models.packing import gemm
    from opendwm_b200 import lib as _lib
    from opendwm_b200 import ops as _ops
    nb, T, H, W = shape
    C = h.shape[1]
    h5 = h.view(nb, T, H, W, C)
    sums = _ops.groupnorm_stats(h5, groups)
    zy = gemm(zq16, p["y"], epilogue=_lib.EPI_F32).view(*zshape, C)
    zb = gemm(zq16, p["b"], epilogue=_lib.EPI_F32).view(*zshape, C)
    out = torch.empty(nb, T + 2, H, W, C, device=h.device, dtype=self.compute_dtype)
    g = p["norm"]
    _ops.spatialnorm_silu(h5, sums, g[0], g[1], out, groups=groups,
                          eps=g[2], zy=zy, zb=zb, out_t0=2, silu=True)
    return out


def _pre_fp8_cogvideox_resnet(self, name, h, shape, p, zq16, zshape, groups, cache, new_cache):
    from dwm.models.packing import gemm
    from opendwm_b200 import lib as _lib
    from opendwm_b200 import ops as _ops
    a = self._norm_act(h, shape, p["n1"], zq16, zshape, groups)
    h1 = self._causal_conv(name + ".conv1", a, p["c1"], cache, new_cache,
                           epilogue=_lib.EPI_F32)
    b = self._norm_act(h1, shape, p["n2"], zq16, zshape, groups)
    if "sc" in p:
        h16 = torch.empty(h.shape, device=h.device, dtype=self.compute_dtype)
        _ops.act_cast(h, h16)
        skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
    else:
        skip = h
    return self._causal_conv(name + ".conv2", b, p["c2"], cache, new_cache,
                             epilogue=_lib.EPI_RESID, resid=skip)


def _pre_fp8_autoencoder_kl_resnet(self, h, shape, p):
    from dwm.models.packing import conv, gemm
    from opendwm_b200 import lib as _lib
    from opendwm_b200 import ops as _ops
    a = self._norm(h, shape, p["n1"], True)
    h1 = conv(a, p["c1"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
    b = self._norm(h1, shape, p["n2"], True)
    if "sc" in p:
        h16 = torch.empty(h.shape, device=h.device, dtype=self.compute_dtype)
        _ops.act_cast(h, h16)
        skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
    else:
        skip = h
    return conv(b, p["c2"], kernel=(1, 3, 3), epilogue=_lib.EPI_RESID, resid=skip)


def _abi_calls(f):
    """(result, the dwm_b200_* C calls f made, in order, with their shape arguments: pointers
    differ between models and are left out)."""
    from opendwm_b200 import lib
    L, calls = lib.load(), []
    saved = {n: getattr(L, n) for n in lib.SYMBOLS}

    def rec(name, fn):
        def call(*args):
            shape = []
            for a in args:
                obj = getattr(a, "_obj", None)          # a byref'd args struct
                if obj is not None:
                    shape.append(tuple((k, getattr(obj, k)) for k, t in obj._fields_
                                       if t in (ctypes.c_int, ctypes.c_int64, ctypes.c_float)))
                elif isinstance(a, (int, float)) and not (isinstance(a, int) and a > 1 << 32):
                    shape.append(a)
            calls.append((name, tuple(shape)))
            return fn(*args)
        return call
    for n, fn in saved.items():
        setattr(L, n, rec(n, fn))
    try:
        y = f()
        torch.cuda.synchronize()
    finally:
        for n, fn in saved.items():
            setattr(L, n, fn)
    return y, calls


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_gemm_dtype_none_is_the_pre_fp8_decode(dtype):
    """gemm_dtype=None and no argument make the C calls (kernel entries and shape arguments,
    in order) and give the bits of the decode methods as they read before the FP8 path (multi-chunk CogVideoX clip with shortcut
    ResNets, AutoencoderKL with its mid-block attention)."""
    import types
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    o = fve.cogvideox_oracle()
    z = fve.cogvideox_latents(2, 5, 4, 6).cuda()
    models = [AutoencoderKLCogVideoX(**fve.COGVIDEOX, compute_dtype=dtype),
              AutoencoderKLCogVideoX(**fve.COGVIDEOX, compute_dtype=dtype, gemm_dtype=None),
              AutoencoderKLCogVideoX(**fve.COGVIDEOX, compute_dtype=dtype)]
    old = models[2]
    old._causal_conv = types.MethodType(_pre_fp8_cogvideox_causal_conv, old)
    old._norm_act = types.MethodType(_pre_fp8_cogvideox_norm_act, old)
    old._resnet = types.MethodType(_pre_fp8_cogvideox_resnet, old)
    runs = []
    for m in models:
        m.load_state_dict(o.state_dict())
        m.cuda()
        m.decode(z, return_dict=False)        # packs the weights outside the profiled call
        runs.append(_abi_calls(lambda: m.decode(z, return_dict=False)[0]))
    assert all(r[c].scale is None for r in models[1]._pk["mid"] for c in ("c1", "c2"))
    for y, names in runs[:2]:
        assert names == runs[2][1], "other C calls than before the FP8 path"
        assert torch.equal(y, runs[2][0]), "other bits than before the FP8 path"
    ok = fve.autoencoder_kl_oracle()
    zk = torch.randn(2, 16, 8, 12, generator=torch.Generator().manual_seed(1)).cuda().to(dtype)
    models = [AutoencoderKL(**fve.SD_KL, compute_dtype=dtype),
              AutoencoderKL(**fve.SD_KL, compute_dtype=dtype, gemm_dtype=None),
              AutoencoderKL(**fve.SD_KL, compute_dtype=dtype)]
    models[2]._resnet = types.MethodType(_pre_fp8_autoencoder_kl_resnet, models[2])
    runs = []
    for m in models:
        m.load_state_dict(ok.state_dict())
        m.cuda()
        m.decode(zk, return_dict=False)
        runs.append(_abi_calls(lambda: m.decode(zk, return_dict=False)[0]))
    for y, names in runs[:2]:
        assert names == runs[2][1], "other C calls than before the FP8 path"
        assert torch.equal(y, runs[2][0]), "other bits than before the FP8 path"


# ------------------------------------------------------------------ loud errors
def test_errors_are_loud():
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    from opendwm_b200 import lib, ops
    with pytest.raises(ValueError, match="gemm_dtype"):
        AutoencoderKLCogVideoX(**fve.COGVIDEOX, gemm_dtype=torch.float8_e5m2)
    m = _cogvideox(fve.cogvideox_oracle(), torch.bfloat16)
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        m.decode(torch.zeros(1, 16, 1, 4, 6))
    x = torch.randn(2, 1, 4, 8, 128).cuda()
    sums = ops.groupnorm_stats(x, 32)
    gamma, beta = torch.ones(128).cuda(), torch.zeros(128).cuda()
    out = torch.empty(2, 3, 4, 8, 128, device="cuda", dtype=F8)
    sc = torch.empty(2).cuda()
    with pytest.raises(TypeError, match="cuda fp32"):
        ops.spatialnorm_silu_e4m3(x.cpu(), sums, gamma, beta, out, sc, groups=32)
    tail = torch.zeros(2, 2, 4, 8, 128, device="cuda", dtype=torch.bfloat16)
    # host operands of the right shape and dtype are refused before any kernel sees them
    for kw in (dict(out_t0=2, tail_in=tail.cpu()), dict(out_t0=2, tail_out=tail.cpu()),
               dict(out_t0=2, tail_in=tail, tail_out=tail.cpu())):
        with pytest.raises(RuntimeError, match="tail_.* is on cpu"):
            ops.spatialnorm_silu_e4m3(x, sums, gamma, beta, out, sc, groups=32, **kw)
    with pytest.raises(RuntimeError, match="out is on cpu"):
        ops.spatialnorm_silu_e4m3(x, sums, gamma, beta, out.cpu(), sc, groups=32)
    with pytest.raises(RuntimeError, match="sums is on cpu"):
        ops.spatialnorm_silu_e4m3(x, sums.cpu(), gamma, beta, out, sc, groups=32)
    with pytest.raises(RuntimeError, match="out_t0 >= 2"):
        ops.spatialnorm_silu_e4m3(x, sums, gamma, beta, out, sc, groups=32, out_t0=1, tail_in=tail)
    with pytest.raises(ValueError, match="tail_in / tail_out"):
        ops.spatialnorm_silu_e4m3(x, sums, gamma, beta, out, sc, groups=32, out_t0=2,
                                  tail_in=tail[:, :1].contiguous())
    # FP8 conv operands without scales, with the F32 epilogue
    x8 = torch.zeros(2, 3, 4, 8, 128, device="cuda", dtype=F8)
    w8 = torch.zeros(27, 128, 128, device="cuda", dtype=F8)
    sw = torch.ones(128).cuda()
    with pytest.raises(ValueError, match="a_scale and w_scale"):
        ops.conv(x8, w8, kernel=(3, 3, 3), epilogue=lib.EPI_F32, w_scale=sw)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.conv(x8.cpu(), w8.cpu(), kernel=(3, 3, 3), epilogue=lib.EPI_F32, a_scale=sc.cpu(),
                 w_scale=sw.cpu())

    def raw(c_out, a_scale):
        a = lib.ConvArgs()
        a.x, a.nb, a.tp, a.h, a.w, a.c_in = x8.data_ptr(), 2, 3, 4, 8, 128
        a.weight, a.kt, a.kh, a.kw, a.c_out = w8.data_ptr(), 3, 3, 3, c_out
        o = torch.empty(64, c_out, device="cuda")
        a.dtype, a.epilogue, a.out, a.ldo = lib.DWM_E4M3, lib.EPI_F32, o.data_ptr(), c_out
        a.a_scale, a.w_scale = a_scale, sw.data_ptr()
        lib.check(lib.load().dwm_b200_conv(ctypes.byref(a), torch.cuda.current_stream().cuda_stream),
                  "dwm_b200_conv")
    with pytest.raises(RuntimeError, match="a_scale"):
        raw(128, None)
    with pytest.raises(RuntimeError, match="C_out % 128"):
        raw(96, sc.data_ptr())
