"""CogVideoX temporal VAE — decode path, H100-native.

Mirror of the part of diffusers==0.31.0 `AutoencoderKLCogVideoX` that the reference uses
on the CTSD hot path (`vae.decode(z / scaling_factor + shift, return_dict=False)[0]`,
reference src/dwm/pipelines/ctsd.py:1628-1643 and :1609-1621; selected by
`common_config["vae"] = "diffusers.AutoencoderKLCogVideoX"`,
examples/ctsd_35_tvae_6views_video_generation_with_layout.json:51-52).

Same constructor / config keys, `from_pretrained(path, subfolder="vae")`, state_dict key
names (`decoder.*`; encoder keys are ignored: encode is not on the path) and the same
numerical contract: latent frames are decoded in chunks of 2 (the first chunk takes the
remainder) with the causal-conv caches carried across chunks, so GroupNorm statistics are
per chunk (SURVEY.md Appendix A.7).

Execution: activations are channels-last; every causal 3x3x3 convolution and the
per-frame 3x3 upsampler convolution is the im2col-free wgmma kernel
(`dwm_b200_conv`, taps iterated inside the MMA loop, spatial padding = TMA OOB fill,
causal temporal padding = two cached frames kept in front of each conv input buffer);
SpatialNorm3D (GroupNorm * conv_y(zq) + conv_b(zq)) + SiLU is one fused pass that emits
the next convolution's 16-bit input; conv_y / conv_b / conv_shortcut (1x1x1) run on the
wgmma GEMM at latent resolution; residual adds are conv epilogues.

gemm_dtype=torch.float8_e4m3fn runs conv1 / conv2 of every decoder ResNet block (mid and up
blocks) in E4M3: one activation scale per volume (one (b v) item of one chunk, cached frames
included), one weight scale per output channel.  The causal-conv cache stays 16-bit: the two
cached frames of the previous chunk are folded into this chunk's amax and quantized with its
scale (an E4M3 tail would carry the previous chunk's scale, which does not factor out of the
sum over taps).  conv_in / conv_out, the upsampler convs, the shortcuts, conv_y / conv_b and
the encoder stay 16-bit.
"""
import json
import math
import os

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops

from .packing import FP8, Operand, conv, gemm, pack_conv, pack_linear, pack_norm


class _Cfg(dict):
    __getattr__ = dict.get


class _P(torch.nn.Module):
    pass


def _causal(cin, cout, k):
    m = _P()
    m.conv = torch.nn.Conv3d(cin, cout, k)
    return m


def _spatial_norm(f, zq, groups):
    m = _P()
    m.norm_layer = torch.nn.GroupNorm(groups, f, eps=1e-6, affine=True)
    m.conv_y = _causal(zq, f, 1)
    m.conv_b = _causal(zq, f, 1)
    return m


def _pack_spatial_norm(m, dt, dev):
    """GroupNorm triple and the conv_y / conv_b (1x1x1) Linears of a SpatialNorm3D."""
    return dict(norm=pack_norm(m.norm_layer),
                y=pack_linear(m.conv_y.conv.weight, m.conv_y.conv.bias, dt, dev),
                b=pack_linear(m.conv_b.conv.weight, m.conv_b.conv.bias, dt, dev))


def _resnet(cin, cout, zq, groups):
    m = _P()
    m.norm1 = _spatial_norm(cin, zq, groups)
    m.conv1 = _causal(cin, cout, 3)
    m.norm2 = _spatial_norm(cout, zq, groups)
    m.conv2 = _causal(cout, cout, 3)
    if cin != cout:
        m.conv_shortcut = torch.nn.Conv3d(cin, cout, 1)
    return m


def _block(cin, cout, layers, zq, upsample, compress_time, groups):
    m = _P()
    m.resnets = torch.nn.ModuleList(
        [_resnet(cin if i == 0 else cout, cout, zq, groups) for i in range(layers)])
    m.compress_time = compress_time
    if upsample:
        up = _P()
        up.conv = torch.nn.Conv2d(cout, cout, 3, padding=1)
        m.upsamplers = torch.nn.ModuleList([up])
    return m


class AutoencoderKLCogVideoX(torch.nn.Module):

    def __init__(self, in_channels=3, out_channels=3,
                 block_out_channels=(128, 256, 256, 512), latent_channels=16,
                 layers_per_block=3, norm_num_groups=32,
                 temporal_compression_ratio=4, scaling_factor=1.15258426,
                 shift_factor=None, compute_dtype=torch.bfloat16, with_encoder=False,
                 gemm_dtype=None, **unused):
        """gemm_dtype=torch.float8_e4m3fn runs the decoder ResNet convolutions in E4M3 (see
        the module docstring); None keeps every convolution 16-bit."""
        super().__init__()
        if gemm_dtype not in (None, torch.float8_e4m3fn):
            raise ValueError(
                "gemm_dtype must be None or torch.float8_e4m3fn, got {!r}".format(gemm_dtype))
        self.config = _Cfg(
            in_channels=in_channels, out_channels=out_channels,
            block_out_channels=tuple(block_out_channels),
            latent_channels=latent_channels, layers_per_block=layers_per_block,
            norm_num_groups=norm_num_groups,
            temporal_compression_ratio=temporal_compression_ratio,
            scaling_factor=scaling_factor, shift_factor=shift_factor,
            down_block_types=("CogVideoXDownBlock3D",) * len(block_out_channels))
        self.compute_dtype = compute_dtype
        self.gemm_dtype = gemm_dtype
        self._ws8 = {}
        self.num_latent_frames_batch_size = 2
        g = norm_num_groups
        rev = list(reversed(block_out_channels))
        d = _P()
        d.conv_in = _causal(latent_channels, rev[0], 3)
        d.mid_block = _block(rev[0], rev[0], 2, latent_channels, False, False, g)
        level = int(math.log2(temporal_compression_ratio))
        d.up_blocks = torch.nn.ModuleList()
        out_ch = rev[0]
        for i in range(len(rev)):
            prev, out_ch = out_ch, rev[i]
            d.up_blocks.append(_block(prev, out_ch, layers_per_block + 1,
                                      latent_channels, i != len(rev) - 1,
                                      i < level, g))
        d.norm_out = _spatial_norm(rev[-1], latent_channels, g)
        d.conv_out = _causal(rev[-1], out_channels, 3)
        self.decoder = d
        self._pk = None
        self._pk_enc = None
        self.num_sample_frames_batch_size = 8
        if with_encoder:       # from_pretrained turns it on when the checkpoint has encoder weights
            self.encoder = self._build_encoder(in_channels, latent_channels, block_out_channels,
                                               layers_per_block, g, level)

    @staticmethod
    def _build_encoder(in_channels, latent_channels, block_out_channels, layers_per_block, g,
                       level):
        def enc_resnet(cin, cout):
            m = _P()
            m.norm1 = torch.nn.GroupNorm(g, cin, eps=1e-6)
            m.conv1 = _causal(cin, cout, 3)
            m.norm2 = torch.nn.GroupNorm(g, cout, eps=1e-6)
            m.conv2 = _causal(cout, cout, 3)
            if cin != cout:
                m.conv_shortcut = torch.nn.Conv3d(cin, cout, 1)
            return m
        boc = list(block_out_channels)
        e = _P()
        e.conv_in = _causal(in_channels, boc[0], 3)
        e.down_blocks = torch.nn.ModuleList()
        out_ch = boc[0]
        for i in range(len(boc)):
            prev, out_ch = out_ch, boc[i]
            b = _P()
            b.resnets = torch.nn.ModuleList(
                [enc_resnet(prev if j == 0 else out_ch, out_ch) for j in range(layers_per_block)])
            b.compress_time = i < level
            if i != len(boc) - 1:
                dn = _P()
                dn.conv = torch.nn.Conv2d(out_ch, out_ch, 3, stride=2, padding=0)
                b.downsamplers = torch.nn.ModuleList([dn])
            e.down_blocks.append(b)
        e.mid_block = _P()
        e.mid_block.resnets = torch.nn.ModuleList(
            [enc_resnet(boc[-1], boc[-1]), enc_resnet(boc[-1], boc[-1])])
        e.norm_out = torch.nn.GroupNorm(g, boc[-1], eps=1e-6)
        e.conv_out = _causal(boc[-1], 2 * latent_channels, 3)
        return e

    # -- diffusers-style plumbing -------------------------------------------------------
    @property
    def dtype(self):
        return self.compute_dtype

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kwargs):
        if subfolder:
            path = os.path.join(path, subfolder)
        with open(os.path.join(path, "config.json")) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        cfg.update(kwargs)
        for name in ("diffusion_pytorch_model.safetensors",
                     "diffusion_pytorch_model.fp16.safetensors"):
            fp = os.path.join(path, name)
            if os.path.exists(fp):
                import safetensors.torch
                state = safetensors.torch.load_file(fp, device="cpu")
                break
        else:
            state = torch.load(os.path.join(path, "diffusion_pytorch_model.bin"),
                               map_location="cpu", weights_only=True)
        # a checkpoint that carries the encoder gets it (validated against the oracle,
        # tests/test_vae_gpu.py::test_encode_matches_oracle), as diffusers' class always does
        has_enc = any(k.startswith("encoder.") for k in state)
        cfg.setdefault("with_encoder", has_enc)
        vae = cls(**cfg)
        keep = ("decoder.", "encoder.") if cfg["with_encoder"] else ("decoder.",)
        vae.load_state_dict({k: v for k, v in state.items() if k.startswith(keep)},
                            strict=True)
        return vae

    def _apply(self, fn, *a, **k):
        self._pk = self._pk_enc = None
        self._ws8 = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, assign=False):
        self._pk = self._pk_enc = None
        self._ws8 = {}
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    # -- weight packing --------------------------------------------------------------------
    @torch.no_grad()
    def _pack(self):
        dev = self.decoder.conv_in.conv.weight.device
        if dev.type != "cuda":
            raise RuntimeError("AutoencoderKLCogVideoX.decode runs on CUDA (sm_90a) "
                               "only; there is no CPU fallback.")
        dt = self.compute_dtype
        fp8 = self.gemm_dtype is not None

        def res(m):
            p = dict(n1=_pack_spatial_norm(m.norm1, dt, dev),
                     c1=pack_conv(m.conv1.conv, dt, dev, fp8),
                     n2=_pack_spatial_norm(m.norm2, dt, dev),
                     c2=pack_conv(m.conv2.conv, dt, dev, fp8))
            if hasattr(m, "conv_shortcut"):
                p["sc"] = pack_linear(m.conv_shortcut.weight, m.conv_shortcut.bias, dt, dev)
            return p

        d = self.decoder
        pk = dict(conv_in=pack_conv(d.conv_in.conv, dt, dev),
                  mid=[res(r) for r in d.mid_block.resnets], ups=[])
        for blk in d.up_blocks:
            b = dict(res=[res(r) for r in blk.resnets], compress=blk.compress_time)
            if hasattr(blk, "upsamplers"):
                b["up"] = pack_conv(blk.upsamplers[0].conv, dt, dev)
            pk["ups"].append(b)
        pk["norm_out"] = _pack_spatial_norm(d.norm_out, dt, dev)
        cout = self.config.out_channels
        pk["conv_out"] = pack_conv(d.conv_out.conv, dt, dev, pad_out=32 if cout < 32 else None)
        self._pk = pk
        return pk

    # -- building blocks ---------------------------------------------------------------------
    def _causal_conv(self, name, x_pad, c, cache, new_cache, **kw):
        """x_pad: 16-bit [nb, T+2, H, W, C] whose frames [2:] are filled; the two leading
        frames become the cached tail of the previous chunk or replicas of frame 0.  An E4M3
        Operand of `_norm_operand` has its cache frames already in place."""
        if isinstance(x_pad, Operand):
            return conv(x_pad, c, kernel=(3, 3, 3), **kw)
        prev = cache.get(name)
        if prev is not None:
            x_pad[:, :2].copy_(prev)
        else:
            x_pad[:, :2].copy_(x_pad[:, 2:3].expand(-1, 2, -1, -1, -1))
        # the cached tail is a VIEW of this chunk's padded input (every x_pad is a fresh buffer
        # that nothing writes again), copied once into the next chunk's padding: one copy per
        # convolution and chunk instead of clone + copy
        new_cache[name] = x_pad[:, -2:]
        return conv(x_pad, c, kernel=(3, 3, 3), **kw)

    def _norm_operands(self, h, shape, p, zq16, zshape, groups):
        """(h as [nb, T, H, W, C], its GroupNorm sums, zy, zb) of a SpatialNorm3D."""
        nb, T, H, W = shape
        C = h.shape[1]
        h5 = h.view(nb, T, H, W, C)
        sums = _ops.groupnorm_stats(h5, groups)
        zy = gemm(zq16, p["y"], epilogue=_lib.EPI_F32).view(*zshape, C)
        zb = gemm(zq16, p["b"], epilogue=_lib.EPI_F32).view(*zshape, C)
        return h5, sums, zy, zb

    def _norm_act(self, h, shape, p, zq16, zshape, groups):
        """SpatialNorm3D + SiLU of fp32 `h` [rows, C] -> 16-bit time-padded conv input."""
        h5, sums, zy, zb = self._norm_operands(h, shape, p, zq16, zshape, groups)
        nb, T, H, W, C = h5.shape
        out = torch.empty(nb, T + 2, H, W, C, device=h.device, dtype=self.compute_dtype)
        g = p["norm"]
        _ops.spatialnorm_silu(h5, sums, g[0], g[1], out, groups=groups,
                              eps=g[2], zy=zy, zb=zb, out_t0=2, silu=True)
        return out

    def _buf8(self, key, shape, dtype):
        """Workspace kept across calls of one geometry: each FP8 conv's 16-bit cache tail
        (2 frames per volume) and the volume scales."""
        k = (key, tuple(shape), dtype)
        if k not in self._ws8:
            self._ws8[k] = torch.empty(shape, device=self.decoder.conv_in.conv.weight.device,
                                       dtype=dtype)
        return self._ws8[k]

    def _operand8(self, shape):
        """The E4M3 operand of an FP8 conv: a view of ONE buffer that every FP8 conv shares
        (each conv reads it before the next SpatialNorm writes it, in stream order), grown to
        the largest operand seen and kept across calls."""
        n = math.prod(shape)
        buf = self._ws8.get("x8")
        if buf is None or buf.numel() < n:
            buf = self._ws8["x8"] = torch.empty(
                n, device=self.decoder.conv_in.conv.weight.device, dtype=FP8)
        return buf[:n].view(shape)

    def _norm_operand(self, name, h, shape, p, c, zq16, zshape, groups, cache, new_cache):
        """SpatialNorm3D + SiLU of fp32 `h` as the operand of the causal conv c (a ResNet conv1 /
        conv2): 16-bit (`_causal_conv` fills its cache frames), or for an E4M3 c an E4M3
        Operand whose volume scale covers the 16-bit cache tail of the previous chunk, with the
        operand's last two frames kept in 16 bit as the next tail."""
        if c.scale is None:
            return self._norm_act(h, shape, p, zq16, zshape, groups)
        h5, sums, zy, zb = self._norm_operands(h, shape, p, zq16, zshape, groups)
        nb, T, H, W, C = h5.shape
        x8 = self._operand8((nb, T + 2, H, W, C))
        scale = self._buf8("x8_scale", (nb,), torch.float32)
        prev = cache.get(name)
        tail = self._buf8(name, (nb, 2, H, W, C), self.compute_dtype)
        g = p["norm"]
        _ops.spatialnorm_silu_e4m3(h5, sums, g[0], g[1], x8, scale, groups=groups, eps=g[2],
                                   zy=zy, zb=zb, out_t0=2, silu=True, tail_in=prev,
                                   tail_out=tail)
        if prev is None:      # replicas of frame 0: its bytes, under the same scale
            b = x8.view(torch.uint8)
            b[:, :2].copy_(b[:, 2:3].expand(-1, 2, -1, -1, -1))
        new_cache[name] = tail
        return Operand(x8, scale)

    def _resnet(self, name, h, shape, p, zq16, zshape, groups, cache, new_cache):
        a = self._norm_operand(name + ".conv1", h, shape, p["n1"], p["c1"], zq16, zshape,
                               groups, cache, new_cache)
        h1 = self._causal_conv(name + ".conv1", a, p["c1"], cache, new_cache,
                               epilogue=_lib.EPI_F32)
        b = self._norm_operand(name + ".conv2", h1, shape, p["n2"], p["c2"], zq16, zshape,
                               groups, cache, new_cache)
        if "sc" in p:
            h16 = torch.empty(h.shape, device=h.device, dtype=self.compute_dtype)
            _ops.act_cast(h, h16)
            skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
        else:
            skip = h
        return self._causal_conv(name + ".conv2", b, p["c2"], cache, new_cache,
                                 epilogue=_lib.EPI_RESID, resid=skip)

    def _decode_chunk(self, z, cache):
        """z: fp32 channels-last latent chunk [nb, Tz, hz, wz, Cz] -> fp32 [nb, T, H, W, 3]."""
        pk, dt = self._pk, self.compute_dtype
        groups = self.config.norm_num_groups
        nb, Tz, hz, wz, Cz = z.shape
        new_cache = {}
        zshape = (nb, Tz, hz, wz)
        z16 = z.to(dt).contiguous()
        zq16 = z16.view(nb * Tz * hz * wz, Cz)
        zin = torch.empty(nb, Tz + 2, hz, wz, Cz, device=z.device, dtype=dt)
        zin[:, 2:].copy_(z16)
        h = self._causal_conv("conv_in", zin, pk["conv_in"], cache, new_cache,
                              epilogue=_lib.EPI_F32)
        shape = (nb, Tz, hz, wz)
        for i, p in enumerate(pk["mid"]):
            h = self._resnet("mid.%d" % i, h, shape, p, zq16, zshape, groups, cache,
                             new_cache)
        for bi, blk in enumerate(pk["ups"]):
            for ri, p in enumerate(blk["res"]):
                h = self._resnet("up%d.%d" % (bi, ri), h, shape, p, zq16, zshape,
                                 groups, cache, new_cache)
            if "up" in blk:
                n, T, H, W = shape
                u = _ops.upsample_nearest(h.view(n, T, H, W, -1), blk["compress"], dt)
                shape = (n, u.shape[1], 2 * H, 2 * W)
                h = conv(u, blk["up"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        a = self._norm_act(h, shape, pk["norm_out"], zq16, zshape, groups)
        y = self._causal_conv("conv_out", a, pk["conv_out"], cache, new_cache,
                              epilogue=_lib.EPI_F32)
        n, T, H, W = shape
        return y.view(n, T, H, W, -1)[..., :self.config.out_channels], new_cache

    # -- encoder (opt-in, `with_encoder=True`) ---------------------------------------------------
    @torch.no_grad()
    def _pack_encoder(self):
        e = self.encoder
        dev = e.conv_in.conv.weight.device
        if dev.type != "cuda":
            raise RuntimeError("AutoencoderKLCogVideoX.encode runs on CUDA (sm_90a) only; "
                               "there is no CPU fallback.")
        dt = self.compute_dtype

        def res(m):
            p = dict(n1=pack_norm(m.norm1), c1=pack_conv(m.conv1.conv, dt, dev),
                     n2=pack_norm(m.norm2), c2=pack_conv(m.conv2.conv, dt, dev))
            if hasattr(m, "conv_shortcut"):
                p["sc"] = pack_linear(m.conv_shortcut.weight, m.conv_shortcut.bias, dt, dev)
            return p
        pk = dict(conv_in=pack_conv(e.conv_in.conv, dt, dev, pad_in=16), downs=[])
        for blk in e.down_blocks:
            b = dict(res=[res(r) for r in blk.resnets], compress=blk.compress_time)
            if hasattr(blk, "downsamplers"):
                b["down"] = pack_conv(blk.downsamplers[0].conv, dt, dev)
            pk["downs"].append(b)
        pk["mid"] = [res(r) for r in e.mid_block.resnets]
        pk["norm_out"] = pack_norm(e.norm_out)
        lc2 = 2 * self.config.latent_channels
        pk["conv_out"] = pack_conv(e.conv_out.conv, dt, dev, pad_out=(lc2 + 31) // 32 * 32)
        self._pk_enc = pk
        return pk

    def _gn_act(self, h, shape, p, groups):
        """GroupNorm + SiLU of fp32 `h` [rows, C] -> 16-bit time-padded conv input."""
        nb, T, H, W = shape
        C = h.shape[1]
        h5 = h.view(nb, T, H, W, C)
        sums = _ops.groupnorm_stats(h5, groups)
        out = torch.empty(nb, T + 2, H, W, C, device=h.device, dtype=self.compute_dtype)
        _ops.spatialnorm_silu(h5, sums, p[0], p[1], out, groups=groups, eps=p[2], out_t0=2,
                              silu=True)
        return out

    def _enc_resnet(self, name, h, shape, p, groups, cache, new_cache):
        a = self._gn_act(h, shape, p["n1"], groups)
        h1 = self._causal_conv(name + ".conv1", a, p["c1"], cache, new_cache,
                               epilogue=_lib.EPI_F32)
        b = self._gn_act(h1, shape, p["n2"], groups)
        if "sc" in p:
            h16 = torch.empty(h.shape, device=h.device, dtype=self.compute_dtype)
            _ops.act_cast(h, h16)
            skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
        else:
            skip = h
        return self._causal_conv(name + ".conv2", b, p["c2"], cache, new_cache,
                                 epilogue=_lib.EPI_RESID, resid=skip)

    def _downsample(self, h, shape, blk):
        """CogVideoXDownsample3D: pairwise temporal mean (an odd frame count keeps its first
        frame), then the stride-2 conv with right / bottom padding = the odd positions of a
        stride-1 'same' convolution."""
        nb, T, H, W = shape
        C = h.shape[1]
        h5 = h.view(nb, T, H, W, C)
        if blk["compress"] and T > 1:
            first = h5[:, :1] if T % 2 == 1 else None
            rest = h5[:, 1:] if T % 2 == 1 else h5
            pairs = rest.shape[1] // 2
            a = rest[:, 0:2 * pairs:2].contiguous()
            b = rest[:, 1:2 * pairs:2].contiguous()
            half = self.__dict__.get("_half")
            if half is None or half.device != h.device:
                half = self._half = torch.full((1,), 0.5, device=h.device)
            pooled = _ops.lincomb2(a, b, half, half, torch.empty_like(a))
            h5 = pooled if first is None else torch.cat([first, pooled], 1)
            T = h5.shape[1]
        x16 = torch.empty(nb, T, H, W, C, device=h.device, dtype=self.compute_dtype)
        _ops.act_cast(h5.contiguous(), x16)
        y = conv(x16, blk["down"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        y = y.view(nb, T, H, W, C)[:, :, 1::2, 1::2].contiguous()
        return y.view(-1, C), (nb, T, H // 2, W // 2)

    def _encode_chunk(self, x, cache):
        """x: fp32 channels-last frames [nb, T, H, W, 3] -> moments rows, shape, new cache."""
        pk, dt = self._pk_enc, self.compute_dtype
        groups = self.config.norm_num_groups
        nb, T, H, W, cin = x.shape
        new_cache = {}
        cp = pk["conv_in"].w.shape[2]
        xin = torch.zeros(nb, T + 2, H, W, cp, device=x.device, dtype=dt)
        xin[:, 2:, ..., :cin] = x
        h = self._causal_conv("enc.conv_in", xin, pk["conv_in"], cache, new_cache,
                              epilogue=_lib.EPI_F32)
        shape = (nb, T, H, W)
        for bi, blk in enumerate(pk["downs"]):
            for ri, p in enumerate(blk["res"]):
                h = self._enc_resnet("enc.down%d.%d" % (bi, ri), h, shape, p, groups, cache,
                                     new_cache)
            if "down" in blk:
                h, shape = self._downsample(h, shape, blk)
        for ri, p in enumerate(pk["mid"]):
            h = self._enc_resnet("enc.mid.%d" % ri, h, shape, p, groups, cache, new_cache)
        a = self._gn_act(h, shape, pk["norm_out"], groups)
        y = self._causal_conv("enc.conv_out", a, pk["conv_out"], cache, new_cache,
                              epilogue=_lib.EPI_F32)
        n, T, H, W = shape
        return y.view(n, T, H, W, -1)[..., :2 * self.config.latent_channels], new_cache

    @torch.no_grad()
    def encode(self, x, return_dict: bool = True):
        """x: [B, 3, T, H, W] frames in [-1, 1] -> `.latent_dist` (mode / sample), frames
        processed in chunks of 8 (the first chunk takes the remainder) with the causal-conv
        caches carried across chunks (diffusers 0.31 `_encode`; reference ctsd.py:1677-1700)."""
        if not hasattr(self, "encoder"):
            raise NotImplementedError("construct AutoencoderKLCogVideoX(with_encoder=True)")
        if not x.is_cuda:
            raise RuntimeError("AutoencoderKLCogVideoX.encode needs CUDA tensors; there is no "
                               "CPU fallback.")
        if self._pk_enc is None:
            self._pack_encoder()
        from dwm.models.autoencoder_kl import DiagonalGaussianDistribution
        xcl = x.float().permute(0, 2, 3, 4, 1).contiguous()
        fb = self.num_sample_frames_batch_size
        n = xcl.shape[1]
        cache, outs = {}, []
        for i in range(max(n // fb, 1)):
            rem = n % fb
            start = fb * i + (0 if i == 0 else rem)
            end = fb * (i + 1) + rem
            y, cache = self._encode_chunk(xcl[:, start:end].contiguous(), cache)
            outs.append(y)
        moments = torch.cat(outs, dim=1).permute(0, 4, 1, 2, 3).contiguous().to(x.dtype)
        dist = DiagonalGaussianDistribution(moments)
        if not return_dict:
            return (dist,)
        return _Cfg(latent_dist=dist)

    # -- public API ------------------------------------------------------------------------------
    @torch.no_grad()
    def decode(self, z, return_dict: bool = True):
        """z: [B, C, T, h, w] latents (already divided by scaling_factor by the caller)."""
        if not z.is_cuda:
            raise RuntimeError("AutoencoderKLCogVideoX.decode needs CUDA tensors; there "
                               "is no CPU fallback.")
        if self._pk is None:
            self._pack()
        zcl = z.float().permute(0, 2, 3, 4, 1).contiguous()   # channels-last
        fb = self.num_latent_frames_batch_size
        num_frames = zcl.shape[1]
        cache, outs = {}, []
        for i in range(max(num_frames // fb, 1)):
            rem = num_frames % fb
            start = fb * i + (0 if i == 0 else rem)
            end = fb * (i + 1) + rem
            y, cache = self._decode_chunk(zcl[:, start:end].contiguous(), cache)
            outs.append(y)
        dec = torch.cat(outs, dim=1).permute(0, 4, 1, 2, 3).contiguous().to(z.dtype)
        if not return_dict:
            return (dec,)
        return _Cfg(sample=dec)
