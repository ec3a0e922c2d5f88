"""2-D `AutoencoderKL` — decode path, H100-native (SURVEY.md §8(f)1).

Mirror of the part of diffusers==0.31.0 `AutoencoderKL` the reference uses at every
emitted frame of the SD-2.1 / SD-3.5 image-VAE configs
(`vae.decode(latents / scaling_factor + shift_factor, return_dict=False)[0]`, reference
src/dwm/pipelines/ctsd.py:1633-1640 and :2095-2098, VAE built at :953-964).  Same
constructor / config keys, `from_pretrained(path, subfolder="vae")`, state_dict key names
(`decoder.*`, `post_quant_conv.*`; encoder / quant_conv keys are ignored: encode is not on
the path).

Execution: activations are channels-last; every 3x3 convolution is the im2col-free wgmma
kernel (`dwm_b200_conv`, taps iterated inside the MMA loop, zero padding = TMA OOB fill)
with the residual add as its epilogue; GroupNorm + SiLU is one statistics pass plus one
fused apply pass that emits the next convolution's 16-bit input; nearest x2 upsampling
writes the upsampler convolution's 16-bit input directly; the 1x1 shortcuts and the
mid-block attention projections run on the wgmma GEMM.  The single-head (head_dim 512)
mid-block attention is computed per image as S = Q K^T (GEMM, fp32 out), a row softmax
kernel, and O = P V against V^T, which the V projection produces directly
(V^T = W_v X^T); the V bias commutes with the softmax average and is folded into the
output-projection bias.

gemm_dtype=torch.float8_e4m3fn runs conv1 / conv2 of every decoder ResNet block (mid and up
blocks) in E4M3, with one activation scale per image and one weight scale per output channel;
conv_in / conv_out, the upsampler convs, the shortcuts, the mid-block attention and the encoder
stay 16-bit.
"""
import json
import math
import os

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops

from .packing import (
    FP8, Linear, Operand, conv, fp32, gemm, pack_conv, pack_linear, pack_norm)


class _Cfg(dict):
    __getattr__ = dict.get


class _P(torch.nn.Module):
    pass


def _resnet(cin, cout, groups):
    m = _P()
    m.norm1 = torch.nn.GroupNorm(groups, cin, eps=1e-6)
    m.conv1 = torch.nn.Conv2d(cin, cout, 3, padding=1)
    m.norm2 = torch.nn.GroupNorm(groups, cout, eps=1e-6)
    m.conv2 = torch.nn.Conv2d(cout, cout, 3, padding=1)
    if cin != cout:
        m.conv_shortcut = torch.nn.Conv2d(cin, cout, 1)
    return m


def _attention(channels, groups):
    m = _P()
    m.group_norm = torch.nn.GroupNorm(groups, channels, eps=1e-6)
    m.to_q = torch.nn.Linear(channels, channels)
    m.to_k = torch.nn.Linear(channels, channels)
    m.to_v = torch.nn.Linear(channels, channels)
    m.to_out = torch.nn.ModuleList([torch.nn.Linear(channels, channels)])
    return m


def _pack_resnet(m, dt, dev, fp8=False):
    p = dict(n1=pack_norm(m.norm1), c1=pack_conv(m.conv1, dt, dev, fp8), n2=pack_norm(m.norm2),
             c2=pack_conv(m.conv2, dt, dev, fp8))
    if hasattr(m, "conv_shortcut"):
        p["sc"] = pack_linear(m.conv_shortcut.weight, m.conv_shortcut.bias, dt, dev)
    return p


def _pack_attention(a, dt, dev):
    """q|k as one Linear, the V projection weight (the A operand of V^T = W_v X^T) and the
    output Linear with the V bias folded into its bias."""
    out = pack_linear(a.to_out[0].weight, a.to_out[0].bias, dt, dev)
    # softmax rows sum to 1: P (V + 1 b_v^T) = P V + b_v^T  =>  fold b_v into b_o
    bo = out.b + a.to_out[0].weight.detach().float().to(dev) @ fp32(a.to_v.bias.to(dev))
    return dict(gn=pack_norm(a.group_norm),
                qk=pack_linear(torch.cat([a.to_q.weight, a.to_k.weight]),
                               torch.cat([a.to_q.bias, a.to_k.bias]), dt, dev),
                wv=pack_linear(a.to_v.weight, None, dt, dev).w,
                out=out._replace(b=bo.contiguous()))


class DiagonalGaussianDistribution:
    """mean | logvar along channels (diffusers vae.py)."""

    def __init__(self, parameters):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def mode(self):
        return self.mean

    def sample(self, generator=None):
        noise = torch.randn(self.mean.shape, generator=generator,
                            device=self.mean.device if generator is None or
                            generator.device.type == "cuda" else "cpu").to(self.mean)
        return self.mean + self.std * noise


class AutoencoderKL(torch.nn.Module):

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None,
                 up_block_types=None, block_out_channels=(64,), layers_per_block=1,
                 act_fn="silu", latent_channels=4, norm_num_groups=32, sample_size=32,
                 scaling_factor=0.18215, shift_factor=None, force_upcast=True,
                 use_quant_conv=True, use_post_quant_conv=True,
                 mid_block_add_attention=True, compute_dtype=torch.bfloat16, gemm_dtype=None,
                 **unused):
        """gemm_dtype=torch.float8_e4m3fn runs the decoder ResNet convolutions in E4M3 (see
        the module docstring); None keeps every convolution 16-bit."""
        super().__init__()
        if gemm_dtype not in (None, torch.float8_e4m3fn):
            raise ValueError(
                "gemm_dtype must be None or torch.float8_e4m3fn, got {!r}".format(gemm_dtype))
        if act_fn != "silu":
            raise NotImplementedError("AutoencoderKL act_fn {}".format(act_fn))
        boc = tuple(block_out_channels)
        self.config = _Cfg(
            in_channels=in_channels, out_channels=out_channels, block_out_channels=boc,
            layers_per_block=layers_per_block, latent_channels=latent_channels,
            norm_num_groups=norm_num_groups, scaling_factor=scaling_factor,
            shift_factor=shift_factor, use_quant_conv=use_quant_conv,
            use_post_quant_conv=use_post_quant_conv,
            mid_block_add_attention=mid_block_add_attention,
            down_block_types=tuple(down_block_types or ("DownEncoderBlock2D",) * len(boc)))
        self.compute_dtype = compute_dtype
        self.gemm_dtype = gemm_dtype
        self._ws8 = {}
        g = norm_num_groups
        rev = list(reversed(boc))
        d = _P()
        d.conv_in = torch.nn.Conv2d(latent_channels, rev[0], 3, padding=1)
        d.mid_block = _P()
        d.mid_block.resnets = torch.nn.ModuleList(
            [_resnet(rev[0], rev[0], g), _resnet(rev[0], rev[0], g)])
        # attention_head_dim = block_out_channels[-1] => one head (vae.py Decoder)
        d.mid_block.attentions = torch.nn.ModuleList(
            [_attention(rev[0], g)] if mid_block_add_attention else [])
        d.up_blocks = torch.nn.ModuleList()
        out = rev[0]
        for i, ch in enumerate(rev):
            prev, out = out, ch
            b = _P()
            b.resnets = torch.nn.ModuleList(
                [_resnet(prev if j == 0 else out, out, g)
                 for j in range(layers_per_block + 1)])
            if i != len(rev) - 1:
                up = _P()
                up.conv = torch.nn.Conv2d(out, out, 3, padding=1)
                b.upsamplers = torch.nn.ModuleList([up])
            d.up_blocks.append(b)
        d.conv_norm_out = torch.nn.GroupNorm(g, rev[-1], eps=1e-6)
        d.conv_out = torch.nn.Conv2d(rev[-1], out_channels, 3, padding=1)
        self.decoder = d
        if use_post_quant_conv:
            self.post_quant_conv = torch.nn.Conv2d(latent_channels, latent_channels, 1)
        # encoder (reference-frame conditioning, ctsd.py:1681-1700): same building blocks
        e = _P()
        e.conv_in = torch.nn.Conv2d(in_channels, boc[0], 3, padding=1)
        e.down_blocks = torch.nn.ModuleList()
        out = boc[0]
        for i, ch in enumerate(boc):
            prev, out = out, ch
            b = _P()
            b.resnets = torch.nn.ModuleList(
                [_resnet(prev if j == 0 else out, out, g) for j in range(layers_per_block)])
            if i != len(boc) - 1:
                dn = _P()
                dn.conv = torch.nn.Conv2d(out, out, 3, stride=2, padding=0)
                b.downsamplers = torch.nn.ModuleList([dn])
            e.down_blocks.append(b)
        e.mid_block = _P()
        e.mid_block.resnets = torch.nn.ModuleList(
            [_resnet(boc[-1], boc[-1], g), _resnet(boc[-1], boc[-1], g)])
        e.mid_block.attentions = torch.nn.ModuleList(
            [_attention(boc[-1], g)] if mid_block_add_attention else [])
        e.conv_norm_out = torch.nn.GroupNorm(g, boc[-1], eps=1e-6)
        e.conv_out = torch.nn.Conv2d(boc[-1], 2 * latent_channels, 3, padding=1)
        self.encoder = e
        if use_quant_conv:
            self.quant_conv = torch.nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self._pk = None
        self._pk_enc = None

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
        vae = cls(**cfg)
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
        vae.load_state_dict(state)
        return vae

    def _apply(self, fn, *a, **k):
        self._pk = self._pk_enc = None
        self._ws8 = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, assign=False):
        """Accepts full VAE checkpoints and decoder-only ones (missing encoder / quant_conv
        keys keep their initial values); the pre-0.20 attention names (query/key/value/
        proj_attn) are accepted like diffusers' `_convert_deprecated_attention_blocks` does."""
        self._pk = self._pk_enc = None
        self._ws8 = {}
        ren = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
        sd = {}
        for k, v in state_dict.items():
            parts = k.split(".")
            if "attentions" in parts and parts[-2] in ren:
                k = ".".join(parts[:-2] + [ren[parts[-2]], parts[-1]])
                if v.dim() == 4:
                    v = v.flatten(1)
            sd[k] = v
        own = super().state_dict()
        sd = {k: v for k, v in sd.items() if k in own or
              not (k.startswith("encoder.") or k.startswith("quant_conv."))}
        decoder_only = not any(k.startswith("encoder.") for k in sd)
        if decoder_only:
            for k, v in own.items():
                if k.startswith("encoder.") or k.startswith("quant_conv."):
                    sd.setdefault(k, v)
        return super().load_state_dict(sd, strict=strict, assign=assign)

    # -- weight packing --------------------------------------------------------------------
    @torch.no_grad()
    def _pack(self):
        d = self.decoder
        dev = d.conv_in.weight.device
        if dev.type != "cuda":
            raise RuntimeError("AutoencoderKL.decode runs on CUDA (sm_90a) only; there "
                               "is no CPU fallback.")
        dt = self.compute_dtype
        lc = self.config.latent_channels
        cp = (lc + 7) // 8 * 8
        if hasattr(self, "post_quant_conv"):
            # 1x1 conv as a GEMM whose N is padded to the 32-column tile granule; conv_in
            # then reads those 32 (zero-extended) channels
            cq = (lc + 31) // 32 * 32
            w = torch.zeros(cq, cp, device=dev, dtype=dt)
            w[:lc, :lc] = self.post_quant_conv.weight.detach().reshape(lc, lc).to(dev, dt)
            b = torch.zeros(cq, device=dev)
            b[:lc] = self.post_quant_conv.bias.detach().float()
            pk = dict(pq=Linear(w, b), conv_in=pack_conv(d.conv_in, dt, dev, pad_in=cq))
        else:
            pk = dict(conv_in=pack_conv(d.conv_in, dt, dev, pad_in=cp))
        fp8 = self.gemm_dtype is not None
        pk["mid"] = [_pack_resnet(r, dt, dev, fp8) for r in d.mid_block.resnets]
        pk["attn"] = None
        if len(d.mid_block.attentions):
            pk["attn"] = _pack_attention(d.mid_block.attentions[0], dt, dev)
        pk["ups"] = []
        for blk in d.up_blocks:
            b = dict(res=[_pack_resnet(r, dt, dev, fp8) for r in blk.resnets])
            if hasattr(blk, "upsamplers"):
                b["up"] = pack_conv(blk.upsamplers[0].conv, dt, dev)
            pk["ups"].append(b)
        pk["norm_out"] = pack_norm(d.conv_norm_out)
        co = self.config.out_channels
        pk["conv_out"] = pack_conv(d.conv_out, dt, dev, pad_out=(co + 31) // 32 * 32)
        self._pk = pk
        return pk

    # -- building blocks ---------------------------------------------------------------------
    def _norm(self, h, shape, p, silu):
        """GroupNorm (+SiLU) of fp32 rows [nb*H*W, C] -> 16-bit [nb, 1, H, W, C]."""
        nb, H, W = shape
        C = h.shape[1]
        h5 = h.view(nb, 1, H, W, C)
        groups = self.config.norm_num_groups
        sums = _ops.groupnorm_stats(h5, groups)
        out = torch.empty(nb, 1, H, W, C, device=h.device, dtype=self.compute_dtype)
        _ops.spatialnorm_silu(h5, sums, p[0], p[1], out, groups=groups, eps=p[2], silu=silu)
        return out

    def _norm_silu_operand(self, h, shape, g, c):
        """GroupNorm + SiLU of fp32 rows as the operand of conv c: 16-bit, or for an E4M3 c
        E4M3 with one scale per image (in a workspace kept across calls of one geometry)."""
        if c.scale is None:
            return self._norm(h, shape, g, True)
        nb, H, W = shape
        C = h.shape[1]
        h5 = h.view(nb, 1, H, W, C)
        groups = self.config.norm_num_groups
        sums = _ops.groupnorm_stats(h5, groups)
        ws = self._ws8.get((nb, H, W, C))
        if ws is None:
            ws = self._ws8[nb, H, W, C] = (
                torch.empty(nb, 1, H, W, C, device=h.device, dtype=FP8),
                torch.empty(nb, device=h.device, dtype=torch.float32))
        return Operand(*_ops.groupnorm_silu_e4m3(h5, sums, g[0], g[1], *ws, groups=groups,
                                                 eps=g[2], silu=True))

    def _resnet(self, h, shape, p):
        a = self._norm_silu_operand(h, shape, p["n1"], p["c1"])
        h1 = conv(a, p["c1"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        b = self._norm_silu_operand(h1, shape, p["n2"], p["c2"])
        if "sc" in p:
            h16 = torch.empty(h.shape, device=h.device, dtype=self.compute_dtype)
            _ops.act_cast(h, h16)
            skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
        else:
            skip = h
        return conv(b, p["c2"], kernel=(1, 3, 3), epilogue=_lib.EPI_RESID, resid=skip)

    def _attn(self, h, shape, p):
        nb, H, W = shape
        C, HW = h.shape[1], H * W
        if HW % 8:
            raise ValueError("AutoencoderKL mid attention needs H*W % 8 == 0 at latent "
                             "resolution (16-byte TMA pitch); got {}x{}".format(H, W))
        dt = self.compute_dtype
        xn = self._norm(h, shape, p["gn"], False).view(nb * HW, C)
        qk = gemm(xn, p["qk"])                                      # [P, 2C] 16-bit
        vt = _ops.linear(p["wv"], xn)                               # V^T [C, P]
        o = torch.empty(nb * HW, C, device=h.device, dtype=dt)
        s = torch.empty(HW, HW, device=h.device, dtype=torch.float32)
        pr = torch.empty(HW, HW, device=h.device, dtype=dt)
        scale = 1.0 / math.sqrt(C)                                  # one head of dim C
        for i in range(nb):
            r = slice(i * HW, (i + 1) * HW)
            _ops.linear(qk[r, :C], qk[r, C:], epilogue=_lib.EPI_F32, out=s)
            _ops.softmax_rows(s, scale, pr)
            _ops.linear(pr, vt[:, r], out=o[r])
        return gemm(o, p["out"], epilogue=_lib.EPI_RESID, resid=h)

    # -- encoder ---------------------------------------------------------------------------------
    @torch.no_grad()
    def _pack_encoder(self):
        """Packed separately (first `encode`), so the decode path never depends on it."""
        e = self.encoder
        dev = e.conv_in.weight.device
        if dev.type != "cuda":
            raise RuntimeError("AutoencoderKL.encode runs on CUDA (sm_90a) only; there is no "
                               "CPU fallback.")
        dt = self.compute_dtype
        # 16 = smallest validated C_in
        pk = dict(conv_in=pack_conv(e.conv_in, dt, dev, pad_in=16), downs=[])
        for blk in e.down_blocks:
            b = dict(res=[_pack_resnet(r, dt, dev) for r in blk.resnets])
            if hasattr(blk, "downsamplers"):
                b["down"] = pack_conv(blk.downsamplers[0].conv, dt, dev)
            pk["downs"].append(b)
        pk["mid"] = [_pack_resnet(r, dt, dev) for r in e.mid_block.resnets]
        pk["attn"] = None
        if len(e.mid_block.attentions):
            pk["attn"] = _pack_attention(e.mid_block.attentions[0], dt, dev)
        pk["norm_out"] = pack_norm(e.conv_norm_out)
        lc2 = 2 * self.config.latent_channels
        cq = (lc2 + 31) // 32 * 32
        pk["conv_out"] = pack_conv(e.conv_out, dt, dev, pad_out=cq)
        if hasattr(self, "quant_conv"):
            w = torch.zeros(cq, cq, device=dev, dtype=dt)
            w[:lc2, :lc2] = self.quant_conv.weight.detach().reshape(lc2, lc2).to(dev, dt)
            b = torch.zeros(cq, device=dev)
            b[:lc2] = self.quant_conv.bias.detach().float()
            pk["quant"] = Linear(w, b)
        self._pk_enc = pk
        return pk

    @torch.no_grad()
    def encode(self, x, return_dict: bool = True):
        """x: [n, 3, H, W] images in [-1, 1] -> `.latent_dist` with `mode()` / `sample()`
        (reference ctsd.py:1689-1700: `vae.encode(t).latent_dist.mode()`).  The stride-2
        down-sampling convolutions (right / bottom zero padding, no left / top padding) run as
        stride-1 'same' convolutions whose odd output positions are kept."""
        if not x.is_cuda:
            raise RuntimeError("AutoencoderKL.encode needs CUDA tensors; there is no CPU "
                               "fallback.")
        pk = self._pk_enc or self._pack_encoder()
        dt = self.compute_dtype
        nb, cin, H, W = x.shape
        if H % 2 ** (len(pk["downs"]) - 1) or W % 2 ** (len(pk["downs"]) - 1):
            raise ValueError("image size must be divisible by the VAE down-sampling factor")
        x16 = torch.zeros(nb, 1, H, W, pk["conv_in"].w.shape[2], device=x.device, dtype=dt)
        x16[..., :cin] = x.permute(0, 2, 3, 1).unsqueeze(1)
        h = conv(x16, pk["conv_in"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        shape = (nb, H, W)
        for blk in pk["downs"]:
            for p in blk["res"]:
                h = self._resnet(h, shape, p)
            if "down" in blk:
                n, H, W = shape
                h16 = torch.empty(h.shape, device=h.device, dtype=dt)
                _ops.act_cast(h, h16)
                y = conv(h16.view(n, 1, H, W, -1), blk["down"], kernel=(1, 3, 3),
                         epilogue=_lib.EPI_F32)
                C = y.shape[1]
                h = y.view(n, H, W, C)[:, 1::2, 1::2].contiguous().view(-1, C)
                shape = (n, H // 2, W // 2)
        h = self._resnet(h, shape, pk["mid"][0])
        if pk["attn"] is not None:
            h = self._attn(h, shape, pk["attn"])
        h = self._resnet(h, shape, pk["mid"][1])
        a = self._norm(h, shape, pk["norm_out"], True)
        if "quant" in pk:
            m16 = conv(a, pk["conv_out"], kernel=(1, 3, 3), epilogue=_lib.EPI_STORE)
            moments = gemm(m16, pk["quant"], epilogue=_lib.EPI_F32)
        else:
            moments = conv(a, pk["conv_out"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        n, H, W = shape
        lc = self.config.latent_channels
        moments = moments.view(n, H, W, -1)[..., :2 * lc].permute(0, 3, 1, 2).contiguous()
        dist = DiagonalGaussianDistribution(moments.to(x.dtype))
        if not return_dict:
            return (dist,)
        return _Cfg(latent_dist=dist)

    # -- public API ------------------------------------------------------------------------------
    @torch.no_grad()
    def decode(self, z, return_dict: bool = True, generator=None):
        """z: [n, C, h, w] latents (already divided by scaling_factor by the caller)."""
        if not z.is_cuda:
            raise RuntimeError("AutoencoderKL.decode needs CUDA tensors; there is no CPU "
                               "fallback.")
        if self._pk is None:
            self._pack()
        pk, dt = self._pk, self.compute_dtype
        nb, lc, H, W = z.shape
        cp = pk["pq"].w.shape[1] if "pq" in pk else pk["conv_in"].w.shape[2]
        x16 = torch.zeros(nb, 1, H, W, cp, device=z.device, dtype=dt)
        x16[..., :lc] = z.permute(0, 2, 3, 1).unsqueeze(1)
        if "pq" in pk:
            x16 = gemm(x16.view(-1, cp), pk["pq"]).view(nb, 1, H, W, -1)
        h = conv(x16, pk["conv_in"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        shape = (nb, H, W)
        h = self._resnet(h, shape, pk["mid"][0])
        if pk["attn"] is not None:
            h = self._attn(h, shape, pk["attn"])
        h = self._resnet(h, shape, pk["mid"][1])
        for blk in pk["ups"]:
            for p in blk["res"]:
                h = self._resnet(h, shape, p)
            if "up" in blk:
                n, H, W = shape
                u = _ops.upsample_nearest(h.view(n, 1, H, W, -1), False, dt)
                shape = (n, 2 * H, 2 * W)
                h = conv(u, blk["up"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        a = self._norm(h, shape, pk["norm_out"], True)
        y = conv(a, pk["conv_out"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        n, H, W = shape
        dec = y.view(n, H, W, -1)[..., :self.config.out_channels]\
            .permute(0, 3, 1, 2).contiguous().to(z.dtype)
        if not return_dict:
            return (dec,)
        return _Cfg(sample=dec)
