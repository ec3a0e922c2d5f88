"""ImageAdapter — layout-condition encoder (3D-box + HD-map images -> per-layer
residuals).  Mirror of reference src/dwm/models/adapters.py:6-60 with the T2I-Adapter
blocks of diffusers.models.adapter (AdapterBlock / AdapterResnetBlock).

The adapter does not depend on the latents or the timestep, yet the reference
re-runs it inside every denoising forward (crossview_temporal_dit.py:459-462).  Here
it is evaluated ONCE per condition set by the model's condition cache and its
residuals are kept in token layout.  Its 1x1 convolutions run on the wgmma GEMM,
its 3x3 convolutions on the im2col-free wgmma convolution (`dwm_b200_conv`, taps
iterated inside the MMA loop over the channels-last feature map); no cuDNN kernel is
involved.
"""
from typing import Optional

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops


class AdapterResnetBlock(torch.nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.block1 = torch.nn.Conv2d(channels, channels, 3, padding=1)
        self.act = torch.nn.ReLU()
        self.block2 = torch.nn.Conv2d(channels, channels, 1)


class AdapterBlock(torch.nn.Module):
    def __init__(self, in_channels, out_channels, num_res_blocks, down=False):
        super().__init__()
        self.downsample = torch.nn.AvgPool2d(2, 2, ceil_mode=True) \
            if down else None
        self.in_conv = torch.nn.Conv2d(in_channels, out_channels, 1) \
            if in_channels != out_channels else None
        self.resnets = torch.nn.Sequential(
            *[AdapterResnetBlock(out_channels) for _ in range(num_res_blocks)])


class ImageAdapter(torch.nn.Module):
    def __init__(
        self, in_channels: int = 3,
        channels: list = [320, 320, 640, 1280, 1280],
        is_downblocks: list = [False, True, True, True, False],
        num_res_blocks: int = 2, downscale_factor: int = 8,
        use_zero_convs: bool = False, zero_gate_coef: Optional[float] = None,
        gradient_checkpointing: bool = True
    ):
        super().__init__()
        if zero_gate_coef:
            raise NotImplementedError("zero_gate_coef is unused by CTSD configs")
        self.downscale_factor = downscale_factor
        in_channels = in_channels * downscale_factor ** 2
        self.unshuffle = torch.nn.PixelUnshuffle(downscale_factor)
        self.body = torch.nn.ModuleList([
            AdapterBlock(
                in_channels if i == 0 else channels[i - 1], channels[i],
                num_res_blocks, down=is_downblocks[i])
            for i in range(len(channels))
        ])
        self.gradient_checkpointing = gradient_checkpointing
        self.zero_convs = torch.nn.ModuleList([
            torch.nn.Conv2d(channel, channel, 1) for channel in channels
        ]) if use_zero_convs else [None for _ in channels]
        for i in self.zero_convs:
            if i is not None:
                torch.nn.init.zeros_(i.weight)
                torch.nn.init.zeros_(i.bias)
        self.zero_gate_coef = zero_gate_coef
        self.zero_gates = None

    @torch.no_grad()
    def token_features(self, x: torch.Tensor, dtype, chunk_items: int = 48):
        """x: [..., C, H, W] condition images.  Returns a list of fp32 token-layout
        residuals [items*h*w, channels[i]] (the reference's features, flattened as
        `.flatten(0, 2).flatten(2).permute(0, 2, 1)` does at
        crossview_temporal_dit.py:491-494)."""
        x = x.flatten(0, -4)
        n_items = x.shape[0]
        outs = None
        for s in range(0, n_items, chunk_items):
            feats = self._chunk(x[s:s + chunk_items], dtype)
            if outs is None:
                outs = [[] for _ in feats]
            for o, f in zip(outs, feats):
                o.append(f)
        return [torch.cat(o) for o in outs]

    def _conv1x1(self, tok, conv, dtype, epilogue=_lib.EPI_STORE, **kw):
        w = conv.weight.detach().reshape(conv.out_channels, -1)\
            .to(dtype).contiguous()
        b = conv.bias.detach().float().contiguous()
        return _ops.linear(tok, w, b, epilogue=epilogue, **kw)

    def _chunk(self, x, dtype):
        dev = x.device
        n = x.shape[0]
        # PixelUnshuffle + NCHW -> NHWC tokens: pure data movement
        x = torch.nn.functional.pixel_unshuffle(x.float(), self.downscale_factor)
        feats = []
        h, w = x.shape[-2:]
        tok32 = x.permute(0, 2, 3, 1).reshape(n * h * w, -1).contiguous()
        for block, zero_conv in zip(self.body, self.zero_convs):
            if block.downsample is not None:
                c = tok32.shape[1]
                t = tok32.view(n, h, w, c).permute(0, 3, 1, 2)
                t = torch.nn.functional.avg_pool2d(t, 2, 2, ceil_mode=True)
                h, w = t.shape[-2:]
                tok32 = t.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()
            if block.in_conv is not None:
                k = tok32.shape[1]
                kp = (k + 7) // 8 * 8
                a = torch.zeros(tok32.shape[0], kp, dtype=dtype, device=dev)
                a[:, :k] = tok32.to(dtype)
                conv = block.in_conv
                wgt = torch.zeros(conv.out_channels, kp, dtype=dtype, device=dev)
                wgt[:, :k] = conv.weight.detach().reshape(conv.out_channels, -1)
                tok32 = _ops.linear(
                    a, wgt, conv.bias.detach().float().contiguous(),
                    epilogue=_lib.EPI_F32)
            for res in block.resnets:
                c1 = res.block1
                x5 = tok32.to(dtype).view(n, 1, h, w, -1)      # channels-last map
                hmid = _ops.conv(
                    x5, _ops.pack_conv_weight(c1.weight, dtype),
                    c1.bias.detach().float().contiguous(), kernel=(1, 3, 3),
                    epilogue=_lib.EPI_STORE, act=_lib.ACT_RELU)
                tok32 = self._conv1x1(hmid, res.block2, dtype,
                                      epilogue=_lib.EPI_RESID, resid=tok32)
            if zero_conv is not None:
                f = self._conv1x1(tok32.to(dtype), zero_conv, dtype,
                                  epilogue=_lib.EPI_F32)
            else:
                f = tok32.clone()
            feats.append(f)
        return feats
