"""Packed weights and GEMM / convolution operands, in 16 bit or E4M3.

The one place that knows how a packed weight and an operand are represented.  A packed
linear or convolution carries its fp32 per-channel E4M3 scales next to the weight, and an
operand carries its fp32 E4M3 row (or volume) scales next to the tensor; in 16 bit the
scales are None.  `gemm`, `conv` and `layernorm` hand those fields to the kernels as they
are, so the model code runs either precision without a branch.
"""
from typing import NamedTuple, Optional

import torch

from opendwm_b200 import ops as _ops

FP8 = torch.float8_e4m3fn


class Linear(NamedTuple):
    """A packed linear: w [N, K] 16-bit or E4M3, b fp32 [N] or None, scale fp32 [N] (E4M3
    only) and out_dtype, the 16-bit type an E4M3 GEMM writes (None for 16 bit)."""
    w: torch.Tensor
    b: Optional[torch.Tensor] = None
    scale: Optional[torch.Tensor] = None
    out_dtype: Optional[torch.dtype] = None

    def rows(self, start, stop):
        """The linear of output channels [start, stop) (views of this one)."""
        return Linear(self.w[start:stop], None if self.b is None else self.b[start:stop],
                      None if self.scale is None else self.scale[start:stop], self.out_dtype)


class Conv(NamedTuple):
    """A packed convolution: tap-major w [taps, C_out, C_in] 16-bit or E4M3, b fp32 [C_out]
    (zero-padded to w's C_out) and scale fp32 [C_out] (E4M3 only)."""
    w: torch.Tensor
    b: torch.Tensor
    scale: Optional[torch.Tensor] = None


class Operand(NamedTuple):
    """A GEMM / convolution operand: x 16-bit, or E4M3 with its fp32 scales."""
    x: torch.Tensor
    scale: Optional[torch.Tensor] = None


def fp32(t):
    """t as a contiguous fp32 tensor on its device (None stays None)."""
    return None if t is None else t.detach().to(torch.float32).contiguous()


def pack_linear(w, b, dtype, device, fp8=False):
    """Linear of weight w (reshaped to [N, -1], so a 1x1 convolution's weight works too) and
    bias b: w cast to dtype, or with fp8 quantized to E4M3 with one scale per output channel
    from the weight's own precision, writing dtype."""
    w = w.detach().to(device).reshape(w.shape[0], -1)
    b = None if b is None else fp32(b.to(device))
    if fp8:
        w8, s = _ops.quantize_weight_rows(w)
        return Linear(w8, b, s, dtype)
    return Linear(w.to(dtype).contiguous(), b)


def pack_conv(m, dtype, device, fp8=False, pad_in=None, pad_out=None):
    """Conv of torch Conv2d / Conv3d m: tap-major weight cast to dtype (C_in / C_out zero-padded
    to pad_in / pad_out), or with fp8 E4M3 with one scale per output channel."""
    if fp8:
        w, s = _ops.pack_conv_weight_fp8(m.weight.to(device))
    else:
        w, s = _ops.pack_conv_weight(m.weight.to(device), dtype, pad_out_to=pad_out,
                                     pad_in_to=pad_in), None
    b = torch.zeros(w.shape[1], device=device)
    b[:m.out_channels] = m.bias.detach().float()
    return Conv(w, b, s)


def pack_norm(m):
    """(weight, bias, eps) of a LayerNorm / GroupNorm, weight and bias fp32."""
    return fp32(m.weight), fp32(m.bias), m.eps


def fp8_bytes_saved(pk):
    """Weight bytes the E4M3 Linears anywhere in pack pk save against 16-bit ones, their
    scales included."""
    if isinstance(pk, Linear):
        return 0 if pk.scale is None else \
            pk.w.numel() * (pk.out_dtype.itemsize - 1) - 4 * pk.scale.numel()
    if isinstance(pk, dict):
        pk = pk.values()
    elif not isinstance(pk, (list, tuple)):
        return 0
    return sum(fp8_bytes_saved(v) for v in pk)


def gemm(a, lin, **kw):
    """ops.linear of operand a (an Operand, or a bare 16-bit tensor) with Linear lin."""
    a_scale = None
    if isinstance(a, Operand):
        a, a_scale = a
    return _ops.linear(a, lin.w, lin.b, a_scale=a_scale, w_scale=lin.scale,
                       out_dtype=lin.out_dtype, **kw)


def conv(a, c, **kw):
    """ops.conv of operand a (an Operand, or a bare 16-bit tensor) with Conv c."""
    a_scale = None
    if isinstance(a, Operand):
        a, a_scale = a
    return _ops.conv(a, c.w, c.b, a_scale=a_scale, w_scale=c.scale, **kw)


def layernorm(src, dst, out2=None, **kw):
    """ops.layernorm of src into the Operands dst (and out2)."""
    if out2 is not None:
        kw.update(out2=out2.x, out2_scale=out2.scale)
    return _ops.layernorm(src, dst.x, out_scale=dst.scale, **kw)


def requantize(t, buf):
    """The 16-bit GEMM output t as the next GEMM's operand: t itself when buf is None (16
    bit), else t quantized to E4M3 with row scales into the leading rows / columns of the
    Operand buffer buf."""
    if buf is None:
        return t
    M, K = t.shape
    return Operand(*_ops.quantize_rows(t, buf.x[:M, :K], buf.scale[:M]))
