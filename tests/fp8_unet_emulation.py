"""Fake-quant oracle of the FP8 CTSD-2.1 UNet (gemm_dtype=torch.float8_e4m3fn).

The fp32 UNet oracle (oracle/unet.py) with
- every FP8 linear of the model computing dequant(q(x)) . dequant(q(W))^T + b, one scale per
  activation row and per weight row: the BasicTransformerBlock linears except the text K/V
  projections (attn2.to_k / to_v), and every linear of the cross-view / temporal blocks;
- every FP8 convolution (the spatial and temporal ResBlock conv1 / conv2) computing on an input
  quantized with ONE scale per volume (dim 0 of the conv input: the (b t v) item for the
  spatial convs, the (b v) volume of T frames for the temporal ones, the model's `nb`) and a
  weight quantized with one scale per output channel over all taps and input channels.
The quantizer is tests/fp8_emulation.py's, the one the kernels implement."""
import contextlib

import torch

import fp8_emulation as fe

_CONVS = ("spatial_res_block.conv1", "spatial_res_block.conv2",
          "temporal_res_block.conv1", "temporal_res_block.conv2")
_TEXT_KV = ("attn2.to_k", "attn2.to_v")


def fp8_modules(oracle):
    """(FP8 linears, FP8 convs) of the UNet oracle, by name."""
    lins, convs = {}, {}
    for name, m in oracle.named_modules():
        if isinstance(m, torch.nn.Linear) and "transformer_blocks." in name and \
                not name.endswith(_TEXT_KV):
            lins[name] = m
        elif isinstance(m, (torch.nn.Conv2d, torch.nn.Conv3d)) and name.endswith(_CONVS):
            convs[name] = m
    return lins, convs


def fake_quant_volumes(x):
    """dequant(q(x)) with one scale per x[n] (the whole volume)."""
    return fe.fake_quant_rows(x.reshape(x.shape[0], -1)).reshape(x.shape)


@contextlib.contextmanager
def fake_quant_unet(oracle):
    lins, convs = fp8_modules(oracle)
    assert lins and convs, "no FP8 layers found"
    lins, convs = set(lins.values()), set(convs.values())
    wq = {m: fe.fake_quant_rows(m.weight.detach().float().reshape(m.weight.shape[0], -1))
          .reshape(m.weight.shape) for m in lins | convs}
    lin_fwd, c2_fwd, c3_fwd = torch.nn.Linear.forward, torch.nn.Conv2d.forward, \
        torch.nn.Conv3d.forward

    def linear(self, x):
        if self in lins:
            return torch.nn.functional.linear(fe.fake_quant_rows(x), wq[self].to(x.dtype),
                                              self.bias)
        return lin_fwd(self, x)

    def conv2d(self, x):
        if self in convs:
            return self._conv_forward(fake_quant_volumes(x), wq[self].to(x.dtype), self.bias)
        return c2_fwd(self, x)

    def conv3d(self, x):
        if self in convs:
            return self._conv_forward(fake_quant_volumes(x), wq[self].to(x.dtype), self.bias)
        return c3_fwd(self, x)

    torch.nn.Linear.forward, torch.nn.Conv2d.forward, torch.nn.Conv3d.forward = \
        linear, conv2d, conv3d
    try:
        yield
    finally:
        torch.nn.Linear.forward, torch.nn.Conv2d.forward, torch.nn.Conv3d.forward = \
            lin_fwd, c2_fwd, c3_fwd


def emulated_error(oracle, sample, timesteps, cond):
    """(max|fake-quant - oracle| / max|oracle|, fp32 oracle output)."""
    with torch.no_grad():
        ref = oracle(sample, timesteps, **cond)[0]
        with fake_quant_unet(oracle):
            y = oracle(sample, timesteps, **cond)[0]
    return fe.rel_err(y, ref), ref


# full channel widths (320 / 640 / 1280) with one ResBlock per level, for a small latent
FULL_WIDTH = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280),
                  num_attention_heads=(5, 10, 20, 20), cross_attention_dim=96,
                  projection_class_embeddings_input_dim=11 * 256, layers_per_block=1,
                  enable_rowwise_crossview=True, enable_rowwise_temporal=True)
