"""Fake-quant oracle of the FP8 VAE decoders (gemm_dtype=torch.float8_e4m3fn).

The fp32 oracles oracle/cogvideox.py and oracle/autoencoder_kl.py with conv1 / conv2 of every
decoder ResNet block (mid and up blocks) computing on dequant(q(x)), one scale per volume, and
dequant(q(W)), one scale per output channel over all taps and input channels.  A volume is one
batch item of the conv input: a (b v) item of one CogVideoX chunk with its two leading cache
frames, one AutoencoderKL image.

The CogVideoX causal-conv cache follows the model's rule: the tail (the operand's last two
frames) is rounded to the compute dtype and kept; the next chunk's amax covers it and the new
frames, and the tail is quantized with that chunk's scale.  A first chunk's replicated frames
are copies of frame 0, under the same scale.

`bug` selects one of two wrong kernels for the CPU self-test: "previous chunk's scale" reuses
the previous chunk's E4M3 tail bytes under the new chunk's scale (amax over the new frames
only), "next volume's scale" dequantizes volume n with the scale of volume n + 1."""
import contextlib

import torch
import torch.nn.functional as F

import fp8_emulation as fe

BUGS = ("previous chunk's scale", "next volume's scale")


def decoder_resnet_convs(oracle):
    """conv1 / conv2 modules of the oracle's decoder ResNet blocks, by name (CogVideoX: the
    CausalConv3d wrappers)."""
    out = {}
    for name, m in oracle.named_modules():
        if name.startswith("decoder.") and name.endswith((".conv1", ".conv2")) and \
                ".resnets." in name:
            out[name] = m
    return out


def _quant(x, bug):
    """(q, scale) of x [nb, ...] with one scale per volume, and the dequantized x (with `bug`
    "next volume's scale": each volume dequantized with the next one's scale)."""
    q, s = fe.quantize_rows(x.reshape(x.shape[0], -1))
    q = q.float().reshape(x.shape)
    if bug == "next volume's scale":
        s = s.roll(-1)
    return q, s, q * s.view(-1, *[1] * (x.dim() - 1))


def _weight(m):
    w = m.weight.detach().float()
    return fe.fake_quant_rows(w.reshape(w.shape[0], -1)).reshape(w.shape)


@contextlib.contextmanager
def fake_quant_cogvideox(oracle, dtype, bug=None):
    """Within the block, the CogVideoX oracle's decoder ResNet convs compute in fake-quant FP8;
    the cache a converted conv hands on is its 16-bit (dtype) tail."""
    from oracle.cogvideox import CausalConv3d
    convs = set(decoder_resnet_convs(oracle).values())
    assert convs and all(isinstance(m, CausalConv3d) for m in convs)
    wq = {m: _weight(m.conv) for m in convs}
    orig = CausalConv3d.forward

    def forward(self, inputs, conv_cache=None):
        if self not in convs:
            return orig(self, inputs, conv_cache)
        if bug == "previous chunk's scale" and conv_cache is not None:
            # the previous chunk's bytes, under this chunk's scale of the new frames
            q_tail = conv_cache
            q_new, s, _ = _quant(inputs, None)
            q = torch.cat([q_tail, q_new], dim=2)
            x = q * s.view(-1, 1, 1, 1, 1)
        else:
            cached = [conv_cache] if conv_cache is not None else [inputs[:, :, :1]] * 2
            q, s, x = _quant(torch.cat(cached + [inputs], dim=2), bug)
        if bug == "previous chunk's scale":
            new_cache = q[:, :, -2:]
        else:
            new_cache = torch.cat(cached + [inputs], dim=2)[:, :, -2:].to(dtype).float()
        y = F.conv3d(F.pad(x, (1, 1, 1, 1)), wq[self].to(x.dtype), self.conv.bias)
        return y, new_cache

    CausalConv3d.forward = forward
    try:
        yield
    finally:
        CausalConv3d.forward = orig


@contextlib.contextmanager
def fake_quant_autoencoder_kl(oracle, bug=None):
    """Within the block, the AutoencoderKL oracle's decoder ResNet convs compute in fake-quant
    FP8 (one scale per image)."""
    convs = set(decoder_resnet_convs(oracle).values())
    assert convs and all(isinstance(m, torch.nn.Conv2d) for m in convs)
    wq = {m: _weight(m) for m in convs}
    orig = torch.nn.Conv2d.forward

    def forward(self, x):
        if self not in convs:
            return orig(self, x)
        return self._conv_forward(_quant(x, bug)[2], wq[self].to(x.dtype), self.bias)

    torch.nn.Conv2d.forward = forward
    try:
        yield
    finally:
        torch.nn.Conv2d.forward = orig


def cogvideox_outputs(oracle, z, dtype, bugs=()):
    """{"ref": fp32 decode, "fq": fake-quant decode, bug: wrong-kernel decode} of z [B, C, T, h, w]."""
    with torch.no_grad():
        out = {"ref": oracle.decode(z)}
        for b in (None,) + tuple(bugs):
            with fake_quant_cogvideox(oracle, dtype, b):
                out[b or "fq"] = oracle.decode(z)
    return out


def autoencoder_kl_outputs(oracle, z, bugs=()):
    """As cogvideox_outputs, for the AutoencoderKL oracle and latents z [n, C, h, w]."""
    with torch.no_grad():
        out = {"ref": oracle.decode(z, return_dict=False)[0]}
        for b in (None,) + tuple(bugs):
            with fake_quant_autoencoder_kl(oracle, b):
                out[b or "fq"] = oracle.decode(z, return_dict=False)[0]
    return out


# widths at which every decoder ResNet conv has C_out % 128 == 0 (the E4M3 conv1's F32 tiles)
COGVIDEOX = dict(block_out_channels=(128, 256), layers_per_block=1, norm_num_groups=32)
SD_KL = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256), layers_per_block=1,
             latent_channels=16, norm_num_groups=32, use_quant_conv=False,
             use_post_quant_conv=False)

# the bound of the model test: max|model - oracle| / max|oracle| <= 1.5 emu + spread, with the
# model's run-to-run spread asserted below SPREAD_CAP
SPREAD_CAP = 0.02


def cogvideox_latents(views, frames, h, w, seed=0):
    """Seeded latents [views, 16, frames, h, w] whose views and chunks (frames 0-2 / 3-4 of a
    5-frame clip) differ in magnitude, so a scale taken from the wrong volume or chunk shows."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(views, 16, frames, h, w, generator=g)
    z *= torch.tensor([1.0, 3.0, 0.5, 2.0, 1.5, 0.75][:views]).view(-1, 1, 1, 1, 1)
    if frames > 3:
        z[:, :, 3:] *= 4.0
    return z


def cogvideox_oracle(seed=0):
    """The CogVideoX decoder oracle at COGVIDEOX widths, parameters drawn as in
    tests/test_vae_gpu.py."""
    from oracle.cogvideox import AutoencoderKLCogVideoXDecoder
    torch.manual_seed(seed)
    o = AutoencoderKLCogVideoXDecoder(**COGVIDEOX)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in o.named_parameters():
            if p.dim() == 1 and "norm_layer.weight" in n:
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * p[0].numel() ** -0.5)
    return o.eval()


def autoencoder_kl_oracle(seed=0):
    from test_autoencoder_kl import _oracle
    return _oracle(SD_KL, seed)
