"""Parity at the REAL widths of BASELINE.json's other configs (VERDICT r01 weak #3: the UNet,
both VAEs and the row-wise-temporal DiT were only checked at toy widths).  Every case runs
the CUDA path and the fp32 oracle ON THE SAME GPU (TF32 off) with identical weights and inputs:

* config 2 — the full ctsd_21 UNet (block_out_channels 320/640/1280/1280: GroupNorm groups of
  10/20/40 channels, C_out = 320..1280 convolution tiles, 77-token cross-attention, row-wise
  cross-view attention over 6 views) on a CFG-doubled 6-view image batch [2,1,6,4,32,56];
* config 5 — the full CogVideoX decoder (128/256/256/512) on one view clip [16,5,32,56] ->
  17 frames 256x448: chunks of 3 + 2 latent frames with the causal caches, C_out = 128 tiles at
  256x448, SpatialNorm3D;
* north star / config 3 VAE — the full SD-3.5 AutoencoderKL decoder (128/256/512/512) on two
  views [16,32,56] -> 256x448, incl. the head_dim-512 mid attention;
* config 3 — ctsd_35 with row-wise cross-view AND row-wise temporal attention at D = 1536,
  T = 19 (sequence T*Wp = 532), 6 views, 2 joint blocks + one graft of each kind.

Tolerance is stated on the MODEL OUTPUT: max|y - ref| / max|ref|, fp16 operands (the
reference's own compute type).
"""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESULTS = {}


def _rel(y, ref):
    return ((y.float() - ref.float()).abs().max() / ref.float().abs().max()).item()


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _record(name, **kw):
    RESULTS[name] = kw


def _randomize(model, seed, scale=1.0):
    """Fan-in scaled weights (activations stay O(1) through the depth), non-trivial norms,
    biases and blend factors; rounded to fp16 so both paths hold identical values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith("mix_factor"):
                p.fill_(0.4)
            elif p.dim() == 1 and n.endswith(".weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g, device="cuda"))
            elif p.dim() == 1:
                p.copy_(0.02 * torch.randn(p.shape, generator=g, device="cuda"))
            else:
                p.copy_(torch.randn(p.shape, generator=g, device="cuda") *
                        (scale / p[0].numel()) ** 0.5)
            p.copy_(p.half().float())


def test_unet_config2_full_width():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from unet_bench import MODEL
    from oracle import unet as ounet
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    _no_tf32()
    dev = torch.device("cuda", 0)
    with torch.device(dev):
        o = ounet.UNetCrossviewTemporalConditionModel(**MODEL)
    o.to(dev).eval()
    _randomize(o, 1)
    with torch.device(dev):
        m = U(**MODEL, compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    B, T, V = 2, 1, 6
    g = torch.Generator().manual_seed(0)
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    x = torch.randn(B, T, V, 4, 32, 56, generator=g).to(dev)
    t = (torch.rand(B, T, V, generator=g) * 999).round().to(dev)
    cond = dict(
        encoder_hidden_states=(torch.randn(B, T, V, 77, 1024, generator=g) * 0.5).to(dev),
        condition_image_tensor=None,
        disable_crossview=torch.zeros(B, dtype=torch.bool, device=dev),
        disable_temporal=torch.ones(B, dtype=torch.bool, device=dev),
        crossview_attention_mask=ring.unsqueeze(0).repeat(B, 1, 1).to(dev),
        added_time_ids=torch.randn(B, T, V, 11, generator=g).to(dev))
    with torch.no_grad():
        ref = o(x, t, **cond)[0]
    del o
    torch.cuda.empty_cache()
    c16 = {k: (v.half() if v is not None and v.is_floating_point() else v)
           for k, v in cond.items()}
    y = m(x, t, **c16)[0][0]
    err = _rel(y, ref)
    _record("unet_config2", shape=list(x.shape), rel=err, ref_absmax=ref.abs().max().item())
    assert y.shape == ref.shape
    assert err < 8e-3, err


def test_cogvideox_decoder_full_width():
    from oracle import cogvideox as oc
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    _no_tf32()
    dev = torch.device("cuda", 0)
    with torch.device(dev):
        o = oc.AutoencoderKLCogVideoXDecoder()
    o.to(dev).eval()
    _randomize(o, 2, scale=1.5)
    with torch.device(dev):
        m = AutoencoderKLCogVideoX(compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    z = torch.randn(1, 16, 5, 32, 56, generator=torch.Generator().manual_seed(5)).to(dev)
    with torch.no_grad():
        ref = o.decode(z)
    del o
    torch.cuda.empty_cache()
    y = m.decode(z, return_dict=False)[0]
    err = _rel(y, ref)
    _record("cogvideox_decode", out_shape=list(y.shape), rel=err,
            ref_absmax=ref.abs().max().item())
    assert y.shape == ref.shape == (1, 3, 17, 256, 448)
    assert err < 8e-3, err


def test_autoencoder_kl_sd35_decoder_full_width():
    from oracle import autoencoder_kl as oa
    from dwm.models.autoencoder_kl import AutoencoderKL
    _no_tf32()
    dev = torch.device("cuda", 0)
    cfg = dict(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=16,
               norm_num_groups=32, scaling_factor=1.5305, shift_factor=0.0609,
               use_quant_conv=False, use_post_quant_conv=False)
    with torch.device(dev):
        o = oa.AutoencoderKL(**cfg)
    o.to(dev).eval()
    _randomize(o, 3, scale=1.5)
    with torch.device(dev):
        m = AutoencoderKL(**cfg, compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    z = torch.randn(2, 16, 32, 56, generator=torch.Generator().manual_seed(6)).to(dev)
    with torch.no_grad():
        ref = o.decode(z, return_dict=False)[0]
    del o
    torch.cuda.empty_cache()
    y = m.decode(z.half(), return_dict=False)[0]
    err = _rel(y, ref)
    _record("autoencoder_kl_sd35_decode", out_shape=list(y.shape), rel=err,
            ref_absmax=ref.abs().max().item())
    assert y.shape == ref.shape == (2, 3, 256, 448)
    assert err < 8e-3, err


def test_dit_rowwise_temporal_T19_full_width():
    from oracle import ctsd as octsd
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    _no_tf32()
    with open(os.path.join(ROOT, "tests", "golden", "example_pipeline_blocks.json")) as f:
        blk = json.load(f)["ctsd_35_6views_video_generation.json"]["pipeline"]["model"]
    cfg = {k: v for k, v in blk.items() if k != "_class_name"}
    cfg.update(num_layers=2, dual_attention_layers=[0], crossview_block_layers=[0],
               temporal_block_layers=[1], pos_embed_max_size=96)
    assert cfg["temporal_attention_type"] == "rowwise" and \
        cfg["crossview_attention_type"] == "rowwise"
    dev = torch.device("cuda", 0)
    with torch.device(dev):
        o = octsd.DiTCrossviewTemporalConditionModel(**cfg)
    o.to(dev).eval()
    _randomize(o, 4)
    with torch.device(dev):
        m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.float16)
    missing, unexpected = m.load_state_dict(o.state_dict(), strict=False)
    assert not missing and not unexpected, (missing[:4], unexpected[:4])
    B, T, V, C, H, W = 1, 19, 6, 16, 32, 56
    g = torch.Generator().manual_seed(7)
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    x = torch.randn(B, T, V, C, H, W, generator=g).to(dev)
    t = (torch.rand(B, T, V, generator=g) * 1000).to(dev)
    cond = dict(
        encoder_hidden_states=(torch.randn(B, T, V, 154, 4096, generator=g) * 0.2).to(dev),
        pooled_projections=torch.randn(B, T, V, 2048, generator=g).to(dev),
        condition_image_tensor=None,
        disable_crossview=torch.zeros(B, dtype=torch.bool, device=dev),
        disable_temporal=torch.zeros(B, dtype=torch.bool, device=dev),
        crossview_attention_mask=ring.unsqueeze(0).repeat(B, 1, 1).to(dev),
        added_time_ids=torch.randn(B, T, V, 11, generator=g).to(dev))
    with torch.no_grad():
        ref = o(x, t, **cond)[0][0]
    del o
    torch.cuda.empty_cache()
    c16 = {k: (v.half() if v is not None and v.is_floating_point() else v)
           for k, v in cond.items()}
    y = m(x, t, **c16)[0][0]
    err = _rel(y, ref)
    _record("dit_rowwise_T19", shape=list(x.shape), temporal_seq=T * (W // 2), rel=err,
            ref_absmax=ref.abs().max().item())
    assert y.shape == ref.shape
    assert err < 4e-3, err
