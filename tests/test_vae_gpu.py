"""Parity of the H100-native CogVideoX decoder against the fp32 oracle restatement:
single chunk, chunked decode with causal caches (odd and even frame counts), the
diffusion-forcing single-frame decode, and state_dict key parity."""
import pytest
import torch

CFG = dict(block_out_channels=(32, 64, 64, 128), layers_per_block=1, norm_num_groups=8)


def _pair(dtype):
    from oracle import cogvideox as oc
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    torch.manual_seed(0)
    o = oc.AutoencoderKLCogVideoXDecoder(**CFG)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n, p in o.named_parameters():
            if p.dim() == 1 and "norm_layer.weight" in n:
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            else:
                fan = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * fan ** -0.5)
    m = AutoencoderKLCogVideoX(**CFG, compute_dtype=dtype)
    return o, m


def test_state_dict_keys_cpu():
    o, m = _pair(torch.bfloat16)
    so, sm = o.state_dict(), m.state_dict()
    assert set(so) == set(sm), sorted(set(so) ^ set(sm))[:8]
    for k in so:
        assert so[k].shape == sm[k].shape, k
    z = torch.randn(1, 16, 3, 4, 6)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.decode(z)


@pytest.mark.gpu
@pytest.mark.parametrize("frames,dtype,tol", [
    (1, torch.float16, 5e-3), (2, torch.float16, 5e-3), (3, torch.bfloat16, 3e-2),
    (5, torch.float16, 5e-3), (5, torch.bfloat16, 3e-2)])
def test_decode_matches_oracle(frames, dtype, tol):
    o, m = _pair(dtype)
    m.load_state_dict(o.state_dict())
    o, m = o.cuda(), m.cuda()
    g = torch.Generator().manual_seed(frames)
    z = torch.randn(2, 16, frames, 4, 7, generator=g).cuda()
    with torch.no_grad():
        ref = o.decode(z)
    y = m.decode(z, return_dict=False)[0]
    assert y.shape == ref.shape and y.shape[0] == 2 and y.shape[-2:] == (32, 56)
    err = ((y.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < tol, err


# -- encoder (opt-in `with_encoder=True`) ---------------------------------------------------------

def _enc_pair(dtype):
    from oracle import cogvideox as oc
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    torch.manual_seed(0)
    o = oc.AutoencoderKLCogVideoXEncoder(**CFG)
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for n, p in o.named_parameters():
            if p.dim() == 1 and n.endswith(".weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * (1.5 / p[0].numel()) ** 0.5)
    m = AutoencoderKLCogVideoX(**CFG, compute_dtype=dtype, with_encoder=True)
    return o, m


def test_encoder_state_dict_keys_cpu():
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    o, m = _enc_pair(torch.bfloat16)
    plain = AutoencoderKLCogVideoX(**CFG)
    assert not any(k.startswith("encoder.") for k in plain.state_dict())     # default unchanged
    so = o.state_dict()
    sm = {k: v for k, v in m.state_dict().items() if k.startswith("encoder.")}
    assert set(so) == set(sm)
    for k in so:
        assert so[k].shape == sm[k].shape, k
    m.load_state_dict({**plain.state_dict(), **so}, strict=True)
    with pytest.raises(NotImplementedError):
        plain.encode(torch.zeros(1, 3, 1, 32, 48))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.encode(torch.zeros(1, 3, 1, 32, 48))
    # frame arithmetic of the oracle: 1 -> 1, 9 -> 3, 17 -> 5 latent frames
    with torch.no_grad():
        for t, tz in ((1, 1), (9, 3), (17, 5)):
            assert o.encode_mode(torch.zeros(1, 3, t, 16, 16)).shape == (1, 16, tz, 2, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("frames", [1, 9, 17])
def test_encode_matches_oracle(frames):
    o, m = _enc_pair(torch.float16)
    o = o.cuda()
    sd = dict(m.state_dict())
    sd.update(o.state_dict())
    m.load_state_dict(sd)
    m.cuda()
    g = torch.Generator().manual_seed(frames)
    x = (torch.rand(2, 3, frames, 32, 48, generator=g) * 2 - 1).cuda().half()
    with torch.no_grad():
        ref = o.encode_moments(x.float())
    d = m.encode(x).latent_dist
    assert d.parameters.shape == ref.shape
    err = ((d.parameters.float() - ref).abs().max() / ref.abs().max()).item()
    assert err < 8e-3, err


def test_from_pretrained_builds_the_encoder_when_the_checkpoint_has_one_cpu(tmp_path):
    """diffusers' AutoencoderKLCogVideoX always has an encoder; the mirror builds (and strictly
    loads) it whenever the checkpoint carries `encoder.*` weights, and stays decoder-only for a
    decoder-only checkpoint."""
    import json
    import safetensors.torch
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    full = AutoencoderKLCogVideoX(**CFG, with_encoder=True)
    g = torch.Generator().manual_seed(3)
    state = {k: torch.randn(v.shape, generator=g) for k, v in full.state_dict().items()}
    for sub, keep in (("both", lambda k: True), ("dec", lambda k: k.startswith("decoder."))):
        d = tmp_path / sub / "vae"
        d.mkdir(parents=True)
        with open(d / "config.json", "w") as f:
            json.dump(dict(CFG, _class_name="AutoencoderKLCogVideoX", scaling_factor=1.15258426), f)
        safetensors.torch.save_file({k: v for k, v in state.items() if keep(k)},
                                    str(d / "diffusion_pytorch_model.safetensors"))
    v = AutoencoderKLCogVideoX.from_pretrained(str(tmp_path / "both"), subfolder="vae")
    assert hasattr(v, "encoder")
    sd = v.state_dict()
    assert set(sd) == set(state)
    assert all(torch.equal(sd[k], state[k]) for k in state)
    v2 = AutoencoderKLCogVideoX.from_pretrained(str(tmp_path / "dec"), subfolder="vae")
    assert not hasattr(v2, "encoder")
    assert torch.equal(v2.state_dict()["decoder.conv_in.conv.weight"],
                       state["decoder.conv_in.conv.weight"])
