"""CPU side of the FP8 VAE decoders: the gemm_dtype argument of both VAEs and its route through
from_pretrained and the pipeline's common_config["vae_gemm_dtype"], the layer selection of the
fake-quant oracle, and a self-test of the model-level bound of tests/test_fp8_vae_gpu.py: it
must reject a kernel that quantizes the cached tail with the previous chunk's scale and one
that uses the next volume's scale."""
import json

import pytest
import torch

import fp8_emulation as fe
import fp8_vae_emulation as fve

F8 = torch.float8_e4m3fn
SPEC = {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}


def _classes():
    from dwm.models.autoencoder_kl import AutoencoderKL
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    return ((AutoencoderKLCogVideoX, fve.COGVIDEOX, fve.cogvideox_oracle),
            (AutoencoderKL, fve.SD_KL, fve.autoencoder_kl_oracle))


def _checkpoint(tmp_path, name, cfg, oracle):
    import safetensors.torch
    d = tmp_path / name / "vae"
    d.mkdir(parents=True)
    with open(d / "config.json", "w") as f:
        json.dump(dict(cfg, _class_name=name), f)
    safetensors.torch.save_file(oracle().state_dict(), str(d / "diffusion_pytorch_model.safetensors"))
    return str(tmp_path / name)


def test_gemm_dtype_argument_and_from_pretrained(tmp_path):
    for cls, cfg, oracle in _classes():
        with pytest.raises(ValueError, match="gemm_dtype must be None or torch.float8_e4m3fn"):
            cls(**cfg, gemm_dtype=torch.float16)
        assert cls(**cfg).gemm_dtype is None
        assert cls(**cfg, gemm_dtype=F8).gemm_dtype is F8
        path = _checkpoint(tmp_path, cls.__name__, cfg, oracle)
        assert cls.from_pretrained(path, subfolder="vae").gemm_dtype is None
        v = cls.from_pretrained(path, subfolder="vae", gemm_dtype=F8)
        assert v.gemm_dtype is F8
        with pytest.raises(ValueError, match="gemm_dtype"):
            cls.from_pretrained(path, subfolder="vae", gemm_dtype=torch.bfloat16)
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            v.decode(torch.zeros(1, 16, 1, 4, 6) if "CogVideoX" in cls.__name__
                     else torch.zeros(1, 16, 8, 8))


def test_pipeline_vae_gemm_dtype_resolution(tmp_path):
    from dwm.pipelines.ctsd import load_vae
    for cls, cfg, oracle in _classes():
        path = _checkpoint(tmp_path, cls.__name__, cfg, oracle)
        assert load_vae(cls, path, {}).gemm_dtype is None
        assert load_vae(cls, path, {"vae_gemm_dtype": None}).gemm_dtype is None
        assert load_vae(cls, path, {"vae_gemm_dtype": SPEC}).gemm_dtype is F8
        assert load_vae(cls, path, {"vae_gemm_dtype": F8}).gemm_dtype is F8
        with pytest.raises(ValueError, match="gemm_dtype"):
            load_vae(cls, path, {"vae_gemm_dtype": {"_class_name": "get_class",
                                                    "class_name": "torch.float16"}})


def test_fake_quant_oracle_layer_selection():
    for oracle in (fve.cogvideox_oracle(), fve.autoencoder_kl_oracle()):
        names = fve.decoder_resnet_convs(oracle)
        # conv1 / conv2 of every decoder ResNet block (mid and up); no conv_in / conv_out,
        # upsampler, shortcut, SpatialNorm conv_y / conv_b or encoder conv
        assert names and all(n.startswith(("decoder.mid_block.resnets.", "decoder.up_blocks."))
                             and n.split(".")[-1] in ("conv1", "conv2") for n in names)
        n_res = sum(1 for n, _ in oracle.named_modules()
                    if n.startswith("decoder.") and n.split(".")[-2] == "resnets")
        assert len(names) == 2 * n_res


def test_model_bound_rejects_wrong_scales():
    """The bound the GPU test puts on the model, err <= 1.5 emu + spread with spread <=
    SPREAD_CAP, holds for the fake-quant oracle itself and fails for each wrong kernel on a
    multi-chunk CogVideoX clip (5 latent frames, chunks 3 + 2).  (The AutoencoderKL has no
    cache, and its GroupNorm leaves the images of a batch at one magnitude, so a wrong volume's
    scale moves its error too little for this bound to see.)"""
    z = fve.cogvideox_latents(2, 5, 4, 6)
    out = fve.cogvideox_outputs(fve.cogvideox_oracle(), z, torch.bfloat16, fve.BUGS)
    emu = fe.rel_err(out["fq"], out["ref"])
    bound = 1.5 * emu + fve.SPREAD_CAP
    errs = {b: fe.rel_err(out[b], out["ref"]) for b in fve.BUGS}
    print("cogvideox fake-quant error", emu, "wrong kernels", errs)
    assert 0 < emu < 0.1
    for b, e in errs.items():
        assert e > bound, (b, e, bound)
