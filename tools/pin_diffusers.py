"""Pin-on-arrival of the diffusers-side arithmetic (VERDICT r01 item 8 / SURVEY.md §8(c)).

The reference pins `diffusers==0.31.0` (requirements.txt:6); the package is neither vendored
under /root/reference nor installable offline, so oracle/d31.py, oracle/cogvideox.py,
oracle/autoencoder_kl.py and the diffusers blocks inside oracle/unet.py are restatements whose
parity is UNPINNED (DESIGN.md §5).  The moment the real package is importable this script

 1. re-generates every reference golden from /root/reference/src running on the REAL diffusers
    (tests/golden/make_reference_golden.py with DWM_REAL_DIFFUSERS=1) and compares each tensor
    with the committed fixture (generated on the name shim that maps diffusers.* to oracle/d31.py):
    agreement to 1e-6 pins oracle/d31.py and the UNet blocks of oracle/unet.py;
 2. compares oracle/cogvideox.py and oracle/autoencoder_kl.py with diffusers'
    AutoencoderKLCogVideoX / AutoencoderKL (decode and encode) on shared seeded weights.

Exit code 0 = pinned, 1 = a mismatch, 2 = diffusers 0.31.0 is not importable (status quo).

    python tools/pin_diffusers.py
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-6


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _load_shards(d):
    import glob
    import safetensors.torch
    out = {}
    for f in sorted(glob.glob(os.path.join(d, "reference_outputs_*.safetensors"))):
        out.update(safetensors.torch.load_file(f))
    return out


def main():
    try:
        import diffusers
    except Exception as e:      # noqa: BLE001
        print("diffusers is not importable (%r): oracle/d31.py, oracle/cogvideox.py, "
              "oracle/autoencoder_kl.py, oracle/unet.py stay PARITY UNPINNED" % (e,))
        return 2
    stub = os.path.join(ROOT, "tests", "golden", "diffusers_stub")
    if os.path.abspath(os.path.dirname(os.path.dirname(diffusers.__file__))) == stub:
        print("only the name shim is importable as `diffusers`: parity unpinned")
        return 2
    if not diffusers.__version__.startswith("0.31"):
        print("diffusers %s found, the reference pins 0.31.0: not used for pinning" %
              diffusers.__version__)
        return 2
    import safetensors.torch
    import torch
    bad = 0
    # ---- 1. goldens regenerated on the real package -------------------------------------
    with tempfile.TemporaryDirectory() as tmp:
        env = dict(os.environ, DWM_REAL_DIFFUSERS="1", DWM_GOLDEN_OUT=tmp)
        subprocess.run([sys.executable, os.path.join(ROOT, "tests", "golden",
                                                     "make_reference_golden.py")],
                       check=True, env=env)
        new = _load_shards(tmp)
    old = _load_shards(os.path.join(ROOT, "tests", "golden"))
    for k in sorted(old):
        if k not in new:
            print("MISSING", k)
            bad += 1
            continue
        a, b = new[k], old[k]
        if a.dtype in (torch.bool, torch.uint8, torch.int32, torch.int64):
            ok, err = bool(torch.equal(a, b)), 0.0
        else:
            err = _rel(a, b)
            ok = a.shape == b.shape and err <= TOL
        print("%-40s %s rel %.2e" % (k, "ok " if ok else "BAD", err))
        bad += 0 if ok else 1
    # ---- 2. the two VAEs -------------------------------------------------------------------
    sys.path.insert(0, ROOT)
    from oracle import autoencoder_kl as oa, cogvideox as oc
    torch.manual_seed(0)
    cfg = dict(block_out_channels=(32, 64, 64, 128), layers_per_block=1, norm_num_groups=8)
    d = diffusers.AutoencoderKLCogVideoX(
        block_out_channels=cfg["block_out_channels"], layers_per_block=1, norm_num_groups=8,
        down_block_types=("CogVideoXDownBlock3D",) * 4, up_block_types=("CogVideoXUpBlock3D",) * 4)
    o_dec, o_enc = oc.AutoencoderKLCogVideoXDecoder(**cfg), oc.AutoencoderKLCogVideoXEncoder(**cfg)
    sd = d.state_dict()
    o_dec.load_state_dict({k: v for k, v in sd.items() if k.startswith("decoder.")}, strict=True)
    o_enc.load_state_dict({k: v for k, v in sd.items() if k.startswith("encoder.")}, strict=True)
    z = torch.randn(1, 16, 5, 4, 6)
    x = torch.rand(1, 3, 17, 32, 48) * 2 - 1
    with torch.no_grad():
        pairs = [("cogvideox.decode", o_dec.decode(z), d.decode(z).sample),
                 ("cogvideox.encode", o_enc.encode_moments(x), d.encode(x).latent_dist.parameters)]
    for variant, kw in (("sd35", dict(latent_channels=16, use_quant_conv=False,
                                     use_post_quant_conv=False, shift_factor=0.0609)),
                        ("sd21", dict(latent_channels=4))):
        da = diffusers.AutoencoderKL(
            block_out_channels=(32, 64, 128, 128), layers_per_block=2, norm_num_groups=8,
            down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4,
            **kw)
        ok_ = oa.AutoencoderKL(block_out_channels=(32, 64, 128, 128), layers_per_block=2,
                               norm_num_groups=8, **kw)
        ok_.load_state_dict(da.state_dict(), strict=True)
        zz = torch.randn(2, kw["latent_channels"], 8, 12)
        xx = torch.rand(2, 3, 64, 96) * 2 - 1
        with torch.no_grad():
            pairs.append(("autoencoder_kl.%s.decode" % variant, ok_.decode(zz, return_dict=False)[0],
                          da.decode(zz).sample))
            pairs.append(("autoencoder_kl.%s.encode" % variant, ok_.encode(xx).latent_dist.mean,
                          da.encode(xx).latent_dist.mean))
    for name, a, b in pairs:
        err = _rel(a, b)
        ok = a.shape == b.shape and err <= 10 * TOL
        print("%-40s %s rel %.2e" % (name, "ok " if ok else "BAD", err))
        bad += 0 if ok else 1
    print("PINNED" if bad == 0 else "%d MISMATCHES" % bad)
    return 0 if bad == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
