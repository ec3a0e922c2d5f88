"""Times the SD-3.5 2-D AutoencoderKL decode of one emitted 6-view frame
(6 x [16, 32, 56] latents -> 6 x [3, 256, 448]; reference ctsd.py:2095-2098), the decode
on the north-star streaming config's per-frame path (SURVEY.md §8(f)1)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "src"))
import torch
from dwm.models.autoencoder_kl import AutoencoderKL
from opendwm_b200 import ops

SD35_VAE = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512),
                layers_per_block=2, latent_channels=16, norm_num_groups=32,
                scaling_factor=1.5305, shift_factor=0.0609, use_quant_conv=False,
                use_post_quant_conv=False)


def decoder_flops(cfg, h, w):
    rev = list(reversed(cfg["block_out_channels"]))
    px = h * w
    f = 2 * px * 9 * cfg["latent_channels"] * rev[0]

    def res(cin, cout, px):
        return 2 * px * 9 * (cin * cout + cout * cout) + (2 * px * cin * cout if cin != cout else 0)
    f += 2 * res(rev[0], rev[0], px)
    c = rev[0]
    f += 2 * px * 4 * c * c + 4 * px * px * c          # q,k,v,out projections + QK^T + PV
    ch = rev[0]
    for i, out in enumerate(rev):
        for j in range(cfg["layers_per_block"] + 1):
            f += res(ch if j == 0 else out, out, px)
        ch = out
        if i != len(rev) - 1:
            px *= 4
            f += 2 * px * 9 * out * out
    f += 2 * px * 9 * rev[-1] * cfg["out_channels"]
    return f


def main():
    torch.manual_seed(0)
    views = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    with torch.device("cuda"):
        vae = AutoencoderKL(**SD35_VAE, compute_dtype=torch.bfloat16)
    z = torch.randn(views, 16, 32, 56, device="cuda").bfloat16()
    vae.decode(z, return_dict=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 5
    ops.profile_begin()
    e0.record()
    for _ in range(n):
        y = vae.decode(z, return_dict=False)[0]
    e1.record()
    torch.cuda.synchronize()
    prof = ops.profile_end()
    ms = e0.elapsed_time(e1) / n
    fl = decoder_flops(SD35_VAE, 32, 56) * views
    res = dict(workload="SD-3.5 AutoencoderKL decode, %d views 32x56 -> 256x448" % views,
               out_shape=list(y.shape), ms=ms, tflop=fl / 1e12, tflops=fl / ms / 1e9,
               launches=prof["launches"] / n, finite=bool(torch.isfinite(y.float()).all()))
    print(json.dumps(res))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "bench_out", "vae2d_bench.json"), "w"))


if __name__ == "__main__":
    main()
