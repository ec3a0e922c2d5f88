"""Times the CogVideoX temporal-VAE decode of BASELINE config 5: per view 5 latent frames
[16, 5, 32, 56] -> 17 frames 256x448 (36.5 TFLOP per view-clip, SURVEY.md §8(a) A12),
`memory_efficient_batch` = 2 views per call like the reference example."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "src"))
import torch
from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
from opendwm_b200 import ops


def decoder_flops(vae, frames, h, w):
    """2*MAC of every convolution / 1x1 of the decoder for one view clip (chunked 3+2)."""
    import math
    cfgv = vae.config
    rev = list(reversed(cfgv.block_out_channels))
    total = 0.0
    fb, rem = 2, frames % 2
    chunks = [(0, min(frames, fb + rem))] + [(fb * i + rem, fb * (i + 1) + rem) for i in range(1, frames // fb)]
    for a, b in chunks:
        T, H, W = b - a, h, w
        total += 2 * T * H * W * 27 * cfgv.latent_channels * rev[0]
        def res(cin, cout, T, H, W):
            f = 2 * T * H * W * 27 * (cin * cout + cout * cout)
            if cin != cout:
                f += 2 * T * H * W * cin * cout
            return f
        for _ in range(2):
            total += res(rev[0], rev[0], T, H, W)
        ch = rev[0]
        level = int(math.log2(cfgv.temporal_compression_ratio))
        for i, out in enumerate(rev):
            for j in range(cfgv.layers_per_block + 1):
                total += res(ch if j == 0 else out, out, T, H, W)
            ch = out
            if i != len(rev) - 1:
                if i < level:
                    T = (1 + 2 * (T - 1)) if (T > 1 and T % 2 == 1) else (2 * T if T > 1 else 1)
                H, W = 2 * H, 2 * W
                total += 2 * T * H * W * 9 * out * out
        total += 2 * T * H * W * 27 * rev[-1] * cfgv.out_channels
    return total


def main():
    torch.manual_seed(0)
    views = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    with torch.device("cuda"):
        vae = AutoencoderKLCogVideoX(compute_dtype=torch.bfloat16)
    z = torch.randn(views, 16, 5, 32, 56, device="cuda")
    vae.decode(z, return_dict=False)   # warm-up (packs weights)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ops.profile_begin()
    e0.record()
    y = vae.decode(z, return_dict=False)[0]
    e1.record()
    torch.cuda.synchronize()
    prof = ops.profile_end()
    ms = e0.elapsed_time(e1)
    fl = decoder_flops(vae, 5, 32, 56) * views
    res = dict(views=views, out_shape=list(y.shape), ms=ms, tflop=fl / 1e12,
               tflops=fl / ms / 1e9, launches=prof["launches"],
               ms_per_6view_window=ms * 6 / views)
    print(json.dumps(res))
    os.makedirs("bench_out", exist_ok=True)
    json.dump(res, open("bench_out/vae_bench.json", "w"))


if __name__ == "__main__":
    main()
