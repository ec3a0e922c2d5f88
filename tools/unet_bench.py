"""Times one CFG-doubled denoise step of BASELINE config 2 (ctsd_21 6-view image generation,
examples/ctsd_21_6views_image_generation.json): UNetCrossviewTemporalConditionModel on
[2, 1, 6, 4, 32, 56] latents, text [2,1,6,77,1024], added_time_ids [...,11], ring cross-view
mask, disable_temporal (T = 1) + the fused CFG/DDIM update.  SURVEY.md §8(d): 680 GFLOP per
view-frame item, 8.16 TFLOP per step."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "src"))
import torch
from opendwm_b200 import ops

MODEL = dict(
    addition_time_embed_dim=256, block_out_channels=[320, 640, 1280, 1280],
    cross_attention_dim=1024, in_channels=4, layers_per_block=2,
    num_attention_heads=[5, 10, 20, 20], out_channels=4,
    projection_class_embeddings_input_dim=2816, sample_size=96,
    transformer_layers_per_block=1, enable_crossview=True, enable_rowwise_crossview=True,
    enable_temporal=True, enable_rowwise_temporal=True, merge_factor=2)
F_STEP_TFLOP = 8.16


def main():
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    dev = torch.device("cuda", 0)
    dtype = torch.bfloat16
    torch.manual_seed(0)
    with torch.device(dev):
        m = U(**MODEL, compute_dtype=dtype)
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("mix_factor"):
                continue
            if p.dim() == 1 and n.endswith(".weight"):
                p.fill_(1.0)
            elif n.endswith(".bias"):
                p.zero_()
            else:
                p.copy_(torch.randn(p.shape, generator=g, device="cuda") * 0.02)
    pipe = CrossviewTemporalSD(
        None, {"generator_seed": 0}, dev, {"frame_prediction_style": "ctsd"}, {},
        {"guidance_scale": 3, "inference_steps": 50}, None, m, model_dtype=dtype)
    pipe.test_scheduler.set_timesteps(50, dev)
    B, T, V = 1, 1, 6
    gen = torch.Generator().manual_seed(0)
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    cond = dict(
        encoder_hidden_states=(torch.randn(2 * B, T, V, 77, 1024, generator=gen) * 0.1).to(dev, dtype),
        condition_image_tensor=None,
        disable_crossview=torch.zeros(2 * B, dtype=torch.bool, device=dev),
        disable_temporal=torch.ones(2 * B, dtype=torch.bool, device=dev),
        crossview_attention_mask=ring.unsqueeze(0).repeat(2 * B, 1, 1).to(dev),
        added_time_ids=torch.randn(2 * B, T, V, 11, generator=gen).to(dev))
    lat = torch.randn(B, T, V, 4, 32, 56, generator=gen).to(dev)
    tsched = pipe.test_scheduler.timesteps

    ts_list = [tsched[k].to(torch.int32).expand(B, T, V).contiguous() for k in range(50)]

    def run(fn, count_launches):
        for k in range(3):
            fn(lat, cond, None, ts_list[k % 50], None)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if count_launches:
            ops.profile_begin()
        e0.record()
        for k in range(steps):
            fn(lat, cond, None, ts_list[(3 + k) % 50], None)
        e1.record()
        torch.cuda.synchronize()
        n = ops.profile_end()["launches"] / steps if count_launches else None
        return e0.elapsed_time(e1) / steps, n

    ms_eager, launches = run(pipe.denoise_step, True)
    if "nograph" in sys.argv:
        ms = ms_eager
    else:
        lat.normal_(generator=None)
        ms, _ = run(pipe.denoise_step_graphed, False)
    res = dict(workload="ctsd_21 6-view image step [2,1,6,4,32,56], CFG 3, DDIM", ms_per_step=ms,
               steps_per_s=1000.0 / ms, tflop_per_step=F_STEP_TFLOP,
               tflops=F_STEP_TFLOP / ms * 1e3, launches_per_step=launches,
               ms_per_step_without_cuda_graph=ms_eager,
               mode="CUDA-graph replay of the step (denoise_step_graphed)",
               finite=bool(torch.isfinite(lat).all()))
    print(json.dumps(res))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "bench_out", "unet_bench.json"), "w"))


if __name__ == "__main__":
    main()
