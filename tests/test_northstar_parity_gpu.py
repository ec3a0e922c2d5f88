"""Parity at BASELINE.json's FULL north-star size (CTSD-3.5 DFoT 6 views x 16 frames,
CFG-doubled [2,16,6,16,32,56], 24 joint blocks + 18 graft blocks + adapter): one
diffusion-forcing denoise step of the bf16 CUDA path against the fp32 oracle run in eager
PyTorch on the same GPU (TF32 off) with identical weights, latents, indices and conditions.

north_star tolerance: per-step output (the updated latents) max-abs-rel error < 1e-3.
Both 16-bit compute types of the CUDA path are checked (fp16 is what the reference's
example config runs; bf16 is what bench.py times); the CFG-combined noise prediction
(42 blocks deep, guidance 2) is also reported and bounded.
"""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _native(cfg, dev, dtype, state=None):
    import bench
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    torch.set_default_dtype(dtype)
    try:
        with torch.device(dev):
            model = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
    finally:
        torch.set_default_dtype(torch.float32)
    if state is None:
        bench.init_weights_(model)
        with torch.no_grad():      # non-trivial blends: sigmoid(mix_factor) away from 0/1
            for n, p in model.named_parameters():
                if n.endswith("mix_factor"):
                    p.fill_(0.4)
    else:
        model.load_state_dict(state)
    return model


def test_northstar_step_matches_fp32_oracle():
    import bench
    from oracle import ctsd as octsd
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = bench.load_config()
    B, T, V, C, H, W = cfg["latent_shape"]
    steps = cfg["inference_steps"]
    spi = steps // T
    g = cfg["guidance_scale"]
    dev = torch.device("cuda", 0)
    model = _native(cfg, dev, torch.bfloat16)
    with torch.device(dev):
        oracle = octsd.DiTCrossviewTemporalConditionModel(**cfg["model"])
    missing, unexpected = oracle.load_state_dict(model.state_dict(), strict=False)
    assert not missing and not unexpected, (missing[:4], unexpected[:4])
    oracle.to(dev).eval()
    state = {k: v.clone() for k, v in oracle.state_dict().items()}   # bf16-exact values

    cond = bench.synthetic_conditions(cfg, 2 * B, T, V, dev, torch.bfloat16)
    lat0 = torch.randn(B, T, V, C, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    i = steps - 2
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(steps)
    sched.timesteps = sched.timesteps.to(dev)
    sched.sigmas = sched.sigmas.to(dev)
    cond32 = {k: (v.float() if v.is_floating_point() else v) for k, v in cond.items()}
    with torch.no_grad():
        ref, noise_ref = octsd.df_denoise_step(
            oracle, sched, lat0.clone(), cond32, i=i, steps_per_inference=spi, guidance_scale=g)
    del oracle
    torch.cuda.empty_cache()

    res = {"shape": [2 * B, T, V, C, H, W], "step_index": i, "guidance_scale": g,
           "noise_ref_absmax": noise_ref.abs().max().item()}
    for tag, dtype in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
        if dtype is not torch.bfloat16:
            del model
            torch.cuda.empty_cache()
            model = _native(cfg, dev, dtype, state)
        # model_dtype fp32: the step output is not re-rounded to 16 bits (the reference
        # rounds prev_sample to model_output.dtype; the oracle above runs in fp32)
        pipe = StreamingCrossviewTemporalSD(
            None, {"generator_seed": 0}, dev, {"frame_prediction_style": "diffusion_forcing"},
            {}, {"guidance_scale": g, "inference_steps": steps,
                 "sequence_length_per_iteration": T}, None, model, model_dtype=torch.float32)
        pipe.reset_streaming((B, T, V, C, H, W), "pt")
        idx, ts, in_range = pipe._df_step_tensors(i, T, spi, 0, B, V)
        lat = lat0.clone()
        c = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in cond.items()}
        pipe.denoise_step(lat, c, idx, ts, in_range)
        torch.cuda.synchronize()
        # the native path's CFG-combined prediction, recovered from its update
        ds = (sched.sigmas[idx.long() + 1] - sched.sigmas[idx.long()]).view(B, T, V, 1, 1, 1)
        noise = (lat - lat0) / ds
        d = noise - noise_ref
        res[tag] = {
            "latents_max_abs_rel": ((lat - ref).abs().max() / ref.abs().max()).item(),
            "noise_pred_max_abs_rel": (d.abs().max() / noise_ref.abs().max()).item(),
            "noise_pred_rms_rel": (d.pow(2).mean().sqrt() / noise_ref.pow(2).mean().sqrt()).item(),
            "latents_changed": (lat - lat0).abs().max().item()}
    print(json.dumps(res))
    for tag in ("bf16", "fp16"):
        assert res[tag]["latents_changed"] > 0
    # north_star: per-step output max-abs-rel error < 1e-3 — met in the reference's own
    # compute type (fp16 autocast, examples/ctsd_35_df16_...json) and in bf16; the CFG-combined
    # prediction (guidance 2 triples rounding noise) is bounded at the bf16 tolerance 3e-2 max
    # (bf16 rounds the operands to 8 mantissa bits, fp16 to 11: bf16 gets the looser bound)
    assert res["fp16"]["latents_max_abs_rel"] < 3e-4, res
    assert res["bf16"]["latents_max_abs_rel"] < 1e-3, res
    assert res["fp16"]["noise_pred_max_abs_rel"] < 5e-3, res
    assert res["bf16"]["noise_pred_max_abs_rel"] < 3e-2, res
