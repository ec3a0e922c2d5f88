"""Generates `tests/golden/reference_*.safetensors` by RUNNING THE REFERENCE'S OWN CODE.

Only works in the build container (needs /root/reference; nothing at test time does).
`diffusers` is not installable offline, so the reference modules are imported on top of the
name-mapping shim in tests/golden/diffusers_stub (every `diffusers.*` name the CTSD path
touches -> the fp32 restatement in oracle/d31.py).  What runs from /root/reference/src:

  dwm/models/crossview_temporal_dit.py   DiTCrossviewTemporalConditionModel (forward, both
                                         graft helpers, embeddings, un-patchify)
  dwm/models/crossview_temporal.py       VTSelfAttentionBlock, AlphaBlender, Mixer
  dwm/models/adapters.py                 ImageAdapter
  dwm/models/crossview_temporal_unet.py  UNetCrossviewTemporalConditionModel + its five block
                                         classes; crossview_temporal.py ResBlock,
                                         TransformerModel, TemporalBasicTransformerBlock
  dwm/pipelines/ctsd.py                  CrossviewTemporalSD.inference_pipeline (full-sequence
                                         loop, reference-frame injection, 3 configurations);
                                         StreamingCrossviewTemporalSD.reset_streaming +
                                         inference_pipeline (the diffusion-forcing loop, 3
                                         steps, CFG) and CrossviewTemporalSD.get_conditions /
                                         get_camera_transform_ids / get_action_ids, incl. its text
                                         branch (flatten_clip_text, sd3_encode_prompt_with_clip,
                                         sd3_encode_prompt_with_t5) on tiny seeded HF encoders;
                                         autoregressive_inference_pipeline (call traces with a
                                         stand-in inference_pipeline, four configurations);
                                         StreamingCrossviewTemporalSD.fifo_inference_pipeline /
                                         send_frame_condition / receive_frame (call + state
                                         trace over 7 frames)
  dwm/schedulers/temporal_independent.py FlowMatchEulerDiscreteScheduler.step_by_indices,
                                         DDIMScheduler.step, DDPMScheduler.add_noise /
                                         get_velocity (tensor timesteps)

The fixtures hold the reference outputs for seeded weights / inputs that the tests rebuild
deterministically (tests/common.py).  tests/test_reference_golden_cpu.py checks the oracle
restatement against them (bit-exact on the build host; 1e-6 elsewhere), which pins the
oracle's restatement of OpenDWM's own code.  Usage:  python tests/golden/make_reference_golden.py
"""
import glob
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference/src"
# order matters: the reference's `dwm`, not this repo's src/dwm mirror.  With
# DWM_REAL_DIFFUSERS=1 (tools/pin_diffusers.py) the name shim is left out and the reference runs
# on the real `diffusers` package; DWM_GOLDEN_OUT redirects the output files.
REAL = os.environ.get("DWM_REAL_DIFFUSERS", "0") == "1"
OUT = os.environ.get("DWM_GOLDEN_OUT", HERE)
sys.path[:0] = [REF] + ([] if REAL else [os.path.join(HERE, "diffusers_stub")]) + \
    [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from common import (AUTOREGRESSIVE_CASES, CONDITION_CASES, CONDITION_COMMON,  # noqa: E402
                    FULL_SEQUENCE_CASES, TINY, VARIANTS, full_sequence_inputs,
                    run_autoregressive_case, run_fifo_case, run_text_case, tiny_text_stack,
                    TEXT_CASES, PREVIEW_CASES, run_preview_case,
                    condition_batch, scheduler_inputs, seeded_oracle, synthetic_inputs,
                    variant_case)

def main():
    import safetensors.torch
    import dwm.models.crossview_temporal_dit as ref_dit
    import dwm.schedulers.temporal_independent as ref_sched
    assert ref_dit.__file__.startswith(REF), ref_dit.__file__
    torch.set_num_threads(1)                      # deterministic reduction order
    out, report = {}, {}
    for name in VARIANTS:
        cfg, sample, timestep, cond, extra = variant_case(name)
        oracle = seeded_oracle(cfg)
        ref = ref_dit.DiTCrossviewTemporalConditionModel(**cfg)
        missing, unexpected = ref.load_state_dict(oracle.state_dict(), strict=True)
        assert not missing and not unexpected
        ref.eval()
        with torch.no_grad():
            yr = ref(sample, timestep, **cond, **extra)
            yo = oracle(sample, timestep, **cond, **extra)
        yr = yr["noise_pred"] if extra else yr[0][0]
        yo = yo["noise_pred"] if extra else yo[0][0]
        out["dit_" + name] = yr.contiguous()
        report["dit_" + name] = {"shape": list(yr.shape), "absmax": yr.abs().max().item(),
                                 "oracle_max_abs_diff": (yr - yo).abs().max().item()}

    import dwm.models.crossview_temporal_unet as ref_unet
    from test_unet import UNET_CASES, _oracle as unet_oracle, unet_case
    assert ref_unet.__file__.startswith(REF), ref_unet.__file__
    for B, T, V, variant in UNET_CASES:
        cfg, x, t, c = unet_case(B, T, V, variant)
        oracle = unet_oracle(cfg)
        ref = ref_unet.UNetCrossviewTemporalConditionModel(**cfg)
        missing, unexpected = ref.load_state_dict(oracle.state_dict(), strict=True)
        assert not missing and not unexpected
        ref.eval()
        with torch.no_grad():
            yr = ref(x, t, **c)[0][0]
            yo = oracle(x, t, **c)[0]
        out["unet_" + variant] = yr.contiguous()
        report["unet_" + variant] = {"shape": list(yr.shape), "absmax": yr.abs().max().item(),
                                     "oracle_max_abs_diff": (yr - yo).abs().max().item()}

    # ---- the reference's own diffusion-forcing loop and condition builder -------------------
    import diffusers
    import dwm.pipelines.ctsd as ref_pipe
    from oracle import ctsd as octsd
    assert ref_pipe.__file__.startswith(REF), ref_pipe.__file__
    oracle = seeded_oracle(TINY)
    ref = ref_dit.DiTCrossviewTemporalConditionModel(**TINY)
    ref.load_state_dict(oracle.state_dict(), strict=True)
    ref.eval()

    class IdentityVae:                       # decode = identity: the loop's VAE call site runs
        class config:
            scaling_factor, shift_factor = 1.0, None
        dtype = torch.float32

        @staticmethod
        def decode(x, return_dict=False):
            return (x,)
    pipe = object.__new__(ref_pipe.StreamingCrossviewTemporalSD)   # no checkpoints to load
    pipe.common_config = {"frame_prediction_style": "diffusion_forcing"}
    pipe.inference_config = {"guidance_scale": 2.0, "inference_steps": 12,
                             "sequence_length_per_iteration": 4}
    pipe.device, pipe.model_dtype = torch.device("cpu"), torch.float32
    pipe.model = pipe.model_wrapper = ref
    pipe.test_scheduler = ref_sched.FlowMatchEulerDiscreteScheduler(
        num_train_timesteps=1000, shift=3.0)
    pipe.vae, pipe.image_processor = IdentityVae(), diffusers.image_processor.VaeImageProcessor()
    sample, _, cond = synthetic_inputs(TINY)
    shape = (1, 4, 3, 16, 8, 12)
    pipe.reset_streaming(shape, "pt")
    pipe.conditions, pipe.latents = cond, sample[:1].clone()
    with torch.no_grad():
        lat = pipe.inference_pipeline(shape, start_timestep=9, stop_timestep=12)
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(12)
    x = sample[:1].clone()
    for i in (9, 10, 11):
        x, _ = octsd.df_denoise_step(oracle, sched, x, cond, i=i, steps_per_inference=3,
                                     guidance_scale=2.0)
    out["pipe_df_latents_steps_9_10_11"] = lat.contiguous()
    out["pipe_df_frame"] = pipe.frames[0].contiguous()
    report["pipe_df_latents_steps_9_10_11"] = {
        "shape": list(lat.shape), "absmax": lat.abs().max().item(),
        "oracle_max_abs_diff": (lat - x).abs().max().item()}

    # ---- the reference's full-sequence inference_pipeline (ctsd.py:1439-1654): noise from the
    #      pipeline generator, get_conditions, scalar-timestep FlowMatch steps, reference-frame
    #      injection, final concatenation, VAE call site (identity VAE), post-processing.  Text
    #      comes pre-encoded: get_conditions is wrapped to add the batch's embeddings (uncond =
    #      zeros), everything else is the reference's ----------------------------------------------
    fcfg, fbatch, fcommon, fshape, f_image_latents = full_sequence_inputs()
    f_oracle = seeded_oracle(fcfg)
    f_ref = ref_dit.DiTCrossviewTemporalConditionModel(**fcfg)
    f_ref.load_state_dict(f_oracle.state_dict(), strict=True)
    f_ref.eval()
    f_ref.depth_net = None
    P = ref_pipe.CrossviewTemporalSD
    orig_gc = P.get_conditions

    def gc_with_text(model, te, tok, common_config, latent_shape, b, device, dtype, **kw):
        rc = orig_gc(model, None, None, common_config, latent_shape, b, device, dtype, **kw)
        t_, p_ = b["text_embeddings"].to(dtype), b["pooled_text_embeddings"].to(dtype)
        if kw.get("do_classifier_free_guidance"):
            t_ = torch.cat([torch.zeros_like(t_), t_])
            p_ = torch.cat([torch.zeros_like(p_), p_])
        rc["encoder_hidden_states"], rc["pooled_projections"] = t_, p_
        return rc
    for name, (inf, nref) in FULL_SEQUENCE_CASES.items():
        fp = object.__new__(P)
        fp.common_config, fp.inference_config = fcommon, inf
        fp.device, fp.model_dtype = torch.device("cpu"), torch.float32
        fp.model = fp.model_wrapper = f_ref
        fp.text_encoders = fp.tokenizers = None
        fp.generator = torch.Generator().manual_seed(0)
        fp.test_scheduler = ref_sched.FlowMatchEulerDiscreteScheduler(
            num_train_timesteps=1000, shift=3.0)
        fp.vae, fp.is_temporal_vae = IdentityVae(), False
        fp.image_processor = diffusers.image_processor.VaeImageProcessor()
        kw = dict(image_latents=f_image_latents, reference_frame_count=nref) if nref else {}
        if name == "no_cfg_partial":
            kw.update(start_timestep=1, stop_timestep=3)
        if name == "df_queue_partial":
            fp.common_config = dict(fcommon, frame_prediction_style="diffusion_forcing")
            kw = dict(image_latents=f_image_latents, reference_frame_count=3, start_timestep=2,
                      stop_timestep=4, take_time=1)
        P.get_conditions = staticmethod(gc_with_text)
        try:
            with torch.no_grad():
                fo = fp.inference_pipeline(fshape, fbatch, "pt", **kw)
        finally:
            P.get_conditions = staticmethod(orig_gc)
        out["fullseq_%s_latents" % name] = fo["latents"].contiguous()
        out["fullseq_%s_images" % name] = fo["images"].contiguous()
        report["fullseq_" + name] = {"shape": list(fo["latents"].shape),
                                     "absmax": fo["latents"].abs().max().item()}

    batch = condition_batch()
    for name, (over, kw) in CONDITION_CASES.items():
        common = dict(CONDITION_COMMON, **over)
        rc = ref_pipe.CrossviewTemporalSD.get_conditions(
            ref, None, None, common, shape, batch, "cpu", torch.float32, **kw)
        keys = []
        for k, v in rc.items():
            if v is not None:
                out["cond_%s_%s" % (name, k)] = (v.to(torch.uint8) if v.dtype == torch.bool
                                                 else v).contiguous()
                keys.append(k)
        report["cond_" + name] = {"keys": keys,
                                  "none_keys": [k for k, v in rc.items() if v is None]}

    si = scheduler_inputs()
    fm = ref_sched.FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, shift=3.0)
    fm.set_timesteps(12)
    out["fm_sigmas"] = fm.sigmas.clone()
    out["fm_timesteps"] = fm.timesteps.clone()
    out["fm_step_by_indices"] = fm.step_by_indices(
        si["model_output"], si["fm_indices"], si["sample"], return_dict=False)[0].contiguous()
    sd21 = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
                steps_offset=1)
    for pt in ("v_prediction", "epsilon", "sample"):
        ddim = ref_sched.DDIMScheduler(prediction_type=pt, **sd21)
        ddim.set_timesteps(50)
        out["ddim_step_" + pt] = ddim.step(
            si["model_output"], si["ddim_timesteps"], si["sample"],
            return_dict=False)[0].contiguous()
    out["ddim_timesteps_50"] = ddim.timesteps.clone()
    ddpm = ref_sched.DDPMScheduler(prediction_type="v_prediction", **sd21)
    out["ddpm_add_noise"] = ddpm.add_noise(si["sample"], si["noise"], si["ddpm_timesteps"]).contiguous()
    out["ddpm_get_velocity"] = ddpm.get_velocity(
        si["sample"], si["noise"], si["ddpm_timesteps"]).contiguous()

    # ---- orchestration of autoregressive_inference_pipeline (ctsd.py:1656-1833): how the
    #      reference drives inference_pipeline window after window, recorded with a stand-in ----
    traces = {name: run_autoregressive_case(ref_pipe.CrossviewTemporalSD, name)
              for name in AUTOREGRESSIVE_CASES}
    # streaming FIFO (ctsd.py:2012-2278): reset_streaming / send_frame_condition /
    # receive_frame / fifo_inference_pipeline with the real streaming-mode get_conditions
    traces["preview_dispatch"] = {
        name: run_preview_case(ref_pipe.CrossviewTemporalSD,
                               ref_pipe.StreamingCrossviewTemporalSD, name)
        for name in PREVIEW_CASES}
    traces["streaming_fifo"] = run_fifo_case(
        ref_pipe.StreamingCrossviewTemporalSD, object.__new__(diffusers.SD3Transformer2DModel))

    # ---- text branch of get_conditions (flatten_clip_text, sd3_encode_prompt_with_clip / _t5,
    #      CFG / mask handling, broadcast over frames and views) with tiny seeded HF encoders ------
    stack = tiny_text_stack()
    text = {name: run_text_case(
        ref_pipe.CrossviewTemporalSD,
        (diffusers.SD3Transformer2DModel, diffusers.UNetSpatioTemporalConditionModel), name, stack)
        for name in TEXT_CASES}
    with open(os.path.join(OUT, "reference_text_conditions.json"), "w") as f:
        json.dump(text, f, indent=1)

    # shards of at most ~900 KB, read back together by tests/test_reference_golden.py
    shards, size = [{}], 0
    for k in sorted(out):
        n = out[k].numel() * out[k].element_size()
        if size + n > 900_000:
            shards.append({})
            size = 0
        shards[-1][k] = out[k]
        size += n
    for old in glob.glob(os.path.join(OUT, "reference_outputs_*.safetensors")):
        os.remove(old)      # a shorter set of shards must not leave stale keys behind
    for i, shard in enumerate(shards):
        safetensors.torch.save_file(shard, os.path.join(OUT, "reference_outputs_%d.safetensors" % i))
    with open(os.path.join(OUT, "reference_autoregressive_traces.json"), "w") as f:
        json.dump(traces, f, indent=1)
    with open(os.path.join(OUT, "reference_outputs.json"), "w") as f:
        json.dump({"generated_from": "/root/reference/src (OpenDWM @ b0ecc3d) on " +
                                     ("the real diffusers package" if REAL else
                                      "the diffusers shim tests/golden/diffusers_stub"),
                   "torch": torch.__version__, "cases": report}, f, indent=1)
    for k, v in report.items():
        print(k, v)


if __name__ == "__main__":
    main()
