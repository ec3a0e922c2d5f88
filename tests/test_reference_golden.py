"""Fixtures produced by RUNNING THE REFERENCE'S OWN CODE (tests/golden/make_reference_golden.py:
/root/reference/src/dwm models + schedulers imported on the diffusers name-mapping shim) pin

  * the oracle restatement (CPU, fp32): bit-exact on the build host, <= 1e-5 elsewhere;
  * the CUDA path (GPU): DiT forward in fp16 against the reference outputs directly, and the
    mirrored per-frame schedulers.

The fixtures do not need /root/reference at test time."""
import os

import pytest
import torch

from common import (AUTOREGRESSIVE_CASES, CONDITION_CASES, CONDITION_COMMON, FULL_SEQUENCE_CASES,
                    TINY, VARIANTS, full_sequence_inputs,
                    condition_batch, run_autoregressive_case, run_fifo_case, run_text_case,
                    TEXT_CASES, tiny_text_stack, PREVIEW_CASES, run_preview_case,
                    scheduler_inputs, seeded_oracle, synthetic_inputs, variant_case)

HERE = os.path.dirname(os.path.abspath(__file__))
SD21 = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
            beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
            steps_offset=1)


@pytest.fixture(scope="module")
def golden():
    import glob
    import safetensors.torch
    out = {}
    for f in sorted(glob.glob(os.path.join(HERE, "golden", "reference_outputs_*.safetensors"))):
        out.update(safetensors.torch.load_file(f))
    return out


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()


@pytest.mark.parametrize("name", VARIANTS)
def test_oracle_dit_matches_reference(name, golden):
    torch.set_num_threads(1)
    cfg, sample, timestep, cond, extra = variant_case(name)
    o = seeded_oracle(cfg)
    with torch.no_grad():
        y = o(sample, timestep, **cond, **extra)
    y = y["noise_pred"] if extra else y[0][0]
    ref = golden["dit_" + name]
    assert y.shape == ref.shape
    assert (y - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def _unet_cases():
    from test_unet import UNET_CASES
    return UNET_CASES


@pytest.mark.parametrize("B,T,V,variant", _unet_cases())
def test_oracle_unet_matches_reference(B, T, V, variant, golden):
    from test_unet import _oracle, unet_case
    torch.set_num_threads(1)
    cfg, x, t, c = unet_case(B, T, V, variant)
    with torch.no_grad():
        y = _oracle(cfg)(x, t, **c)[0]
    ref = golden["unet_" + variant]
    assert y.shape == ref.shape
    assert (y - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_oracle_schedulers_match_reference(golden):
    from oracle import ctsd as octsd
    si = scheduler_inputs()
    fm = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    fm.set_timesteps(12)
    assert torch.equal(fm.sigmas, golden["fm_sigmas"])
    assert torch.equal(fm.timesteps, golden["fm_timesteps"])
    y = fm.step_by_indices(si["model_output"], si["fm_indices"], si["sample"])
    assert torch.equal(y, golden["fm_step_by_indices"])
    for pt in ("v_prediction", "epsilon", "sample"):
        ddim = octsd.DDIMSchedulerOracle(prediction_type=pt, beta_start=0.00085, beta_end=0.012)
        ddim.set_timesteps(50)
        y = ddim.step(si["model_output"], si["ddim_timesteps"], si["sample"])
        assert torch.allclose(y, golden["ddim_step_" + pt], rtol=0, atol=2e-6), pt
    assert torch.equal(ddim.timesteps, golden["ddim_timesteps_50"])
    ddpm = octsd.DDPMSchedulerOracle(beta_start=0.00085, beta_end=0.012)
    assert torch.allclose(ddpm.add_noise(si["sample"], si["noise"], si["ddpm_timesteps"]),
                          golden["ddpm_add_noise"], rtol=0, atol=1e-6)
    assert torch.allclose(ddpm.get_velocity(si["sample"], si["noise"], si["ddpm_timesteps"]),
                          golden["ddpm_get_velocity"], rtol=0, atol=1e-6)


def test_oracle_df_loop_matches_reference_loop(golden):
    """Three iterations (i = 9, 10, 11 of 12; CFG 2.0) of the reference's
    StreamingCrossviewTemporalSD.inference_pipeline vs the oracle's df_denoise_step."""
    from oracle import ctsd as octsd
    torch.set_num_threads(1)
    o = seeded_oracle(TINY)
    sample, _, cond = synthetic_inputs(TINY)
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(12)
    x = sample[:1].clone()
    for i in (9, 10, 11):
        x, _ = octsd.df_denoise_step(o, sched, x, cond, i=i, steps_per_inference=3,
                                     guidance_scale=2.0)
    ref = golden["pipe_df_latents_steps_9_10_11"]
    assert (x - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    # the emitted frame = identity-VAE decode of the exiting latent frame, post-processed
    frame = (ref[:, 0].flatten(0, 1) / 2 + 0.5).clamp(0, 1)
    assert torch.allclose(frame, golden["pipe_df_frame"], atol=1e-6)


@pytest.mark.parametrize("name", list(CONDITION_CASES))
def test_mirror_get_conditions_matches_reference(name, golden):
    """The mirrored CrossviewTemporalSD.get_conditions / get_camera_transform_ids /
    get_action_ids (pure PyTorch host code) against the reference's own, key by key."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    over, kw = CONDITION_CASES[name]
    common = dict(CONDITION_COMMON, **over)
    model = DiTCrossviewTemporalConditionModel(**TINY)       # isinstance checks only
    batch = condition_batch()
    got = CrossviewTemporalSD.get_conditions(
        model, None, None, common, (1, 4, 3, 16, 8, 12), batch, "cpu", torch.float32, **kw)
    prefix = "cond_%s_" % name
    want = {k[len(prefix):]: v for k, v in golden.items() if k.startswith(prefix)}
    assert want, name
    for k, v in want.items():
        g = got[k]
        assert g is not None, k
        g = g.to(torch.uint8) if g.dtype == torch.bool else g
        assert g.shape == v.shape and g.dtype == v.dtype, (k, g.shape, v.shape, g.dtype)
        assert torch.allclose(g.float(), v.float(), rtol=1e-5, atol=1e-5), k
    for k, g in got.items():                                 # nothing extra is non-None
        if g is not None and k != "pooled_projections":
            assert k in want, k


@pytest.mark.parametrize("name", list(FULL_SEQUENCE_CASES))
def test_full_sequence_algorithm_matches_reference(name, golden):
    """The mirror's full-sequence step algorithm — reference frames written into the latents
    at timestep 0 before each step, Euler update of every frame, reference frames restored at
    the end — evaluated with the fp32 oracle model, the mirror's get_conditions and scheduler
    tables on the CPU, against the latents / images the reference's own inference_pipeline
    produced (which instead swaps the reference frames into the model input only)."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from oracle import ctsd as octsd
    torch.set_num_threads(1)
    inf, nref = FULL_SEQUENCE_CASES[name]
    cfg, batch, common, shape, image_latents = full_sequence_inputs()
    o = seeded_oracle(cfg)
    do_cfg = "guidance_scale" in inf
    cond = CrossviewTemporalSD.get_conditions(
        object.__new__(DiTCrossviewTemporalConditionModel), object(), None, common, shape,
        batch, "cpu", torch.float32, do_classifier_free_guidance=do_cfg)
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(inf["inference_steps"])
    lat = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    start, stop = (1, 3) if name == "no_cfg_partial" else (0, inf["inference_steps"])
    if name == "df_queue_partial":
        # diffusion-forcing branch: the queue comes in as image_latents, steps 2..3 of 6 with
        # take_time 1, the emitted frame is queue slot 1
        x = image_latents.clone()
        with torch.no_grad():
            for i in (2, 3):
                x, _ = octsd.df_denoise_step(o, sched, x, cond, i=i, steps_per_inference=2,
                                             guidance_scale=inf["guidance_scale"], take_time=1)
        ref = golden["fullseq_%s_latents" % name]
        assert (x - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
        img = (x[:, 1].flatten(0, 1) / 2 + 0.5).clamp(0, 1)
        assert torch.allclose(img, golden["fullseq_%s_images" % name], atol=1e-5)
        return
    with torch.no_grad():
        for i in range(start, stop):
            ts = sched.timesteps[i].expand(shape[:3]).clone()
            if nref:
                lat[:, :nref] = image_latents[:, :nref]
                ts[:, :nref] = 0
            x, t = (torch.cat([lat, lat]), torch.cat([ts, ts])) if do_cfg else (lat, ts)
            pred = o(x, t, **cond)[0][0]
            if do_cfg:
                u, c = pred.chunk(2)
                pred = u + inf["guidance_scale"] * (c - u)
            lat = lat + (sched.sigmas[i + 1] - sched.sigmas[i]) * pred
    if nref:
        lat = torch.cat([image_latents[:, :nref], lat[:, nref:]], 1)
    ref = golden["fullseq_%s_latents" % name]
    assert (lat - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    img = (lat.flatten(0, 2) / 2 + 0.5).clamp(0, 1)
    assert torch.allclose(img, golden["fullseq_%s_images" % name], atol=1e-5)


@pytest.mark.parametrize("name", list(AUTOREGRESSIVE_CASES))
def test_mirror_autoregressive_orchestration_matches_reference(name):
    """Window / queue orchestration of long sequences (full-sequence with reference frames,
    temporal-VAE frame arithmetic, diffusion-forcing warm-up / rotate / flush): the mirror
    must call inference_pipeline exactly like the reference does — same windows, reference
    frame counts, step ranges, take_time, and the same latent state handed from call to call."""
    import json
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    with open(os.path.join(HERE, "golden", "reference_autoregressive_traces.json")) as f:
        want = json.load(f)[name]
    got = json.loads(json.dumps(run_autoregressive_case(CrossviewTemporalSD, name)))
    assert len(got["calls"]) == len(want["calls"])
    for a, b in zip(got["calls"], want["calls"]):
        assert a == b
    assert got["images_shape"] == want["images_shape"]
    assert got["images_sum"] == want["images_sum"]


def test_mirror_streaming_fifo_matches_reference():
    """FIFO streaming (condition queue, latent queue rotation with fresh noise, streaming-mode
    get_conditions with the previous ego pose, flush): per denoising call the step range,
    take_time, every condition tensor's shape + checksum and the latent state must equal the
    reference's, and so must the emitted frames."""
    import json
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    with open(os.path.join(HERE, "golden", "reference_autoregressive_traces.json")) as f:
        want = json.load(f)["streaming_fifo"]
    got = json.loads(json.dumps(run_fifo_case(
        StreamingCrossviewTemporalSD, object.__new__(DiTCrossviewTemporalConditionModel))))
    assert len(got["calls"]) == len(want["calls"]) == 7
    for a, b in zip(got["calls"], want["calls"]):
        assert a == b
    assert got["images_shape"] == want["images_shape"] and got["images_sum"] == want["images_sum"]


@pytest.fixture(scope="module")
def text_stack():
    return tiny_text_stack()


@pytest.mark.parametrize("name", list(TEXT_CASES))
def test_mirror_text_conditions_match_reference(name, text_stack):
    """Prompts (`clip_text`) through real (tiny, seeded) CLIP / T5 encoders: nested prompt
    flattening, CFG "" prompts, condition masks, CLIP-L|CLIP-G padding to the T5 width,
    broadcast over frames / views — fingerprints of the tensors the reference's get_conditions
    produced with the same encoder objects."""
    import json
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    with open(os.path.join(HERE, "golden", "reference_text_conditions.json")) as f:
        want = json.load(f)[name]
    got = run_text_case(CrossviewTemporalSD, (DiTCrossviewTemporalConditionModel,
                                              UNetCrossviewTemporalConditionModel),
                        name, text_stack)
    assert set(got) == set(want)
    for k in want:
        assert got[k]["shape"] == want[k]["shape"] and got[k]["dtype"] == want[k]["dtype"]
        for f in ("sum", "weighted", "abs"):
            assert got[k][f] == pytest.approx(want[k][f], rel=1e-6, abs=1e-6), (k, f)
        assert got[k]["samples"] == pytest.approx(want[k]["samples"], rel=1e-5, abs=1e-6)


@pytest.mark.parametrize("name", list(PREVIEW_CASES))
def test_mirror_preview_pipeline_dispatch_matches_reference(name):
    """`preview_pipeline` (what src/dwm/preview.py calls): latent shape derived from the batch
    image size / VAE config / temporal-VAE frame arithmetic, and which generation pipeline is
    run, equal to the reference's for both pipeline classes."""
    import json
    from dwm.pipelines.ctsd import CrossviewTemporalSD, StreamingCrossviewTemporalSD
    with open(os.path.join(HERE, "golden", "reference_autoregressive_traces.json")) as f:
        want = json.load(f)["preview_dispatch"][name]
    assert run_preview_case(CrossviewTemporalSD, StreamingCrossviewTemporalSD, name) == want


def test_df_index_schedule_matches_reference_loop_arithmetic():
    """The diffusion-forcing index expression of the reference loop (ctsd.py:2048-2055 and
    :2083-2088) evaluated literally, against the oracle and the mirrored helpers."""
    from oracle import ctsd as octsd
    from dwm.schedulers import temporal_independent as ti
    for steps, T in ((48, 16), (32, 16), (24, 6), (12, 4)):
        spi = steps // T
        for take in (0, 1):
            for i in range(take * spi, steps):
                want = [min(i - take * spi, max(0, i - j * spi)) for j in range(T)]
                rng = [i - j * spi >= 0 for j in range(T)]
                assert octsd.df_timestep_indices(i, T, spi, take) == want
                assert ti.df_timestep_indices(i, T, spi, take) == want
                assert octsd.df_in_schedule_range(i, T, spi) == rng
                assert ti.df_in_schedule_range(i, T, spi) == rng


@pytest.mark.gpu
@pytest.mark.parametrize("name", VARIANTS)
def test_cuda_dit_matches_reference(name, golden):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    cfg, sample, timestep, cond, extra = variant_case(name)
    o = seeded_oracle(cfg)
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    m.cuda()
    cond = {k: (v.cuda() if v is not None else None) for k, v in cond.items()}
    y = m(sample.cuda(), timestep.cuda(), **cond, **extra)
    y = y["noise_pred"] if extra else y[0][0]
    assert _rel(y.cpu(), golden["dit_" + name]) < 4e-3


@pytest.mark.gpu
def test_cuda_df_loop_matches_reference_loop(golden):
    """The mirrored pipeline's denoise_step for i = 9, 10, 11 (fp16 compute) against the
    latents the reference's own streaming loop produced."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    o = seeded_oracle(TINY)
    m = DiTCrossviewTemporalConditionModel(**TINY, compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    pipe = StreamingCrossviewTemporalSD(
        None, {"generator_seed": 0}, "cuda", {"frame_prediction_style": "diffusion_forcing"},
        {}, {"guidance_scale": 2.0, "inference_steps": 12, "sequence_length_per_iteration": 4},
        None, m, model_dtype=torch.float32)
    sample, _, cond = synthetic_inputs(TINY, device="cuda")
    pipe.reset_streaming((1, 4, 3, 16, 8, 12), "pt")
    lat = sample[:1].clone().float()
    for i in (9, 10, 11):
        idx, ts, in_range = pipe._df_step_tensors(i, 4, 3, 0, 1, 3)
        pipe.denoise_step(lat, cond, idx, ts, in_range)
    assert _rel(lat.cpu(), golden["pipe_df_latents_steps_9_10_11"]) < 4e-3


class _IdentityVae:
    """decode = identity, as in tests/golden/make_reference_golden.py: the loop's VAE call
    site and its post-processing run."""
    class config:
        scaling_factor, shift_factor = 1.0, None
    dtype = torch.float32

    @staticmethod
    def decode(x, return_dict=False):
        return (x,)


@pytest.mark.gpu
def test_cuda_streaming_loop_emits_reference_frame(golden):
    """The mirror's REAL StreamingCrossviewTemporalSD.inference_pipeline (steps 9..11, identity
    VAE) against what the reference's own loop produced: the returned latents and the frame it
    appended to `frames` — i.e. VAE call site + image_processor.postprocess (reference
    ctsd.py:2092-2101), values in [0, 1]."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    o = seeded_oracle(TINY)
    m = DiTCrossviewTemporalConditionModel(**TINY, compute_dtype=torch.float16)
    m.load_state_dict(o.state_dict())
    pipe = StreamingCrossviewTemporalSD(
        None, {"generator_seed": 0}, "cuda",
        {"frame_prediction_style": "diffusion_forcing", "vae_instance": _IdentityVae()},
        {}, {"guidance_scale": 2.0, "inference_steps": 12, "sequence_length_per_iteration": 4},
        None, m, model_dtype=torch.float32)
    sample, _, cond = synthetic_inputs(TINY, device="cuda")
    shape = (1, 4, 3, 16, 8, 12)
    pipe.reset_streaming(shape, "pt")
    pipe.conditions, pipe.latents = cond, sample[:1].clone().float()
    lat = pipe.inference_pipeline(shape, start_timestep=9, stop_timestep=12)
    assert _rel(lat.cpu(), golden["pipe_df_latents_steps_9_10_11"]) < 4e-3
    assert len(pipe.frames) == 1
    frame, want = pipe.frames[0].cpu(), golden["pipe_df_frame"]
    assert frame.shape == want.shape
    assert frame.min().item() >= 0.0 and frame.max().item() <= 1.0
    assert (frame - want).abs().max().item() < 4e-3        # post-processed range is [0, 1]
    # and the golden itself is NOT the raw latent frame (the test would be vacuous otherwise)
    raw = golden["pipe_df_latents_steps_9_10_11"][:, 0].flatten(0, 1)
    assert (raw - want).abs().max().item() > 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FULL_SEQUENCE_CASES))
def test_cuda_full_sequence_pipeline_matches_reference(name, golden):
    """CrossviewTemporalSD.inference_pipeline of the mirror (fp16 compute) against the
    reference's own inference_pipeline outputs: same generator noise, conditions, reference
    frame handling, step range."""
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    inf, nref = FULL_SEQUENCE_CASES[name]
    cfg, batch, common, shape, image_latents = full_sequence_inputs()
    if name == "df_queue_partial":
        common = dict(common, frame_prediction_style="diffusion_forcing")
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.float16)
    m.load_state_dict(seeded_oracle(cfg).state_dict())
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {}, dict(inf), None,
                               m, model_dtype=torch.float32)
    kw = dict(image_latents=image_latents.cuda(), reference_frame_count=nref) if nref else {}
    if name == "no_cfg_partial":
        kw.update(start_timestep=1, stop_timestep=3)
    if name == "df_queue_partial":
        kw = dict(image_latents=image_latents.cuda(), reference_frame_count=3, start_timestep=2,
                  stop_timestep=4, take_time=1)
    r = pipe.inference_pipeline(shape, batch, "pt", **kw)
    assert _rel(r["latents"].cpu(), golden["fullseq_%s_latents" % name]) < 8e-3
    assert r["images"].shape == golden["fullseq_%s_images" % name].shape


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,V,variant", _unet_cases())
def test_cuda_unet_matches_reference(B, T, V, variant, golden):
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from test_unet import _oracle, unet_case
    cfg, x, t, c = unet_case(B, T, V, variant)
    m = U(**cfg, compute_dtype=torch.float16)
    m.load_state_dict(_oracle(cfg).state_dict())
    m.cuda()
    c = {k: (v.cuda() if v is not None else None) for k, v in c.items()}
    y = m(x.cuda(), t.cuda(), **c)[0][0]
    assert _rel(y.cpu(), golden["unet_" + variant]) < 6e-3


@pytest.mark.gpu
def test_cuda_schedulers_match_reference(golden):
    from dwm.schedulers import temporal_independent as ti
    si = {k: v.cuda() for k, v in scheduler_inputs().items()}
    fm = ti.FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, shift=3.0)
    fm.set_timesteps(12, "cuda")
    assert torch.equal(fm.sigmas.cpu(), golden["fm_sigmas"])
    y = fm.step_by_indices(si["model_output"], si["fm_indices"], si["sample"],
                           return_dict=False)[0]
    torch.testing.assert_close(y.cpu(), golden["fm_step_by_indices"], rtol=1e-5, atol=1e-5)
    for pt in ("v_prediction", "epsilon", "sample"):
        ddim = ti.DDIMScheduler(prediction_type=pt, **SD21)
        ddim.set_timesteps(50, "cuda")
        y = ddim.step(si["model_output"], si["ddim_timesteps"], si["sample"],
                      return_dict=False)[0]
        torch.testing.assert_close(y.cpu(), golden["ddim_step_" + pt], rtol=2e-5, atol=2e-5)
    assert torch.equal(ddim.timesteps.cpu(), golden["ddim_timesteps_50"])
    ddpm = ti.DDPMScheduler(prediction_type="v_prediction", **SD21)
    torch.testing.assert_close(
        ddpm.add_noise(si["sample"], si["noise"], si["ddpm_timesteps"]).cpu(),
        golden["ddpm_add_noise"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(
        ddpm.get_velocity(si["sample"], si["noise"], si["ddpm_timesteps"]).cpu(),
        golden["ddpm_get_velocity"], rtol=1e-5, atol=1e-5)
