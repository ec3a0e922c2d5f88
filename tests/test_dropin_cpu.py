"""Drop-in surface: every `_class_name` / scheduler / VAE string the reference's CTSD example
configs use (examples/ctsd_*.json, class names listed here verbatim) resolves — through the
mirrored JSON factory — to a class of this repository with the constructor / method surface the
reference's entry script (examples/ctsd_generation_example.py:41-69) and pipeline rely on."""
import inspect

import pytest

PIPELINES = ["dwm.pipelines.ctsd.CrossviewTemporalSD",
             "dwm.pipelines.ctsd.StreamingCrossviewTemporalSD"]
MODELS = ["dwm.models.crossview_temporal_dit.DiTCrossviewTemporalConditionModel",
          "dwm.models.crossview_temporal_unet.UNetCrossviewTemporalConditionModel"]
SCHEDULERS = ["dwm.schedulers.temporal_independent.FlowMatchEulerDiscreteScheduler",
              "dwm.schedulers.temporal_independent.DDIMScheduler",
              "dwm.schedulers.temporal_independent.DDPMScheduler"]


def test_example_config_class_names_resolve_to_the_mirror():
    import dwm.common
    import dwm.pipelines.ctsd as ctsd
    for name in PIPELINES + MODELS + SCHEDULERS:
        cls = dwm.common.get_class(name)
        assert cls.__module__ == name.rsplit(".", 1)[0]
        assert "/src/dwm/" in inspect.getsourcefile(cls).replace("\\\\", "/")
    # {"_class_name": "get_class", "class_name": "torch.float16"} (model_dtype in the examples)
    import torch
    assert dwm.common.create_instance_from_config(
        {"_class_name": "get_class", "class_name": "torch.float16"}) is torch.float16
    # pipeline surface used by the entry script and by preview / streaming callers
    for method in ("inference_pipeline", "autoregressive_inference_pipeline", "get_conditions",
                   "load_state"):
        assert callable(getattr(ctsd.CrossviewTemporalSD, method))
    for method in ("reset_streaming", "send_frame_condition", "receive_frame",
                   "fifo_inference_pipeline"):
        assert callable(getattr(ctsd.StreamingCrossviewTemporalSD, method))
    ctor = inspect.signature(ctsd.CrossviewTemporalSD.__init__).parameters
    for kw in ("output_path", "config", "device", "common_config", "training_config",
               "inference_config", "pretrained_model_name_or_path", "model", "model_dtype",
               "model_checkpoint_path", "model_load_state_args"):
        assert kw in ctor, kw
    ar = inspect.signature(ctsd.CrossviewTemporalSD.autoregressive_inference_pipeline).parameters
    assert list(ar)[1:] == ["latent_shape", "batch", "output_type"]
    ip = inspect.signature(ctsd.CrossviewTemporalSD.inference_pipeline).parameters
    assert list(ip)[1:] == ["latent_shape", "batch", "output_type", "image_latents",
                            "reference_frame_count", "start_timestep", "stop_timestep",
                            "take_time"]


def test_pipeline_refuses_to_run_without_cuda():
    import torch
    import dwm.pipelines.ctsd as ctsd
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from common import TINY
    with pytest.raises(RuntimeError, match="no CPU"):
        ctsd.CrossviewTemporalSD(None, {}, "cpu", {}, {}, {"inference_steps": 2}, None,
                                 DiTCrossviewTemporalConditionModel(**TINY))


def test_scheduler_name_mapping_covers_the_example_strings():
    """`inference_config["scheduler"]` strings of the examples: the dwm.* one, the two diffusers
    names and the default; the mapping lives in the pipeline constructor."""
    import dwm.pipelines.ctsd as ctsd
    src = inspect.getsource(ctsd.CrossviewTemporalSD.__init__)
    for s in ("diffusers.DDIMScheduler", "diffusers.DPMSolverMultistepScheduler",
              "diffusers.FlowMatchEulerDiscreteScheduler"):
        assert s in src


# -- the example configs themselves (not a string list): tests/golden/example_pipeline_blocks.json
#    holds the `pipeline` block of every examples/ctsd_*.json of the reference ------------------
def _example_blocks():
    import json
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "golden", "example_pipeline_blocks.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(_example_blocks()))
def test_example_pipeline_block_instantiates_through_the_factory(name):
    """Every class named by the example resolves to the mirror and the `model` block builds
    through dwm.common.create_instance_from_config with the reference's own kwargs (on the
    meta device: shapes only).  The UniMLVG example (explicit perspective modelling) is outside
    the CTSD hot path (SURVEY.md §2) and must refuse loudly instead of building something else."""
    import torch
    import dwm.common
    blk = _example_blocks()[name]["pipeline"]
    pipe_cls = dwm.common.get_class(blk["_class_name"])
    assert pipe_cls.__module__ == "dwm.pipelines.ctsd"
    ctor = inspect.signature(pipe_cls.__init__).parameters
    for k in blk:
        if k not in ("_class_name",):
            assert k in ctor, (name, k)
    if "model_dtype" in blk:
        assert dwm.common.create_instance_from_config(blk["model_dtype"]) is torch.float16
    sched = blk["inference_config"].get("scheduler")
    if sched is not None and sched.startswith("dwm."):
        assert dwm.common.get_class(sched).__module__ == "dwm.schedulers.temporal_independent"
    model_cls = dwm.common.get_class(blk["model"]["_class_name"])
    assert model_cls.__module__.startswith("dwm.models.crossview_temporal_")
    if "unimlvg" in name:
        with pytest.raises(NotImplementedError):
            with torch.device("meta"):
                dwm.common.create_instance_from_config(blk["model"])
        return
    with torch.device("meta"):
        model = dwm.common.create_instance_from_config(blk["model"])
    assert isinstance(model, model_cls)
    n = sum(p.numel() for p in model.parameters())
    assert n > 1.5e9, n          # full-size SD-2.1 UNet (1.9 B) / SD-3.5-medium graft (3.8-4.1 B)
    # the configured grafts exist
    mc = blk["model"]
    if mc.get("enable_temporal") and "temporal_block_layers" in mc:
        assert len(model.temporal_transformer_blocks) == len(mc["temporal_block_layers"])
    if mc.get("enable_crossview") and "crossview_block_layers" in mc:
        assert len(model.crossview_transformer_blocks) == len(mc["crossview_block_layers"])
