"""Host-side checks of the bench tooling (no GPU): the synthetic per-frame batch of
`streaming_e2e` goes through the real streaming-mode `get_conditions`, the example model blocks
the `workloads` use exist in the fixture, and the JSON line helpers keep their contract keys."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def test_streaming_frame_batch_feeds_get_conditions():
    import bench
    import bench_extras as bx
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from common import TINY
    cfg = bench.load_config()
    B, T, V, C, H, W = cfg["latent_shape"]
    blk = bx._blocks()["ctsd_35_df16_6views_video_generation_with_layout.json"]["pipeline"]
    common = {k: v for k, v in blk["common_config"].items()
              if k not in ("autocast", "text_encoder_load_args")}
    g = torch.Generator().manual_seed(0)
    m = cfg["model"]
    model = DiTCrossviewTemporalConditionModel(**TINY)          # isinstance checks only
    prev = None
    for t in range(2):
        fb = bx.frame_batch(g, V, (H * 8, W * 8), cfg["text_tokens"], m["joint_attention_dim"],
                            m["pooled_projection_dim"], t)
        c = CrossviewTemporalSD.get_conditions(
            model, "pre-encoded", None, common, (B, 1, V, C, H, W), fb, "cpu", torch.float32,
            streaming_mode=True, prev_ego_transforms=prev, do_classifier_free_guidance=True)
        prev = fb["ego_transforms"]
        assert c["encoder_hidden_states"].shape == (2 * B, 1, V, cfg["text_tokens"],
                                                     m["joint_attention_dim"])
        assert c["pooled_projections"].shape == (2 * B, 1, V, m["pooled_projection_dim"])
        assert c["condition_image_tensor"].shape == (2 * B, 1, V, 6, H * 8, W * 8)
        # fps + 10 camera ids + 2 action ids = projection_class_embeddings_input_dim / 256
        assert c["added_time_ids"].shape == (2 * B, 1, V,
                                             m["projection_class_embeddings_input_dim"] // 256)
        assert c["crossview_attention_mask"].shape == (2 * B, V, V)
        assert torch.isfinite(c["added_time_ids"][B:]).all()


def test_workload_blocks_exist_and_match_the_configs_named_in_baseline():
    import bench_extras as bx
    b = bx._blocks()
    c3 = b["ctsd_35_6views_video_generation.json"]["pipeline"]
    assert c3["model"]["temporal_attention_type"] == "rowwise"
    assert c3["inference_config"]["sequence_length_per_iteration"] == 19
    c5 = b["ctsd_35_tvae_6views_video_generation_with_layout.json"]["pipeline"]
    assert c5["common_config"]["vae"].endswith("AutoencoderKLCogVideoX")
    assert (c5["inference_config"]["sequence_length_per_iteration"] - 1) // 4 + 1 == 5
    with open(os.path.join(ROOT, "BASELINE.json")) as f:
        base = json.load(f)
    assert any("ctsd_35_6views_video_generation.json" in c for c in base["configs"])
    assert any("ctsd_35_tvae_6views_video_generation_with_layout.json" in c
               for c in base["configs"])

