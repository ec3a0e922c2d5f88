"""Parity of the H100-native DiT forward against the fp32 oracle (same state_dict,
same seeded inputs).  Metric: max|y - ref| / max|ref| (SURVEY.md §7 tolerance policy).
Stated tolerances: bf16 operands 2e-2, fp16 operands 4e-3 for this 4-layer model
(16-bit GEMM operands, fp32 accumulation / statistics / residual stream)."""
import pytest
import torch

from common import TINY, seeded_oracle, synthetic_inputs

pytestmark = pytest.mark.gpu
TOL = {torch.bfloat16: 2e-2, torch.float16: 4e-3}


def _pair(cfg, dtype):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    o = seeded_oracle(cfg).cuda()
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=dtype)
    m.load_state_dict(o.state_dict())
    return o, m.cuda()


def _rel(y, ref):
    return ((y.float() - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_tiny_forward(dtype):
    o, m = _pair(TINY, dtype)
    sample, timestep, cond = synthetic_inputs(TINY, device="cuda")
    with torch.no_grad():
        ref = o(sample, timestep, **cond)[0][0]
    out, a, b = m(sample, timestep, **cond)
    y = out[0]
    assert y.shape == ref.shape and (a, b) == (4, 4)
    assert _rel(y, ref) < TOL[dtype], _rel(y, ref)
    # second call hits the condition cache and must be bit-identical
    y2 = m(sample, timestep, **cond)[0][0]
    assert torch.equal(y, y2)
    # different timesteps change the result
    y3 = m(sample, timestep * 0.5, **cond)[0][0]
    assert not torch.equal(y, y3)


@pytest.mark.parametrize("variant", ["temporal_rowwise", "temporal_full", "crossview_full",
                                     "no_adapter", "no_qknorm_extra", "disabled_batch1",
                                     "no_perspective"])
def test_variants(variant):
    cfg = dict(TINY)
    kw = {}
    if variant == "temporal_rowwise":
        cfg["temporal_attention_type"] = "rowwise"
    elif variant == "temporal_full":
        cfg["temporal_attention_type"] = "full"
    elif variant == "crossview_full":
        cfg["crossview_attention_type"] = "full"
        kw["crossview_attention_mask"] = None
    elif variant == "no_adapter":
        cfg["condition_image_adapter_config"] = None
    elif variant == "no_qknorm_extra":
        cfg["qk_norm_on_additional_modules"] = None
    elif variant == "no_perspective":
        cfg["perspective_modeling_type"] = ""
    o, m = _pair(cfg, torch.float16)
    sample, timestep, cond = synthetic_inputs(cfg, device="cuda")
    cond.update(kw)
    if variant == "disabled_batch1":
        cond["disable_temporal"] = torch.tensor([False, True], device="cuda")
        cond["disable_crossview"] = torch.tensor([True, False], device="cuda")
    with torch.no_grad():
        ref = o(sample, timestep, **cond)[0][0]
    y = m(sample, timestep, **cond)[0][0]
    assert _rel(y, ref) < TOL[torch.float16], _rel(y, ref)


def test_five_dim_input_and_return_dict():
    cfg = dict(TINY, enable_crossview=False, crossview_block_layers=None,
               perspective_modeling_type="", condition_image_adapter_config=None)
    o, m = _pair(cfg, torch.float16)
    sample, timestep, cond = synthetic_inputs(cfg, V=1, device="cuda")
    s5, t5 = sample.squeeze(2), timestep.squeeze(2)
    c5 = dict(encoder_hidden_states=cond["encoder_hidden_states"].squeeze(2),
              pooled_projections=cond["pooled_projections"].squeeze(2),
              disable_temporal=cond["disable_temporal"].unsqueeze(1))
    with torch.no_grad():
        ref = o(s5, t5, return_dict=True, **c5)["noise_pred"]
    y = m(s5, t5, return_dict=True, **c5)["noise_pred"]
    assert y.shape == ref.shape == s5.shape
    assert _rel(y, ref) < TOL[torch.float16]


def test_real_width_two_layers():
    """D = 1536 (24 heads) exercises the production tile shapes."""
    cfg = dict(TINY, num_attention_heads=24, caption_projection_dim=1536, num_layers=2,
               dual_attention_layers=[0], crossview_block_layers=[0],
               temporal_block_layers=[1], joint_attention_dim=256,
               condition_image_adapter_config=dict(
                   in_channels=6, channels=[1536], is_downblocks=[True],
                   num_res_blocks=1, downscale_factor=8, use_zero_convs=True))
    from common import seeded_oracle as so
    o = so(cfg, std=0.02).cuda()
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=torch.bfloat16)
    m.load_state_dict(o.state_dict())
    m.cuda()
    sample, timestep, cond = synthetic_inputs(cfg, T=2, V=6, H=8, W=16, L=20, device="cuda")
    with torch.no_grad():
        ref = o(sample, timestep, **cond)[0][0]
    y = m(sample, timestep, **cond)[0][0]
    assert _rel(y, ref) < 2e-2, _rel(y, ref)


def test_streaming_ring_cache_equals_full_recompute():
    """FIFO moved on by one frame: the incrementally updated condition cache (`_ring_shift`)
    must give the same forward as rebuilding it from the new condition tensors."""
    o, m = _pair(TINY, torch.float16)
    sample, timestep, cond = synthetic_inputs(TINY, device="cuda")
    _, _, nxt = synthetic_inputs(TINY, device="cuda", seed=9)
    m(sample, timestep, **cond)                                   # fills the cache
    moved = {}
    for k, v in cond.items():
        if v is not None and v.dim() > 1 and v.shape[1] == 4 and k != "crossview_attention_mask":
            moved[k] = torch.cat([v[:, 1:], nxt[k][:, :1]], 1).contiguous()
        else:
            moved[k] = v
    m._ring_shift = True
    y_ring = m(sample, timestep, **moved)[0][0]
    assert "_ring_shift" not in m.__dict__
    m._cond_key = None                                            # force the full rebuild
    y_full = m(sample, timestep, **moved)[0][0]
    assert torch.equal(y_ring, y_full)
    with torch.no_grad():
        ref = o(sample, timestep, **moved)[0][0]
    assert _rel(y_ring, ref) < TOL[torch.float16]
