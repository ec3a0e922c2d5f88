"""The FP8 GEMM path without a GPU: the CPU restatement of the E4M3 quantizer, loud errors of
the FP8 ops on CPU tensors, the model's gemm_dtype check, and the error of the fake-quant
oracle (the accuracy the FP8 path is held to) on the two test configs."""
import pytest
import torch

import fp8_emulation as fe
from common import TINY, seeded_oracle, synthetic_inputs


def _cast(v):
    return v.float().clamp(-448, 448).to(torch.float8_e4m3fn).double()


def test_rounding_matches_torch_cast_on_edge_cases():
    sub = 2.0 ** -9                                    # E4M3 subnormal step
    vals = [0.0, -0.0, 448.0, -448.0, 449.0, 463.9, 464.0, 470.0, 1e9, -1e9,
            sub, -sub, 0.5 * sub, 1.5 * sub, 2.5 * sub, 0.49 * sub, 7 * sub, 7.5 * sub,
            2.0 ** -6, 2.0 ** -6 * (1 + 1 / 16), 1 + 1 / 16, 1 + 3 / 16, 1 + 1 / 16 + 2 ** -20,
            -(1 + 3 / 16), 240.0, 248.0, 232.0, 15.5, 0.1, 3.3, 100.0, -0.001]
    v = torch.tensor(vals, dtype=torch.float32)     # the quantizer rounds fp32 products
    r = fe.e4m3_round(v)
    assert torch.equal(r, _cast(v)), torch.stack([v, r, _cast(v)], 1)
    # ties go to the even mantissa
    assert fe.e4m3_round(torch.tensor([1 + 1 / 16]))[0] == 1.0
    assert fe.e4m3_round(torch.tensor([1 + 3 / 16]))[0] == 1.25
    assert fe.e4m3_round(torch.tensor([0.5 * sub]))[0] == 0.0
    assert fe.e4m3_round(torch.tensor([1.5 * sub]))[0] == 2 * sub
    g = torch.Generator().manual_seed(0)
    x = torch.randn(20000, generator=g) * torch.exp2(
        torch.randint(-14, 9, (20000,), generator=g).float())
    assert torch.equal(fe.e4m3_round(x), _cast(x))


def test_quantize_rows_recipe():
    x = torch.zeros(4, 32)
    x[1, 5] = -3.0                     # single non-zero: scaled to -448 exactly
    x[2] = torch.linspace(-2, 1, 32)
    x[3, 0] = 1e-30
    q, s = fe.quantize_rows(x)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
    assert s[0] == 1.0 and not q[0].float().any()
    assert q[1, 5].float() == -448.0 and s[1] == torch.tensor(3.0) / 448
    assert q[2].float().abs().max() == 448.0
    assert s[3] == torch.tensor(1e-30) / 448 and q[3, 0].float() == 448.0
    d = fe.dequant(q, s)
    assert ((d - x).abs() <= 2 ** -4 * x.abs() + 2 ** -10 * s[:, None]).all()


def test_fp8_ops_raise_without_gpu():
    from opendwm_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = torch.zeros(128, 64, dtype=torch.float8_e4m3fn)
    s = torch.ones(128)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(a, a, a_scale=s, w_scale=s, out_dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.quantize_rows(torch.zeros(4, 64))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.quantize_weight_rows(torch.zeros(4, 64))
    with pytest.raises(TypeError, match="cuda fp32"):
        ops.layernorm(torch.zeros(4, 64), torch.zeros(4, 64, dtype=torch.float8_e4m3fn),
                      out_scale=torch.ones(4))


@pytest.mark.parametrize("bad", [torch.float16, torch.bfloat16, torch.float8_e5m2, "fp8", 8])
def test_model_rejects_bad_gemm_dtype(bad):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    with pytest.raises(ValueError, match="gemm_dtype"):
        DiTCrossviewTemporalConditionModel(**TINY, gemm_dtype=bad)
    m = DiTCrossviewTemporalConditionModel(**TINY, gemm_dtype=torch.float8_e4m3fn)
    assert m.gemm_dtype is torch.float8_e4m3fn


def test_gemm_dtype_reaches_the_model_from_a_json_config():
    from dwm.common import create_instance_from_config
    cfg = {"_class_name": "dwm.models.crossview_temporal_dit.DiTCrossviewTemporalConditionModel",
           **TINY, "gemm_dtype": {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}}
    m = create_instance_from_config(cfg)
    assert m.gemm_dtype is torch.float8_e4m3fn


def test_fp8_linear_set():
    names = set(fe.fp8_linears(seeded_oracle(TINY)))
    assert "transformer_blocks.0.attn.to_q" in names
    assert "transformer_blocks.0.ff.net.2" in names
    assert "transformer_blocks.0.attn2.to_out.0" in names
    assert "temporal_transformer_blocks.0.ff_in.net.0.proj" in names
    assert "crossview_transformer_blocks.0.attn1.to_out.0" in names
    assert not any(n.endswith((".norm1.linear", ".norm1_context.linear")) for n in names)
    assert not any(n.startswith(("proj_out", "context_embedder", "time_text_embed", "pos_embed",
                                 "condition_image_adapter", "norm_out")) for n in names)


# Error of per-row x per-channel E4M3 fake quantization against the fp32 oracle, measured on
# the random-init weights of the two configs (max|d| / max|ref|): ~2e-2 (TINY), ~6e-2 (real
# width).  The bounds only catch an emulator that stopped quantizing or broke.
@pytest.mark.parametrize("which", ["tiny", "real_width"])
def test_emulated_error_is_recorded(which):
    if which == "tiny":
        o = seeded_oracle(TINY)
        sample, timestep, cond = synthetic_inputs(TINY)
        lo, hi = 4e-3, 8e-2
    else:
        cfg = dict(TINY, **fe.REAL_WIDTH)
        o = seeded_oracle(cfg, std=fe.REAL_WIDTH_STD)
        sample, timestep, cond = synthetic_inputs(cfg, **fe.REAL_WIDTH_INPUTS)
        lo, hi = 1.5e-2, 0.1
    err, _, _ = fe.emulated_error(o, sample, timestep, cond)
    print("fake-quant E4M3 error", which, err)
    assert lo < err < hi, err
