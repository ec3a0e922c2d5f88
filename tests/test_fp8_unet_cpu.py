"""CPU side of the FP8 CTSD-2.1 UNet: the gemm_dtype argument and its config route, the loud
CPU errors of the FP8 convolution ops, and the layer selection of the fake-quant oracle."""
import pytest
import torch

import fp8_unet_emulation as fue

F8 = torch.float8_e4m3fn


def test_gemm_dtype_argument_and_config_route():
    from dwm.common import create_instance_from_config
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from test_unet import UCFG, _inputs
    with pytest.raises(ValueError, match="gemm_dtype"):
        U(**UCFG, gemm_dtype=torch.float16)
    assert U(**UCFG).gemm_dtype is None
    m = create_instance_from_config(
        {"_class_name": "dwm.models.crossview_temporal_unet.UNetCrossviewTemporalConditionModel",
         **UCFG, "gemm_dtype": {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}})
    assert m.gemm_dtype is F8
    x, t, c = _inputs(1, 1, 2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(x, t, **c)


def test_fp8_conv_ops_raise_on_cpu():
    from opendwm_b200 import lib, ops
    x = torch.zeros(1, 1, 4, 4, 32, dtype=F8)
    w = torch.zeros(9, 32, 32, dtype=F8)
    s = torch.ones(1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.conv(x, w, kernel=(1, 3, 3), epilogue=lib.EPI_RESID, a_scale=s, w_scale=torch.ones(32))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.pack_conv_weight_fp8(torch.zeros(32, 32, 3, 3))
    x32 = torch.zeros(1, 1, 4, 4, 32)
    with pytest.raises(TypeError, match="cuda fp32"):
        ops.groupnorm_silu_e4m3(x32, torch.zeros(1, 32, 2, dtype=torch.float64), torch.ones(32),
                                torch.zeros(32), x, s, groups=32)


def test_fake_quant_oracle_layer_selection():
    from test_unet import UCFG, _oracle
    lins, convs = fue.fp8_modules(_oracle(UCFG))
    assert not any(n.endswith(("attn2.to_k", "attn2.to_v", "proj_in", "proj_out"))
                   for n in lins)
    assert any(n.endswith("attn2.to_q") for n in lins)
    assert any(".crossview_transformer_blocks." in n for n in lins)
    assert any(".temporal_transformer_blocks." in n for n in lins)
    # spatial and temporal conv1 / conv2 of every ResBlock; no conv_in / conv_out / samplers /
    # shortcuts
    assert all(n.split(".")[-2] in ("spatial_res_block", "temporal_res_block") and
               n.split(".")[-1] in ("conv1", "conv2") for n in convs)
    assert any("temporal_res_block" in n for n in convs)
    # one scale per volume: a volume's quantization ignores the others
    x = torch.randn(3, 4, 2, 5, 5) * torch.tensor([1.0, 1e3, 1e-3]).view(3, 1, 1, 1, 1)
    y = fue.fake_quant_volumes(x)
    assert torch.equal(y[1], fue.fake_quant_volumes(x[1:2])[0])
    assert ((y - x).abs() <= 2.0 ** -4 * x.abs() + 1e-12).all()
