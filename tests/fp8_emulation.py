"""CPU restatement of the E4M3 row quantizer of the FP8 GEMM path, and the fake-quant oracle.

The quantizer (dwm_b200_quantize_rows, the E4M3 LayerNorm output, FP8 weight packing):
amax == 0 -> scale 1, q = 0; otherwise inv = 448 / amax, q = rn_satfinite_e4m3(x * inv),
scale = amax / 448, all in IEEE fp32.

The fake-quant oracle is the fp32 oracle with every linear of the FP8 set (the joint blocks'
attention and feed-forward linears, every linear of the cross-view / temporal blocks; not the
AdaLN modulation linears) computing dequant(q(x)) . dequant(q(W))^T + b with per-row activation
and per-output-channel weight scales.  The model packs its FP8 weights with the same quantizer
from the same fp32 parameters, so these are the model's own weights and scales."""
import contextlib

import torch

FMAX = 448.0


def e4m3_round(v):
    """Round-to-nearest-even onto the E4M3 grid (3 mantissa bits, normals from 2^-6,
    subnormal step 2^-9), saturating at +-448; float64 in, float64 out."""
    v = v.double()
    _, e = torch.frexp(v)                       # |v| = m 2^e, m in [0.5, 1)
    quantum = torch.pow(2.0, (e - 1).clamp_min(-6).double() - 3)
    return (torch.round(v / quantum) * quantum).clamp(-FMAX, FMAX)   # torch.round: ties to even


def quantize_rows(x):
    """x [M, K] (any float dtype; converted to fp32 exactly) -> (q float8_e4m3fn [M, K],
    scale fp32 [M])."""
    x = x.float()
    amax = x.abs().amax(dim=-1, keepdim=True)
    nz = amax > 0
    inv = torch.where(nz, torch.tensor(FMAX) / amax, torch.zeros_like(amax))
    scale = torch.where(nz, amax / torch.tensor(FMAX), torch.ones_like(amax))
    q = e4m3_round(x * inv).to(torch.float8_e4m3fn)
    return q, scale.squeeze(-1)


def dequant(q, scale):
    return q.float() * scale.unsqueeze(-1)


def fake_quant_rows(x):
    """dequant(quantize_rows(x)) over the last dim of x, any leading shape."""
    x2 = x.reshape(-1, x.shape[-1])
    return dequant(*quantize_rows(x2)).reshape(x.shape)


_ADALN = (".norm1.linear", ".norm1_context.linear")


def fp8_linears(oracle):
    """The oracle's nn.Linear modules that the model runs in FP8, by name."""
    out = {}
    for name, m in oracle.named_modules():
        if not isinstance(m, torch.nn.Linear):
            continue
        joint = name.startswith("transformer_blocks.") and not name.endswith(_ADALN)
        vt = name.startswith(("crossview_transformer_blocks.", "temporal_transformer_blocks."))
        if joint or vt:
            out[name] = m
    return out


@contextlib.contextmanager
def fake_quant(oracle):
    """Within the block, the oracle's FP8 linears compute with fake-quantized operands."""
    mods = set(fp8_linears(oracle).values())
    assert mods, "no FP8 linears found"
    weights = {m: fake_quant_rows(m.weight.detach().float()) for m in mods}
    orig = torch.nn.Linear.forward

    def forward(self, x):
        if self in mods:
            return torch.nn.functional.linear(fake_quant_rows(x), weights[self].to(x.dtype),
                                              self.bias)
        return orig(self, x)

    torch.nn.Linear.forward = forward
    try:
        yield
    finally:
        torch.nn.Linear.forward = orig


def rel_err(y, ref):
    return ((y.float() - ref.float()).abs().max() / ref.float().abs().max()).item()


def emulated_error(oracle, sample, timestep, cond):
    """(max|fake-quant - oracle| / max|oracle|, fp32 oracle output, fake-quant output)."""
    with torch.no_grad():
        ref = oracle(sample, timestep, **cond)[0][0]
        with fake_quant(oracle):
            y = oracle(sample, timestep, **cond)[0][0]
    return rel_err(y, ref), ref, y


# the real-width 2-layer config of tests/test_model_gpu.py::test_real_width_two_layers
REAL_WIDTH = dict(
    num_attention_heads=24, caption_projection_dim=1536, num_layers=2,
    dual_attention_layers=[0], crossview_block_layers=[0], temporal_block_layers=[1],
    joint_attention_dim=256,
    condition_image_adapter_config=dict(
        in_channels=6, channels=[1536], is_downblocks=[True], num_res_blocks=1,
        downscale_factor=8, use_zero_convs=True))
REAL_WIDTH_INPUTS = dict(T=2, V=6, H=8, W=16, L=20)
REAL_WIDTH_STD = 0.02
