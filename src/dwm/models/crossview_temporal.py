"""Building blocks grafted into the base diffusion model — H100-native mirror of
reference src/dwm/models/crossview_temporal.py (AlphaBlender :9-72,
VTSelfAttentionBlock :536-582).

The modules here only OWN parameters (with the reference's state_dict key names, so
published checkpoints load unchanged) and describe how they execute on the
`opendwm_b200` kernels; no arithmetic runs in PyTorch.
"""
import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops


class ParamGroup(torch.nn.Module):
    """Pure namespace: gives nested parameters the reference's dotted key names."""


def make_feed_forward(dim, dim_out=None, mult=4, activation_fn="geglu"):
    """Parameter layout of diffusers FeedForward: net.0.proj, net.2."""
    inner = int(dim * mult)
    dim_out = dim if dim_out is None else dim_out
    ff = ParamGroup()
    act = ParamGroup()
    act.proj = torch.nn.Linear(
        dim, inner * 2 if activation_fn == "geglu" else inner)
    ff.net = torch.nn.ModuleList(
        [act, torch.nn.Identity(), torch.nn.Linear(inner, dim_out)])
    ff.activation_fn = activation_fn
    return ff


class RMSNormWeight(torch.nn.Module):
    def __init__(self, dim, eps):
        super().__init__()
        self.eps = eps
        self.weight = torch.nn.Parameter(torch.ones(dim))


def make_attention(query_dim, heads, dim_head, bias=False, qk_norm=None,
                   eps=1e-5, added_kv_proj_dim=None, context_pre_only=None):
    """Parameter layout of diffusers Attention (to_q/k/v, to_out.0, norm_q/k,
    add_{q,k,v}_proj, to_add_out, norm_added_{q,k})."""
    inner = heads * dim_head
    at = ParamGroup()
    at.heads, at.dim_head, at.eps, at.qk_norm = heads, dim_head, eps, qk_norm
    at.to_q = torch.nn.Linear(query_dim, inner, bias=bias)
    at.to_k = torch.nn.Linear(query_dim, inner, bias=bias)
    at.to_v = torch.nn.Linear(query_dim, inner, bias=bias)
    if qk_norm == "rms_norm":
        at.norm_q = RMSNormWeight(dim_head, eps)
        at.norm_k = RMSNormWeight(dim_head, eps)
    elif qk_norm is not None:
        raise ValueError("unsupported qk_norm {}".format(qk_norm))
    if added_kv_proj_dim is not None:
        at.add_k_proj = torch.nn.Linear(added_kv_proj_dim, inner)
        at.add_v_proj = torch.nn.Linear(added_kv_proj_dim, inner)
        at.add_q_proj = torch.nn.Linear(added_kv_proj_dim, inner)
        if qk_norm == "rms_norm":
            at.norm_added_q = RMSNormWeight(dim_head, eps)
            at.norm_added_k = RMSNormWeight(dim_head, eps)
    at.to_out = torch.nn.ModuleList(
        [torch.nn.Linear(inner, query_dim), torch.nn.Identity()])
    if context_pre_only is not None and not context_pre_only:
        at.to_add_out = torch.nn.Linear(inner, query_dim)
    return at


class AlphaBlender(torch.nn.Module):
    """alpha * a + (1 - alpha) * b with alpha = 1 where image_only_indicator
    (reference crossview_temporal.py:9-72).  The blend itself is fused into the
    epilogue of the block's last GEMM; this module owns `mix_factor` and yields the
    per-batch alpha vector."""

    strategies = ["fixed", "learned", "learned_with_images"]

    def __init__(self, alpha: float,
                 merge_strategy: str = "learned_with_images"):
        super().__init__()
        self.merge_strategy = merge_strategy
        if merge_strategy not in AlphaBlender.strategies:
            raise ValueError(
                "merge_strategy needs to be in {}"
                .format(AlphaBlender.strategies))
        if merge_strategy == "fixed":
            self.register_buffer("mix_factor", torch.Tensor([alpha]))
        else:
            self.register_parameter(
                "mix_factor", torch.nn.Parameter(torch.Tensor([alpha])))

    def get_alpha(self, image_only_indicator=None):
        mix = self.mix_factor.detach().float()
        if self.merge_strategy == "fixed":
            return mix
        if self.merge_strategy == "learned":
            return torch.sigmoid(mix)
        if image_only_indicator is None:
            raise ValueError(
                "Please provide image_only_indicator to use "
                "learned_with_images merge strategy")
        return torch.where(
            image_only_indicator,
            torch.ones((1,), device=image_only_indicator.device),
            torch.sigmoid(mix).to(image_only_indicator.device))

    def batch_alpha(self, batch_size, image_only_indicator, device):
        """fp32 [batch_size] alpha vector for the fused blend epilogue."""
        a = self.get_alpha(image_only_indicator).to(device)
        return a.flatten().expand(batch_size).contiguous() \
            if a.numel() == 1 else a.flatten().contiguous()


class VTSelfAttentionBlock(torch.nn.Module):
    """LN -> GEGLU-FF + res ; LN -> MHSA(+qk RMSNorm) + res ; LN -> GEGLU-FF + res
    (reference crossview_temporal.py:536-582), executed as 3 LayerNorm launches,
    5 wgmma GEMMs with fused epilogues and one gathered-attention launch."""

    def __init__(self, dim: int, time_mix_inner_dim: int,
                 num_attention_heads: int, attention_head_dim: int,
                 qk_norm=None):
        super().__init__()
        if dim != time_mix_inner_dim:
            raise NotImplementedError(
                "time_mix_inner_dim != dim is not used by any CTSD config")
        self.dim = dim
        self.heads = num_attention_heads
        self.norm_in = torch.nn.LayerNorm(dim)
        self.ff_in = make_feed_forward(dim, dim_out=time_mix_inner_dim)
        self.norm1 = torch.nn.LayerNorm(time_mix_inner_dim)
        self.attn1 = make_attention(
            time_mix_inner_dim, num_attention_heads, attention_head_dim,
            bias=False, qk_norm=qk_norm, eps=1e-5)
        self.norm3 = torch.nn.LayerNorm(time_mix_inner_dim)
        self.ff = make_feed_forward(time_mix_inner_dim)
        self._packed = None

    def pack(self, dtype, device):
        def w16(t):
            return t.detach().to(device=device, dtype=dtype).contiguous()

        def f32(t):
            return None if t is None else \
                t.detach().to(device=device, dtype=torch.float32).contiguous()

        p = {}
        for name, ff in (("ff_in", self.ff_in), ("ff", self.ff)):
            w, b = _ops.pack_geglu(
                ff.net[0].proj.weight.detach().to(device),
                ff.net[0].proj.bias.detach().to(device))
            p[name + "1_w"], p[name + "1_b"] = w16(w), f32(b)
            p[name + "2_w"], p[name + "2_b"] = \
                w16(ff.net[2].weight), f32(ff.net[2].bias)
        at = self.attn1
        p["qkv_w"] = w16(torch.cat(
            [at.to_q.weight, at.to_k.weight, at.to_v.weight]))
        p["qkv_b"] = None if at.to_q.bias is None else f32(torch.cat(
            [at.to_q.bias, at.to_k.bias, at.to_v.bias]))
        D = self.dim
        p["q_w"], p["kv_w"] = p["qkv_w"][:D], p["qkv_w"][D:]   # row slices (views)
        p["q_b"] = None if p["qkv_b"] is None else p["qkv_b"][:D]
        p["kv_b"] = None if p["qkv_b"] is None else p["qkv_b"][D:]
        p["qk_norm"] = at.qk_norm == "rms_norm"
        if p["qk_norm"]:
            p["nq"], p["nk"] = f32(at.norm_q.weight), f32(at.norm_k.weight)
        p["out_w"], p["out_b"] = w16(at.to_out[0].weight), f32(at.to_out[0].bias)
        for n in ("norm_in", "norm1", "norm3"):
            m = getattr(self, n)
            p[n + "_w"], p[n + "_b"], p[n + "_eps"] = \
                f32(m.weight), f32(m.bias), m.eps
        self._packed = p
        return p

    def run(self, p, x, emb, rows_per_item, ws, attend, alpha, rows_per_batch,
            qkv_attend=None):
        """x: fp32 residual stream [M, D] (updated in place with the blended result);
        emb: fp32 [items, D] added before the block (view / frame index embedding);
        attend(qkv, out): launches the regrouped attention; alpha: fp32 [B];
        qkv_attend(p, a16, out): optional replacement of projection + attention
        (frame-sharded temporal attention with a K,V all-gather)."""
        D = self.dim
        y, a16, g16, qkv, o16 = ws["y"], ws["a16"], ws["g16"], ws["qkv_s"], ws["o16"]
        _ops.layernorm(x, a16, weight=p["norm_in_w"], bias=p["norm_in_b"],
                       eps=p["norm_in_eps"], add_item=emb,
                       rows_per_item=rows_per_item, sum_out=y)
        _ops.linear(a16, p["ff_in1_w"], p["ff_in1_b"], epilogue=_lib.EPI_GEGLU,
                    out=g16)
        _ops.linear(g16, p["ff_in2_w"], p["ff_in2_b"], epilogue=_lib.EPI_RESID,
                    resid=y, out=y)
        _ops.layernorm(y, a16, weight=p["norm1_w"], bias=p["norm1_b"],
                       eps=p["norm1_eps"])
        if qkv_attend is not None:
            qkv_attend(p, a16, o16)
        else:
            if p["qk_norm"]:
                _ops.linear(a16, p["qkv_w"], p["qkv_b"], epilogue=_lib.EPI_QKNORM,
                            out=qkv, q_norm_weight=p["nq"], k_norm_weight=p["nk"],
                            qk_region=D, eps=self.attn1.eps)
            else:
                _ops.linear(a16, p["qkv_w"], p["qkv_b"], out=qkv)
            attend(qkv, o16)
        _ops.linear(o16, p["out_w"], p["out_b"], epilogue=_lib.EPI_RESID,
                    resid=y, out=y)
        _ops.layernorm(y, a16, weight=p["norm3_w"], bias=p["norm3_b"],
                       eps=p["norm3_eps"])
        _ops.linear(a16, p["ff1_w"], p["ff1_b"], epilogue=_lib.EPI_GEGLU, out=g16)
        # last GEMM: + residual, then AlphaBlender against the un-grafted stream
        _ops.linear(g16, p["ff2_w"], p["ff2_b"], epilogue=_lib.EPI_RESID,
                    resid=y, out=x, blend_x=x, alpha=alpha,
                    rows_per_batch=rows_per_batch)
