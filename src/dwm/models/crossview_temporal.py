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

from .packing import fp32, gemm, layernorm, pack_linear, pack_norm, requantize


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


def _sharded_qkv_attend(D, eps, rows_full, remap, q_loc, attend, gather, peer_kv, kv_loc,
                        kv_all):
    """qkv_attend of a sharded block: K,V of the local rows are projected (+RMSNorm) straight
    into the gathered buffer [rows_full, 2D], which keeps the UNSHARDED row layout on every
    rank — through the GEMM epilogue's item row mapping `remap` into local AND peer memory
    (fused scatter over NVLink, `peer_kv` a PeerKV of the exchanging group; one group barrier
    per block), or into kv_loc followed by `gather(kv_loc, kv_all)` (an async all-gather) —
    while the Q projection runs into q_loc; then `attend(kv_full, out)`."""

    def project(p, a, w, nw, out, peer_out=None, **kw):
        if p["qk_norm"]:
            gemm(a, w, epilogue=_lib.EPI_QKNORM, out=out,
                 q_norm_weight=nw, qk_region=D, qk_norm_regions=1,
                 eps=eps, peer_out=peer_out, **kw)
        else:
            gemm(a, w, out=out, peer_out=peer_out, **kw)

    def qkv_attend(p, a, out):
        q, kv = p["qkv"].rows(0, D), p["qkv"].rows(D, 3 * D)
        if peer_kv is not None:
            # fused: the K,V GEMM epilogue scatters its tiles into every peer's
            # gathered buffer over NVLink; one group barrier publishes them
            kv_full, peers, hdl = peer_kv.next()
            # the leading rows at this block's width (peers address their buffers the same way)
            kv_full = kv_full.view(-1)[:rows_full * 2 * D].view(rows_full, 2 * D)
            project(p, a, kv, p.get("nk"), kv_full, peers, **remap)
            project(p, a, q, p.get("nq"), q_loc)
            hdl.barrier(channel=0)
        else:
            kv_full = kv_all
            project(p, a, kv, p.get("nk"), kv_loc)
            work = gather(kv_loc, kv_full)
            project(p, a, q, p.get("nq"), q_loc)
            work.wait()
        attend(kv_full, out)
    return qkv_attend


def sharded_temporal_qkv_attend(plan, kind, B, T_loc, V, Hp, Wp, D, heads, q_loc, peer_kv=None,
                                kv_loc=None, kv_all=None, eps=1e-5):
    """`VTSelfAttentionBlock.run`'s qkv_attend for frame-sharded temporal attention (kind
    "full", "rowwise" or "pointwise"; even or uneven frame shards of a ShardPlan): K,V of the
    local frames are projected (+RMSNorm) straight into the gathered buffer, which keeps the
    UNSHARDED row layout (b, t, v, s) on every rank — through the GEMM epilogue's item row
    mapping into local AND peer memory (fused scatter over NVLink, `peer_kv` a PeerKV whose
    buffers hold at least B*T*V*S x 2D), or through an all-gather (kv_loc, kv_all) — while
    the Q projection runs into q_loc; then every local query frame attends to all T frames
    with the single-GPU key addressing.  V is the number of views this rank holds (all
    views, or the V_loc of a view shard: the frame group exchanges the local views)."""
    S, T = Hp * Wp, plan.T
    # local rows -> rows of the unsharded layout: item = batch entry
    remap = dict(rows_per_item=T_loc * V * S, out_item_stride=T * V * S,
                 out_row_offset=plan.t_offset * V * S)

    def attend(kv_all, out):
        if kind == "full":         # (b v) (t hw)
            _ops.attention(
                q_loc, out, D=D, heads=heads, group_dims=[B, V],
                group_strides=[T_loc * V * S, S], seq=T_loc * S, inner=S,
                stride_outer=V * S, stride_inner=1, kv=kv_all, k_col=0, v_col=D,
                kv_group_strides=[T * V * S, S], seq_kv=T * S, inner_kv=S,
                kv_stride_outer=V * S, kv_stride_inner=1)
        elif kind == "rowwise":    # (b v h) (t w)
            _ops.attention(
                q_loc, out, D=D, heads=heads, group_dims=[B, V, Hp],
                group_strides=[T_loc * V * S, S, Wp], seq=T_loc * Wp, inner=Wp,
                stride_outer=V * S, stride_inner=1, kv=kv_all, k_col=0, v_col=D,
                kv_group_strides=[T * V * S, S, Wp], seq_kv=T * Wp, inner_kv=Wp,
                kv_stride_outer=V * S, kv_stride_inner=1)
        else:                      # pointwise: (b v hw) t
            _ops.attention(
                q_loc, out, D=D, heads=heads, group_dims=[B, V * S],
                group_strides=[T_loc * V * S, 1], seq=T_loc, inner=1,
                stride_outer=V * S, stride_inner=0, kv=kv_all, k_col=0, v_col=D,
                kv_group_strides=[T * V * S, 1], seq_kv=T, inner_kv=1,
                kv_stride_outer=V * S, kv_stride_inner=0)

    def gather(kv_loc, kv_full):
        return plan.gather_frames_kv(kv_loc, kv_full, batch=B, async_op=True)
    return _sharded_qkv_attend(D, eps, B * T * V * S, remap, q_loc, attend, gather, peer_kv,
                               kv_loc, kv_all)


def sharded_crossview_qkv_attend(plan, items, Hp, Wp, D, heads, q_loc, mask, mask_div,
                                 peer_kv=None, kv_loc=None, kv_all=None, eps=1e-5):
    """`VTSelfAttentionBlock.run`'s qkv_attend for row-wise cross-view attention
    "(bt v) (h w) -> (bt h) (v w)" on a view shard (plan.V_loc views from plan.v_offset of
    plan.V): K,V of the local views go to the gathered buffer of the local frames
    [items * V * S, 2D] (items = batch entries x local frames) in the unsharded view order,
    through the epilogue remap (item = one (b, t), V_loc * S rows each) with a peer scatter
    over the view group, or an all-gather over it (kv_loc, kv_all).  The local query views
    then attend to all V views; query unit u reads row v_offset + u of the [B, V, V] view mask.
    Without a mask an all-ones one is used: it selects the kernel the unsharded launch runs
    on, and allows every view as no mask does."""
    S, V, V_loc, v_off = Hp * Wp, plan.V, plan.V_loc, plan.v_offset
    remap = dict(rows_per_item=V_loc * S, out_item_stride=V * S, out_row_offset=v_off * S)
    if mask is None:
        mask = torch.ones(1, V, V, dtype=torch.uint8, device=q_loc.device)
        mask_div = items

    def attend(kv_all, out):
        _ops.attention(
            q_loc, out, D=D, heads=heads, group_dims=[items, Hp],
            group_strides=[V_loc * S, Wp], seq=V_loc * Wp, inner=Wp, stride_outer=S,
            stride_inner=1, mask=mask, mask_div=mask_div, mask_q_offset=v_off,
            kv=kv_all, k_col=0, v_col=D, kv_group_strides=[V * S, Wp], seq_kv=V * Wp,
            inner_kv=Wp, kv_stride_outer=S, kv_stride_inner=1)

    def gather(kv_loc, kv_full):
        return plan.gather_views_kv(kv_loc, kv_full, items=items, async_op=True)
    return _sharded_qkv_attend(D, eps, items * V * S, remap, q_loc, attend, gather, peer_kv,
                               kv_loc, kv_all)


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

    def pack(self, dtype, device, fp8=False):
        """Packs the weights for `run`: a dict of `Linear`s (ff_in1, ff_in2, qkv, out, ff1,
        ff2) and LayerNorm triples.  fp8: every linear is E4M3 with one fp32 scale per output
        channel, quantized from the parameters' own precision; 16-bit outputs stay `dtype`."""
        p = {}
        for name, ff in (("ff_in", self.ff_in), ("ff", self.ff)):
            w, b = _ops.pack_geglu(
                ff.net[0].proj.weight.detach().to(device),
                ff.net[0].proj.bias.detach().to(device))
            # FP8: quantized after the GEGLU row packing, scales follow the rows
            p[name + "1"] = pack_linear(w, b, dtype, device, fp8)
            p[name + "2"] = pack_linear(ff.net[2].weight, ff.net[2].bias, dtype, device, fp8)
        at = self.attn1
        p["qkv"] = pack_linear(
            torch.cat([at.to_q.weight, at.to_k.weight, at.to_v.weight]),
            None if at.to_q.bias is None else
            torch.cat([at.to_q.bias, at.to_k.bias, at.to_v.bias]), dtype, device, fp8)
        p["qk_norm"] = at.qk_norm == "rms_norm"
        if p["qk_norm"]:
            p["nq"], p["nk"] = fp32(at.norm_q.weight), fp32(at.norm_k.weight)
        p["out"] = pack_linear(at.to_out[0].weight, at.to_out[0].bias, dtype, device, fp8)
        for n in ("norm_in", "norm1", "norm3"):
            p[n] = pack_norm(getattr(self, n))
        self._packed = p
        return p

    def run(self, p, x, emb, rows_per_item, ws, attend, alpha, rows_per_batch,
            qkv_attend=None):
        """x: fp32 residual stream [M, D] (updated in place with the blended result);
        emb: fp32 [items, D] added before the block (view / frame index embedding);
        attend(qkv, out): launches the regrouped attention; alpha: fp32 [B];
        qkv_attend(p, a, out): optional replacement of projection + attention
        (frame-sharded temporal attention with a K,V all-gather; it receives the LayerNorm
        output Operand).  ws["a"] is the LayerNorm output Operand and ws["q"] the E4M3 buffer
        the GEGLU and attention outputs are requantized into (None in 16 bit)."""
        D = self.dim
        y, g16, qkv, o16, a, q = ws["y"], ws["g16"], ws["qkv_s"], ws["o16"], ws["a"], ws["q"]
        n_in, n1, n3 = p["norm_in"], p["norm1"], p["norm3"]
        layernorm(x, a, weight=n_in[0], bias=n_in[1], eps=n_in[2],
                  add_item=emb, rows_per_item=rows_per_item, sum_out=y)
        gemm(a, p["ff_in1"], epilogue=_lib.EPI_GEGLU, out=g16)
        gemm(requantize(g16, q), p["ff_in2"], epilogue=_lib.EPI_RESID, resid=y, out=y)
        layernorm(y, a, weight=n1[0], bias=n1[1], eps=n1[2])
        if qkv_attend is not None:
            qkv_attend(p, a, o16)
        else:
            if p["qk_norm"]:
                gemm(a, p["qkv"], epilogue=_lib.EPI_QKNORM, out=qkv,
                     q_norm_weight=p["nq"], k_norm_weight=p["nk"], qk_region=D,
                     eps=self.attn1.eps)
            else:
                gemm(a, p["qkv"], out=qkv)
            attend(qkv, o16)
        gemm(requantize(o16, q), p["out"], epilogue=_lib.EPI_RESID, resid=y, out=y)
        layernorm(y, a, weight=n3[0], bias=n3[1], eps=n3[2])
        gemm(a, p["ff1"], epilogue=_lib.EPI_GEGLU, out=g16)
        # last GEMM: + residual, then AlphaBlender against the un-grafted stream
        gemm(requantize(g16, q), p["ff2"], epilogue=_lib.EPI_RESID, resid=y, out=x,
             blend_x=x, alpha=alpha, rows_per_batch=rows_per_batch)
