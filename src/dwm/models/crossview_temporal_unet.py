"""CTSD-2.1 UNet with cross-view / temporal grafts — H100-native mirror of reference
src/dwm/models/crossview_temporal_unet.py:355-835 (`UNetCrossviewTemporalConditionModel`,
a subclass of diffusers `UNetSpatioTemporalConditionModel`) and of the blocks it is made
of (`ResBlock`, `TransformerModel`, `TemporalBasicTransformerBlock`,
src/dwm/models/crossview_temporal.py:75-514).

Same constructor kwargs, forward signature / return value and state_dict key names
(incl. the SD-2.1 -> SVD key renamer `try_to_convert_state_dict`).  Activations are
channels-last token matrices `[(b t v) (h w), C]` (fp32 stream, 16-bit GEMM / conv
operands); every 3x3 convolution is the im2col-free wgmma conv, every Linear the
wgmma GEMM, GroupNorm(+SiLU) one fused pass, attention the gathered / wgmma
attention kernels.  The spatial / cross-view / temporal regroupings are index arithmetic
inside the attention kernel, exactly as in the DiT mirror.
"""
import re

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops

from .. import _compat
from . import adapters as _adapters
from .crossview_temporal import (
    AlphaBlender, ParamGroup, VTSelfAttentionBlock, make_attention, make_feed_forward,
    sharded_crossview_qkv_attend, sharded_temporal_qkv_attend)
from .packing import (
    FP8, Operand, conv, gemm, layernorm, pack_conv, pack_linear, pack_norm, requantize)


def _mlp(i, h, o):
    m = ParamGroup()
    m.linear_1 = torch.nn.Linear(i, h)
    m.linear_2 = torch.nn.Linear(h, o)
    return m


def _resnet2d(cin, cout, temb, eps):
    m = ParamGroup()
    m.norm1 = torch.nn.GroupNorm(32, cin, eps=eps)
    m.conv1 = torch.nn.Conv2d(cin, cout, 3, padding=1)
    m.time_emb_proj = torch.nn.Linear(temb, cout)
    m.norm2 = torch.nn.GroupNorm(32, cout, eps=eps)
    m.conv2 = torch.nn.Conv2d(cout, cout, 3, padding=1)
    if cin != cout:
        m.conv_shortcut = torch.nn.Conv2d(cin, cout, 1)
    return m


def _resnet_t(c, temb, eps):
    m = ParamGroup()
    m.norm1 = torch.nn.GroupNorm(32, c, eps=eps)
    m.conv1 = torch.nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))
    m.time_emb_proj = torch.nn.Linear(temb, c)
    m.norm2 = torch.nn.GroupNorm(32, c, eps=eps)
    m.conv2 = torch.nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))
    return m


class ResBlock(torch.nn.Module):
    """Parameter container of reference crossview_temporal.py:75-164."""

    def __init__(self, in_channels, out_channels=None, temb_channels=512, eps=1e-5,
                 enable_temporal=True, temporal_eps=None, merge_factor=0.5,
                 merge_strategy="learned_with_images"):
        super().__init__()
        oc = out_channels if out_channels is not None else in_channels
        self.in_channels, self.out_channels, self.eps = in_channels, oc, eps
        self.spatial_res_block = _resnet2d(in_channels, oc, temb_channels, eps)
        if enable_temporal:
            self.temporal_res_block = _resnet_t(
                oc, temb_channels, temporal_eps if temporal_eps is not None else eps)
            self.time_mixer = AlphaBlender(merge_factor, merge_strategy=merge_strategy)
        else:
            self.temporal_res_block = None


class _BasicBlock(torch.nn.Module):
    """diffusers BasicTransformerBlock parameters."""

    def __init__(self, dim, heads, head_dim, cross_attention_dim):
        super().__init__()
        self.norm1 = torch.nn.LayerNorm(dim)
        self.attn1 = make_attention(dim, heads, head_dim, bias=False)
        self.norm2 = torch.nn.LayerNorm(dim)
        at = ParamGroup()
        inner = heads * head_dim
        cd = dim if cross_attention_dim is None else cross_attention_dim
        at.to_q = torch.nn.Linear(dim, inner, bias=False)
        at.to_k = torch.nn.Linear(cd, inner, bias=False)
        at.to_v = torch.nn.Linear(cd, inner, bias=False)
        at.to_out = torch.nn.ModuleList([torch.nn.Linear(inner, dim), torch.nn.Identity()])
        self.attn2 = at
        self.norm3 = torch.nn.LayerNorm(dim)
        self.ff = make_feed_forward(dim)


class TransformerModel(torch.nn.Module):
    """Parameter container of reference crossview_temporal.py:269-514."""

    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=320,
                 out_channels=None, enable_crossview=True, enable_temporal=True,
                 enable_rowwise_crossview=False, enable_rowwise_temporal=False,
                 num_layers=1, cross_attention_dim=None, merge_factor=0.5,
                 merge_strategy="learned_with_images"):
        super().__init__()
        if attention_head_dim != 64:
            raise NotImplementedError("attention kernels are built for head_dim 64")
        inner = num_attention_heads * attention_head_dim
        self.heads, self.inner_dim, self.in_channels = num_attention_heads, inner, in_channels
        self.norm = torch.nn.GroupNorm(32, in_channels, eps=1e-6)
        self.proj_in = torch.nn.Linear(in_channels, inner)
        self.transformer_blocks = torch.nn.ModuleList([
            _BasicBlock(inner, num_attention_heads, attention_head_dim, cross_attention_dim)
            for _ in range(num_layers)])
        self.enable_rowwise_crossview = enable_rowwise_crossview
        self.enable_rowwise_temporal = enable_rowwise_temporal
        if enable_crossview:
            self.view_pos_embed = _mlp(in_channels, in_channels * 4, in_channels)
            self.crossview_transformer_blocks = torch.nn.ModuleList([
                VTSelfAttentionBlock(inner, inner, num_attention_heads, attention_head_dim)
                for _ in range(num_layers)])
            self.view_mixer = AlphaBlender(merge_factor, merge_strategy=merge_strategy)
        else:
            self.view_pos_embed = None
        if enable_temporal:
            self.time_pos_embed = _mlp(in_channels, in_channels * 4, in_channels)
            self.temporal_transformer_blocks = torch.nn.ModuleList([
                VTSelfAttentionBlock(inner, inner, num_attention_heads, attention_head_dim)
                for _ in range(num_layers)])
            self.time_mixer = AlphaBlender(merge_factor, merge_strategy=merge_strategy)
        else:
            self.time_pos_embed = None
        self.proj_out = torch.nn.Linear(inner, in_channels)


class _Sampler(torch.nn.Module):
    def __init__(self, channels, stride):
        super().__init__()
        self.conv = torch.nn.Conv2d(channels, channels, 3, stride=stride, padding=1)


class _Block(torch.nn.Module):
    def __init__(self, kind, res_specs, attn_channels, temb, eps, heads, cross_dim, tlayers,
                 sampler, kw):
        super().__init__()
        self.kind = kind
        self.resnets = torch.nn.ModuleList([
            ResBlock(i, o, temb_channels=temb, eps=eps, enable_temporal=kw["enable_temporal"],
                     merge_factor=kw["merge_factor"]) for i, o in res_specs])
        n_attn = 0 if attn_channels is None else len(res_specs) - (1 if kind == "mid" else 0)
        if n_attn:
            self.attentions = torch.nn.ModuleList([
                TransformerModel(heads, attn_channels // heads, in_channels=attn_channels,
                                 num_layers=tlayers, cross_attention_dim=cross_dim, **kw)
                for _ in range(n_attn)])
        else:
            self.attentions = None
        if sampler == "down":
            self.downsamplers = torch.nn.ModuleList([_Sampler(res_specs[-1][1], 2)])
        elif sampler == "up":
            self.upsamplers = torch.nn.ModuleList([_Sampler(res_specs[-1][1], 1)])


class UNetCrossviewTemporalConditionModel(_compat.UNetSpatioTemporalConditionModelMarker):

    @staticmethod
    def try_to_convert_state_dict(state_dict: dict):
        """SD-2.1 checkpoints name their resnets `resnets.N.conv1...`; the SVD-style
        module tree nests them under `spatial_res_block` (reference :358-373)."""
        sd21 = re.compile(r"resnets.(\d+).conv")
        if any(sd21.search(k) is not None for k in state_dict.keys()):
            pattern = re.compile(r"resnets.(\d+)")
            return {(pattern.sub(r"resnets.\1.spatial_res_block", k)
                     if "resnets" in k else k): v for k, v in state_dict.items()}
        return state_dict

    def __init__(self, sample_size=None, in_channels: int = 8, out_channels: int = 4,
                 down_block_types=("CrossAttnDownBlockCrossviewTemporal",) * 3 +
                 ("DownBlockCrossviewTemporal",),
                 up_block_types=("UpBlockCrossviewTemporal",) +
                 ("CrossAttnUpBlockCrossviewTemporal",) * 3,
                 block_out_channels=(320, 640, 1280, 1280),
                 addition_time_embed_dim: int = 256,
                 projection_class_embeddings_input_dim=768, layers_per_block=2,
                 norm_eps: float = 1e-5, cross_attention_dim: int = 1024,
                 transformer_layers_per_block=1, num_attention_heads=(5, 10, 20, 20),
                 merge_factor: float = 0.5, enable_crossview: bool = True,
                 enable_temporal: bool = True, enable_rowwise_crossview: bool = False,
                 enable_rowwise_temporal: bool = False,
                 condition_image_adapter_config=None, depth_net_config=None,
                 depth_frustum_range=None, enforce_align_projection=None,
                 compute_dtype=None, gemm_dtype=None):
        """gemm_dtype=torch.float8_e4m3fn runs the ResBlock convolutions (spatial and temporal
        conv1 / conv2) and the transformer-block linears (except the text K/V projections) in
        E4M3; None keeps every GEMM and convolution 16-bit."""
        super().__init__()
        if gemm_dtype not in (None, torch.float8_e4m3fn):
            raise ValueError(
                "gemm_dtype must be None or torch.float8_e4m3fn, got {!r}".format(gemm_dtype))
        if depth_net_config is not None or enforce_align_projection is not None:
            raise NotImplementedError(
                "depth_net / align projection are not enabled by any shipped CTSD config")
        n = len(block_out_channels)
        boc = tuple(block_out_channels)
        temb = boc[0] * 4
        heads = (num_attention_heads,) * n if isinstance(num_attention_heads, int) \
            else tuple(num_attention_heads)
        lpb = [layers_per_block] * n if isinstance(layers_per_block, int) \
            else list(layers_per_block)
        tl = [transformer_layers_per_block] * n \
            if isinstance(transformer_layers_per_block, int) \
            else list(transformer_layers_per_block)
        kw = dict(enable_crossview=enable_crossview, enable_temporal=enable_temporal,
                  enable_rowwise_crossview=enable_rowwise_crossview,
                  enable_rowwise_temporal=enable_rowwise_temporal, merge_factor=merge_factor)
        self.config = dict(in_channels=in_channels, out_channels=out_channels,
                           block_out_channels=boc, cross_attention_dim=cross_attention_dim)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.compute_dtype = compute_dtype
        self.gemm_dtype = gemm_dtype
        self.norm_eps = norm_eps
        self.gradient_checkpointing = False
        self.conv_in = torch.nn.Conv2d(in_channels, boc[0], 3, padding=1)
        self.time_embedding = _mlp(boc[0], temb, temb)
        self.add_embedding = None if projection_class_embeddings_input_dim is None else \
            _mlp(projection_class_embeddings_input_dim, temb, temb)
        self.addition_time_embed_dim = addition_time_embed_dim
        self.down_blocks = torch.nn.ModuleList()
        oc = boc[0]
        for i, t in enumerate(down_block_types):
            ic, oc = oc, boc[i]
            specs = [(ic if j == 0 else oc, oc) for j in range(lpb[i])]
            self.down_blocks.append(_Block(
                "down", specs, oc if t.startswith("CrossAttn") else None, temb, norm_eps,
                heads[i], cross_attention_dim, tl[i], "down" if i != n - 1 else None, kw))
        self.mid_block = _Block("mid", [(boc[-1], boc[-1])] * 2, boc[-1], temb, norm_eps,
                                heads[-1], cross_attention_dim, tl[-1], None, kw)
        self.up_blocks = torch.nn.ModuleList()
        rboc, rheads = list(reversed(boc)), list(reversed(heads))
        rlpb, rtl = list(reversed(lpb)), list(reversed(tl))
        oc = rboc[0]
        for i, t in enumerate(up_block_types):
            prev, oc = oc, rboc[i]
            ic = rboc[min(i + 1, n - 1)]
            layers = rlpb[i] + 1
            specs = [((prev if j == 0 else oc) + (ic if j == layers - 1 else oc), oc)
                     for j in range(layers)]
            self.up_blocks.append(_Block(
                "up", specs, oc if t.startswith("CrossAttn") else None, temb, norm_eps,
                rheads[i], cross_attention_dim, rtl[i], "up" if i != n - 1 else None, kw))
        self.conv_norm_out = torch.nn.GroupNorm(32, boc[0], eps=1e-5)
        self.conv_out = torch.nn.Conv2d(boc[0], out_channels, 3, padding=1)
        self.condition_image_adapter = None if condition_image_adapter_config is None \
            else _adapters.ImageAdapter(**condition_image_adapter_config)
        self.depth_net = None
        self.depth_frustum_range = depth_frustum_range
        self._pk = None
        self._cond_key = None
        self._cond = None
        self._ws8, self._ws8_key = {}, None
        # opendwm_b200.sharding.ShardPlan: with t_ways > 1, `sample` holds the plan's frame
        # shard of the window; temporal ResBlocks and temporal attention exchange across it
        self.shard = None
        self._peer, self._peer_key = None, None

    # -- plumbing ---------------------------------------------------------------------------
    def enable_gradient_checkpointing(self):
        self.gradient_checkpointing = True

    def _apply(self, fn, *a, **k):
        self._pk, self._cond_key, self._cond = None, None, None
        self._ws8, self._ws8_key = {}, None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, assign=False):
        self._pk, self._cond_key, self._cond = None, None, None
        self._ws8, self._ws8_key = {}, None
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    def _dtype(self):
        if self.compute_dtype is not None:
            return self.compute_dtype
        pd = self.conv_in.weight.dtype
        return pd if pd in (torch.float16, torch.bfloat16) else torch.bfloat16

    # -- packing ------------------------------------------------------------------------------
    @torch.no_grad()
    def _pack(self):
        dev = self.conv_in.weight.device
        if dev.type != "cuda":
            raise RuntimeError("UNetCrossviewTemporalConditionModel runs on CUDA (sm_90a) "
                               "only; there is no CPU fallback. Move the model to the GPU.")
        dt = self._dtype()
        fp8 = self.gemm_dtype is not None

        temb_w, temb_b, off = [], [], [0]

        def temb_slot(linear):
            temb_w.append(linear.weight.detach())
            temb_b.append(linear.bias.detach())
            o = off[0]
            off[0] += linear.weight.shape[0]
            return (o, linear.weight.shape[0])

        def res(rb):
            s = rb.spatial_res_block
            p = dict(n1=pack_norm(s.norm1), c1=pack_conv(s.conv1, dt, dev, fp8),
                     temb=temb_slot(s.time_emb_proj), n2=pack_norm(s.norm2),
                     c2=pack_conv(s.conv2, dt, dev, fp8))
            if hasattr(s, "conv_shortcut"):
                p["sc"] = pack_linear(s.conv_shortcut.weight, s.conv_shortcut.bias, dt, dev)
            if rb.temporal_res_block is not None:
                t = rb.temporal_res_block
                p["t"] = dict(n1=pack_norm(t.norm1), c1=pack_conv(t.conv1, dt, dev, fp8),
                              temb=temb_slot(t.time_emb_proj), n2=pack_norm(t.norm2),
                              c2=pack_conv(t.conv2, dt, dev, fp8))
            return p

        def attn(tm):
            p = dict(norm=pack_norm(tm.norm),
                     proj_in=pack_linear(tm.proj_in.weight, tm.proj_in.bias, dt, dev),
                     proj_out=pack_linear(tm.proj_out.weight, tm.proj_out.bias, dt, dev),
                     blocks=[])
            for b in tm.transformer_blocks:
                a1, a2 = b.attn1, b.attn2
                ff1_w, ff1_b = _ops.pack_geglu(b.ff.net[0].proj.weight.detach().to(dev),
                                               b.ff.net[0].proj.bias.detach().to(dev))
                p["blocks"].append(dict(
                    n1=pack_norm(b.norm1),
                    qkv=pack_linear(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight]),
                                    None, dt, dev, fp8),
                    out=pack_linear(a1.to_out[0].weight, a1.to_out[0].bias, dt, dev, fp8),
                    n2=pack_norm(b.norm2),
                    q2=pack_linear(a2.to_q.weight, a2.to_q.bias, dt, dev, fp8),
                    # the step-invariant text K,V projection stays 16-bit
                    kv2=pack_linear(torch.cat([a2.to_k.weight, a2.to_v.weight]), None, dt, dev),
                    out2=pack_linear(a2.to_out[0].weight, a2.to_out[0].bias, dt, dev, fp8),
                    n3=pack_norm(b.norm3),
                    # FP8: quantized after the GEGLU row packing, scales follow the rows
                    ff1=pack_linear(ff1_w, ff1_b, dt, dev, fp8),
                    ff2=pack_linear(b.ff.net[2].weight, b.ff.net[2].bias, dt, dev, fp8)))
            if tm.view_pos_embed is not None:
                p["vpe"] = tuple(pack_linear(m.weight, m.bias, dt, dev) for m in (
                    tm.view_pos_embed.linear_1, tm.view_pos_embed.linear_2))
                p["cv"] = [b.pack(dt, dev, fp8) for b in tm.crossview_transformer_blocks]
            if tm.time_pos_embed is not None:
                p["tpe"] = tuple(pack_linear(m.weight, m.bias, dt, dev) for m in (
                    tm.time_pos_embed.linear_1, tm.time_pos_embed.linear_2))
                p["tp"] = [b.pack(dt, dev, fp8) for b in tm.temporal_transformer_blocks]
            return p

        def block(b):
            p = dict(res=[res(r) for r in b.resnets],
                     attn=None if b.attentions is None else [attn(a) for a in b.attentions])
            if hasattr(b, "downsamplers"):
                p["down"] = pack_conv(b.downsamplers[0].conv, dt, dev)
            if hasattr(b, "upsamplers"):
                p["up"] = pack_conv(b.upsamplers[0].conv, dt, dev)
            return p

        cin_p = (self.in_channels + 7) // 8 * 8
        pk = dict(dtype=dt, fp8=fp8, cin_p=cin_p,
                  conv_in=pack_conv(self.conv_in, dt, dev, pad_in=cin_p),
                  te=tuple(pack_linear(m.weight, m.bias, dt, dev) for m in (
                      self.time_embedding.linear_1, self.time_embedding.linear_2)),
                  down=[block(b) for b in self.down_blocks], mid=block(self.mid_block),
                  up=[block(b) for b in self.up_blocks],
                  norm_out=pack_norm(self.conv_norm_out),
                  conv_out=pack_conv(self.conv_out, dt, dev,
                                     pad_out=32 if self.out_channels < 32 else None))
        if self.add_embedding is not None:
            pk["ae"] = tuple(pack_linear(m.weight, m.bias, dt, dev) for m in (
                self.add_embedding.linear_1, self.add_embedding.linear_2))
        pk["temb"] = pack_linear(torch.cat(temb_w), torch.cat(temb_b), dt, dev)
        self._pk = pk
        return pk

    # -- helpers --------------------------------------------------------------------------------
    def _gn(self, h, N, H, W, g, silu):
        """GroupNorm(32)(+SiLU) of fp32 tokens [N*H*W, C] -> 16-bit [N, 1, H, W, C]."""
        C = h.shape[1]
        h5 = h.view(N, 1, H, W, C)
        sums = _ops.groupnorm_stats(h5, 32)
        out = torch.empty(N, 1, H, W, C, device=h.device, dtype=self._pk["dtype"])
        _ops.spatialnorm_silu(h5, sums, g[0], g[1], out, groups=32, eps=g[2], silu=silu)
        return out

    def _buf8(self, key, shape, dtype):
        """E4M3 workspace (operands, volume scales) kept across calls of one input geometry,
        so that a CUDA-graph replay reads and writes the buffers the capture recorded.  The
        buffers start zeroed: the temporal convs rely on zero cache frames."""
        k = (key, tuple(shape), dtype)
        if k not in self._ws8:
            self._ws8[k] = torch.zeros(shape, device=self.conv_in.weight.device, dtype=dtype)
        return self._ws8[k]

    def _norm_act(self, x5, g, out_T=None, out_t0=0):
        """GroupNorm(32)+SiLU of fp32 [nb, T, H, W, C] as a conv operand [nb, out_T, H, W, C]
        whose frames outside [out_t0, out_t0 + T) are zero: 16-bit, or with gemm_dtype E4M3
        with one fp32 scale per volume nb (in the persistent `_buf8` workspace)."""
        nb, T, H, W, C = x5.shape
        out_T = T if out_T is None else out_T
        sums = _ops.groupnorm_stats(x5, 32)
        if self._pk["fp8"]:
            out = self._buf8("gn", (nb, out_T, H, W, C), FP8)
            sc = self._buf8("gn_s", (nb,), torch.float32)
            return Operand(*_ops.groupnorm_silu_e4m3(x5, sums, g[0], g[1], out, sc, groups=32,
                                                     eps=g[2], out_t0=out_t0, silu=True))
        # a fresh buffer per call; the frames a temporal conv pads with must be zero
        out = (torch.empty if out_T == T else torch.zeros)(
            nb, out_T, H, W, C, device=x5.device, dtype=self._pk["dtype"])
        return _ops.spatialnorm_silu(x5, sums, g[0], g[1], out, groups=32, eps=g[2],
                                     out_t0=out_t0, silu=True)

    def _frame_sharded(self):
        return self.shard is not None and self.shard.t_ways > 1

    def _view_sharded(self):
        return self.shard is not None and self.shard.v_ways > 1

    def _peer_buffers(self, geo, H, W):
        """Symmetric-memory K,V (PeerKV) and temporal-conv operand (PeerHalo) buffers of the
        frame group, and the K,V buffers (PeerKV) of the view group, sized once per input
        geometry for the largest level (channels x pixels) and shared by all temporal /
        cross-view blocks in forward order: creating them is collective, so it must not happen
        per block or per step.  None for a group the plan does not split, and all None with
        DWM_PEER_SCATTER=0."""
        plan = self.shard
        dt = self._pk["dtype"]
        key = (id(plan), geo, H, W, dt)
        if self._peer_key != key:
            self._peer, self._peer_key = (None, None, None), key
            if plan.use_peer_scatter:
                from opendwm_b200.sharding import PeerHalo, PeerKV
                B, T, V = geo
                widest, h, w = 0, H, W
                for c in self.config["block_out_channels"]:
                    widest = max(widest, c * h * w)
                    h, w = (h + 1) // 2, (w + 1) // 2
                dev = self.conv_in.weight.device
                frames = self._frame_sharded()
                self._peer = (
                    PeerKV(plan, B * plan.T * V * widest, 2, dt, dev) if frames else None,
                    PeerHalo(plan, B * V * (max(plan.counts) + 2) * widest * dt.itemsize, dev)
                    if frames else None,
                    PeerKV(plan, B * T * plan.V * widest, 2, dt, dev, axis="v")
                    if self._view_sharded() else None)
        return self._peer

    def _norm_act_shard(self, x5, g):
        """`_norm_act` of a frame shard x5 [nb, T_loc, H, W, C] into the temporal-conv operand
        [nb, T_loc + 2, H, W, C]: GroupNorm statistics (and in E4M3 the volume amax) reduced
        over the window's frames, frames 0 and T_loc + 1 the neighbour shards' boundary frames
        (zero at the window's ends)."""
        plan = self.shard
        nb, T, H, W, C = x5.shape
        fp8 = self._pk["fp8"]
        dt = FP8 if fp8 else self._pk["dtype"]
        sums = plan.reduce_group_sums(_ops.groupnorm_stats(x5, 32))
        halo = self._peer[1]
        if halo is not None:       # fused: the kernel stores the halo frames into the peers
            out, prev, nxt, hdl = halo.next((nb, T + 2, H, W, C), dt)
        else:
            out, prev, nxt, hdl = torch.empty(nb, T + 2, H, W, C, device=x5.device,
                                              dtype=dt), None, None, None
        kw = dict(groups=32, stat_frames=plan.T, prev_out=prev, next_out=nxt, eps=g[2])
        if fp8:
            amax = torch.empty(nb, device=x5.device, dtype=torch.float32)
            _ops.groupnorm_silu_e4m3_amax(x5, sums, g[0], g[1], amax, groups=32,
                                          stat_frames=plan.T, eps=g[2])
            plan.reduce_amax(amax)
            res = Operand(*_ops.groupnorm_silu_e4m3_halo(
                x5, sums, g[0], g[1], amax, out, torch.empty_like(amax), **kw))
        else:
            res = _ops.groupnorm_silu_halo(x5, sums, g[0], g[1], out, **kw)
        if hdl is not None:
            hdl.barrier(channel=0)
        else:
            plan.exchange_halo(out)
        return res

    def _resblock(self, p, h, N, H, W, temb_all, geo, dis_t, alpha_mod):
        S = H * W

        def norm_act(t, g):    # one scale per item in E4M3
            return self._norm_act(t.view(N, 1, H, W, t.shape[1]), g)
        a = norm_act(h, p["n1"])
        o, n = p["temb"]
        h1 = conv(a, p["c1"], kernel=(1, 3, 3), epilogue=_lib.EPI_RESID,
                  resid=temb_all[:, o:o + n], resid_rows_per_item=S)
        b = norm_act(h1, p["n2"])
        if "sc" in p:
            h16 = torch.empty(h.shape, device=h.device, dtype=self._pk["dtype"])
            _ops.act_cast(h, h16)
            skip = gemm(h16, p["sc"], epilogue=_lib.EPI_F32)
        else:
            skip = h
        out = conv(b, p["c2"], kernel=(1, 3, 3), epilogue=_lib.EPI_RESID, resid=skip)
        if "t" in p and not dis_t["all"]:
            out = self._temporal_res(p["t"], out, N, H, W, temb_all, geo, alpha_mod)
        return out

    def _temporal_res(self, p, x, N, H, W, temb_all, geo, mixer):
        """TemporalResnetBlock (conv3d (3,1,1), GroupNorm over (T,H,W)) + AlphaBlender on
        the `(b v) t` volumes; (b t v) <-> (b v t) regrouping is a data-movement permute."""
        B, T, V = geo
        S, C = H * W, x.shape[1]
        xp = x.view(B, T, V, S, C).permute(0, 2, 1, 3, 4).contiguous()      # [B,V,T,S,C]
        x5 = xp.view(B * V, T, 1, S, C)
        o, n = p["temb"]
        temb_p = temb_all[:, o:o + n].reshape(B, T, V, n).permute(0, 2, 1, 3)\
            .reshape(B * V * T, n).contiguous()

        def norm_act(t5, g):    # T + 2 frames, zero at both ends; E4M3: one scale per (b v)
            if self._frame_sharded():     # ends: the neighbour shards' frames
                return self._norm_act_shard(t5, g)
            return self._norm_act(t5, g, out_T=T + 2, out_t0=1)
        h1 = conv(norm_act(x5, p["n1"]), p["c1"], kernel=(3, 1, 1),
                  epilogue=_lib.EPI_RESID, resid=temb_p, resid_rows_per_item=S)
        xr = xp.view(B * V * T * S, C)
        alpha = mixer["alpha"]
        y = conv(norm_act(h1.view(B * V, T, 1, S, C), p["n2"]), p["c2"],
                 kernel=(3, 1, 1), epilogue=_lib.EPI_RESID, resid=xr, blend_x=xr,
                 alpha=alpha, rows_per_batch=V * T * S)
        return y.view(B, V, T, S, C).permute(0, 2, 1, 3, 4).reshape(B * T * V * S, C)\
            .contiguous()

    def _index_table(self, count, mlp, C, dev, dt):
        idx = torch.arange(count, device=dev, dtype=torch.float32)
        sn = torch.empty(count, C, device=dev, dtype=dt)
        _ops.sinusoid(idx, C, sn, True, 0.0)
        hmid = gemm(sn, mlp[0], act=_lib.ACT_SILU)
        return gemm(hmid, mlp[1], epilogue=_lib.EPI_F32)

    def _transformer(self, tm, p, x, N, H, W, geo, cd, level_key):
        """TransformerModel forward on fp32 tokens x [N*S, C]; returns x + proj_out(...)."""
        B, T, V = geo
        S, dt, dev = H * W, self._pk["dtype"], x.device
        inner, heads = tm.inner_dim, tm.heads
        a16 = self._gn(x, N, H, W, p["norm"], False).view(N * S, -1)
        h = gemm(a16, p["proj_in"], epilogue=_lib.EPI_F32)
        ws = dict(y=torch.empty_like(h), a16=torch.empty(N * S, inner, device=dev, dtype=dt),
                  g16=torch.empty(N * S, 4 * inner, device=dev, dtype=dt),
                  qkv_s=torch.empty(N * S, 3 * inner, device=dev, dtype=dt),
                  o16=torch.empty(N * S, inner, device=dev, dtype=dt))
        # GEMM operands: the LayerNorm output (a) and the E4M3 buffer the 16-bit attention /
        # GEGLU outputs are requantized into (q; None in 16 bit); the VTSelfAttentionBlocks
        # use the same keys
        if self._pk["fp8"]:
            ws["a"], ws["q"] = (
                Operand(self._buf8(k, (N * S, cols), FP8),
                        self._buf8(k + "_s", (N * S,), torch.float32))
                for k, cols in (("a8", inner), ("q8", 4 * inner)))
        else:
            ws["a"], ws["q"] = Operand(ws["a16"]), None
        a, q = ws["a"], ws["q"]
        ctx = cd["ctx16"]
        Lc = cd["ctx_len"]
        key = (level_key, "tabs")
        if key not in cd:
            tabs = {}
            item_v = torch.arange(V, device=dev).view(1, 1, V).expand(B, T, V).reshape(-1)
            item_t = torch.arange(T, device=dev).view(1, T, 1).expand(B, T, V).reshape(-1)
            if "vpe" in p:
                if self._view_sharded():      # view index within all views
                    tab = self._index_table(self.shard.V, p["vpe"], tm.in_channels, dev, dt)
                    item_v = item_v + self.shard.v_offset
                else:
                    tab = self._index_table(V, p["vpe"], tm.in_channels, dev, dt)
                tabs["v"] = tab[item_v].contiguous()
            if "tpe" in p:
                if self._frame_sharded():     # frame index within the whole window
                    tab = self._index_table(self.shard.T, p["tpe"], tm.in_channels, dev, dt)
                    item_t = item_t + self.shard.t_offset
                else:
                    tab = self._index_table(T, p["tpe"], tm.in_channels, dev, dt)
                tabs["t"] = tab[item_t].contiguous()
            cd[key] = tabs
        tabs = cd[key]
        tp_sharded = None
        if "tp" in p and self._frame_sharded():
            plan, rows = self.shard, N * S
            peer_kv = self._peer[0]
            kv_loc = kv_all = None
            if peer_kv is None:
                kv_loc = torch.empty(rows, 2 * inner, device=dev, dtype=dt)
                kv_all = torch.empty(B * plan.T * V * S, 2 * inner, device=dev, dtype=dt)
            tp_sharded = sharded_temporal_qkv_attend(
                plan, "rowwise" if tm.enable_rowwise_temporal else "pointwise", B, T, V, H, W,
                inner, heads, torch.empty(rows, inner, device=dev, dtype=dt), peer_kv=peer_kv,
                kv_loc=kv_loc, kv_all=kv_all)
        cv_sharded = None
        if "cv" in p and self._view_sharded():
            if not tm.enable_rowwise_crossview:
                raise NotImplementedError(
                    "point-wise cross-view attention under a view shard: only row-wise "
                    "cross-view attention is sharded")
            plan, rows = self.shard, N * S
            peer_kv = self._peer[2]
            kv_loc = kv_all = None
            if peer_kv is None:
                kv_loc = torch.empty(rows, 2 * inner, device=dev, dtype=dt)
                kv_all = torch.empty(B * T * plan.V * S, 2 * inner, device=dev, dtype=dt)
            cv_sharded = sharded_crossview_qkv_attend(
                plan, B * T, H, W, inner, heads, torch.empty(rows, inner, device=dev, dtype=dt),
                cd["mask"], T, peer_kv=peer_kv, kv_loc=kv_loc, kv_all=kv_all)
        for li, bp in enumerate(p["blocks"]):
            # --- spatial BasicTransformerBlock: self-attn, cross-attn to text, GEGLU FF
            n = bp["n1"]
            layernorm(h, a, weight=n[0], bias=n[1], eps=n[2])
            gemm(a, bp["qkv"], out=ws["qkv_s"])
            _ops.attention(ws["qkv_s"], ws["o16"], D=inner, heads=heads, group_dims=[N],
                           group_strides=[S], seq=S)
            gemm(requantize(ws["o16"], q), bp["out"], epilogue=_lib.EPI_RESID, resid=h, out=h)
            n = bp["n2"]
            layernorm(h, a, weight=n[0], bias=n[1], eps=n[2])
            q2 = gemm(a, bp["q2"], out=ws["qkv_s"][:, :inner])
            kkey = (level_key, li, "kv")
            if kkey not in cd:        # text K,V are step-invariant
                cd[kkey] = gemm(ctx, bp["kv2"])
            kv = cd[kkey]
            _ops.attention(q2, ws["o16"], D=inner, heads=heads, group_dims=[N],
                           group_strides=[S], seq=S, kv=kv, k_col=0, v_col=inner,
                           kv_group_strides=[Lc], seq_kv=Lc)
            gemm(requantize(ws["o16"], q), bp["out2"], epilogue=_lib.EPI_RESID, resid=h, out=h)
            n = bp["n3"]
            layernorm(h, a, weight=n[0], bias=n[1], eps=n[2])
            gemm(a, bp["ff1"], epilogue=_lib.EPI_GEGLU, out=ws["g16"])
            gemm(requantize(ws["g16"], q), bp["ff2"], epilogue=_lib.EPI_RESID, resid=h, out=h)
            # --- cross-view block
            if "cv" in p and not cd["dis_cv"]["all"]:
                if tm.enable_rowwise_crossview:   # (bt h) x (v w), view mask per (vq, vk)
                    def attend(qkv, out):
                        _ops.attention(qkv, out, D=inner, heads=heads, group_dims=[B * T, H],
                                       group_strides=[V * S, W], seq=V * W, inner=W,
                                       stride_outer=S, stride_inner=1, mask=cd["mask"],
                                       mask_div=T)
                else:                              # (bt hw) x v
                    if cd["mask"] is not None:
                        raise NotImplementedError(
                            "view mask with point-wise cross-view attention")

                    def attend(qkv, out):
                        _ops.attention(qkv, out, D=inner, heads=heads, group_dims=[B * T, S],
                                       group_strides=[V * S, 1], seq=V, inner=1,
                                       stride_outer=S, stride_inner=0)
                tm.crossview_transformer_blocks[li].run(
                    p["cv"][li], h, tabs["v"], S, ws, attend,
                    tm.view_mixer.batch_alpha(B, cd["dis_cv"]["t"], dev), T * V * S,
                    qkv_attend=cv_sharded)
            # --- temporal block
            if "tp" in p and not cd["dis_t"]["all"]:
                if tm.enable_rowwise_temporal:    # (b v h) x (t w)
                    def attend(qkv, out):
                        _ops.attention(qkv, out, D=inner, heads=heads, group_dims=[B, V, H],
                                       group_strides=[T * V * S, S, W], seq=T * W, inner=W,
                                       stride_outer=V * S, stride_inner=1)
                else:                              # (b v hw) x t
                    def attend(qkv, out):
                        _ops.attention(qkv, out, D=inner, heads=heads, group_dims=[B, V * S],
                                       group_strides=[T * V * S, 1], seq=T, inner=1,
                                       stride_outer=V * S, stride_inner=0)
                tm.temporal_transformer_blocks[li].run(
                    p["tp"][li], h, tabs["t"], S, ws, attend,
                    tm.time_mixer.batch_alpha(B, cd["dis_t"]["t"], dev), T * V * S,
                    qkv_attend=tp_sharded)
        h16 = torch.empty(h.shape, device=dev, dtype=dt)
        _ops.act_cast(h, h16)
        return gemm(h16, p["proj_out"], epilogue=_lib.EPI_RESID, resid=x)

    def _run_block(self, blk, p, h, N, H, W, temb_all, geo, cd, name, skips=None):
        outs = []
        dis_t = cd["dis_t"]

        def mixer(rb):
            return None if rb.temporal_res_block is None else dict(
                alpha=rb.time_mixer.batch_alpha(geo[0], dis_t["t"], h.device))
        if blk.kind == "mid":
            h = self._resblock(p["res"][0], h, N, H, W, temb_all, geo, dis_t,
                               mixer(blk.resnets[0]))
            for j, (tm, ap) in enumerate(zip(blk.attentions, p["attn"])):
                h = self._transformer(tm, ap, h, N, H, W, geo, cd, (name, j))
                h = self._resblock(p["res"][j + 1], h, N, H, W, temb_all, geo, dis_t,
                                   mixer(blk.resnets[j + 1]))
            return h, outs, H, W
        for j, rp in enumerate(p["res"]):
            if skips is not None:
                h = torch.cat([h, skips[-1 - j]], dim=1)          # channel concat
            h = self._resblock(rp, h, N, H, W, temb_all, geo, dis_t, mixer(blk.resnets[j]))
            if p["attn"] is not None:
                h = self._transformer(blk.attentions[j], p["attn"][j], h, N, H, W, geo, cd,
                                      (name, j))
            outs.append(h)
        dt = self._pk["dtype"]
        if "down" in p:
            # stride-2 conv == stride-1 conv sampled at even pixels (padding 1)
            C = h.shape[1]
            h16 = torch.empty(h.shape, device=h.device, dtype=dt)
            _ops.act_cast(h, h16)
            full = conv(h16.view(N, 1, H, W, C), p["down"], kernel=(1, 3, 3),
                        epilogue=_lib.EPI_F32)
            h = full.view(N, H, W, C)[:, ::2, ::2].reshape(-1, C).contiguous()
            H, W = (H + 1) // 2, (W + 1) // 2
            outs.append(h)
        if "up" in p:
            C = h.shape[1]
            u = _ops.upsample_nearest(h.view(N, 1, H, W, C), False, dt)
            H, W = 2 * H, 2 * W
            h = conv(u, p["up"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        return h, outs, H, W

    # -- conditions cache ------------------------------------------------------------------------
    @staticmethod
    def _tkey(t):
        return None if t is None else (t.data_ptr(), tuple(t.shape), t.dtype, t._version)

    def _conditions(self, geo, H, W, encoder_hidden_states, condition_image_tensor,
                    added_time_ids, disable_crossview, disable_temporal, mask):
        # the frame / view index tables depend on where a shard sits in the window
        shard = (self.shard.T, self.shard.t_offset, self.shard.V, self.shard.v_offset) \
            if self._frame_sharded() or self._view_sharded() else None
        key = (geo, H, W, shard) + tuple(self._tkey(t) for t in (
            encoder_hidden_states, condition_image_tensor, added_time_ids, disable_crossview,
            disable_temporal, mask))
        if key == self._cond_key:
            return self._cond
        # keep the keyed tensors alive so their addresses cannot be recycled under the key
        self._cond_refs = (encoder_hidden_states, condition_image_tensor, added_time_ids,
                           disable_crossview, disable_temporal, mask)
        B, T, V = geo
        pk, dt = self._pk, self._pk["dtype"]
        dev = encoder_hidden_states.device
        N = B * T * V
        cd = {}
        ehs = encoder_hidden_states.flatten(0, 2)
        cd["ctx_len"] = ehs.shape[1]
        cd["ctx16"] = ehs.reshape(N * ehs.shape[1], -1).to(dt).contiguous()
        cd["aug"] = None
        if added_time_ids is not None and "ae" in pk:
            ids = added_time_ids.flatten().float().contiguous()
            sn = torch.empty(ids.numel(), self.addition_time_embed_dim, device=dev, dtype=dt)
            _ops.sinusoid(ids, self.addition_time_embed_dim, sn, True, 0.0)
            hm = gemm(sn.view(N, -1), pk["ae"][0], act=_lib.ACT_SILU)
            cd["aug"] = gemm(hm, pk["ae"][1], epilogue=_lib.EPI_F32)

        def flags(t):
            t = torch.zeros(B, dtype=torch.bool, device=dev) if t is None else \
                t.flatten().to(dev)
            return dict(t=t, all=bool(t.all().item()))     # one sync per condition set
        cd["dis_cv"], cd["dis_t"] = flags(disable_crossview), flags(disable_temporal)
        cd["mask"] = None if mask is None else mask.to(dev).ne(0).to(torch.uint8).contiguous()
        cd["residuals"] = []
        if self.condition_image_adapter is not None and condition_image_tensor is not None:
            cd["residuals"] = self.condition_image_adapter.token_features(
                condition_image_tensor.to(dev), dt)
        self._cond_key, self._cond = key, cd
        return cd

    # -- forward ------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timesteps, frustum_bev_residuals=None,
                encoder_hidden_states=None, condition_image_tensor=None,
                disable_crossview=None, disable_temporal=None,
                crossview_attention_mask=None, camera_intrinsics=None,
                camera_transforms=None, added_time_ids=None, camera_intrinsics_norm=None,
                camera2referego=None, return_dict=False):
        if frustum_bev_residuals is not None or isinstance(encoder_hidden_states, dict):
            raise NotImplementedError("frustum_bev_residuals / dict conditions (HoloDrive, "
                                      "align projection) are outside the CTSD hot path")
        if not sample.is_cuda:
            raise RuntimeError("UNetCrossviewTemporalConditionModel needs CUDA tensors; "
                               "there is no CPU fallback.")
        should_add_dim = len(sample.shape) < 6
        if should_add_dim:        # reference :698-707
            sample = sample.unsqueeze(2)
            timesteps = timesteps.unsqueeze(2)
            if condition_image_tensor is not None:
                condition_image_tensor = condition_image_tensor.unsqueeze(2)
            if encoder_hidden_states is not None:
                encoder_hidden_states = encoder_hidden_states.unsqueeze(2)
        if self._pk is None:
            self._pack()
        pk, dt = self._pk, self._pk["dtype"]
        B, T, V, Cin, H, W = sample.shape
        N, geo, dev = B * T * V, (B, T, V), sample.device
        if self._ws8_key != (B, T, V, H, W):     # one live E4M3 workspace
            self._ws8, self._ws8_key = {}, (B, T, V, H, W)
        if self._frame_sharded() and T != self.shard.T_loc:
            raise ValueError("sample holds {} frames, the ShardPlan's shard {}".format(
                T, self.shard.T_loc))
        if self._view_sharded() and V != self.shard.V_loc:
            raise ValueError("sample holds {} views, the ShardPlan's shard {}".format(
                V, self.shard.V_loc))
        if self._frame_sharded() or self._view_sharded():
            self._peer_buffers(geo, H, W)
        cd = self._conditions(geo, H, W, encoder_hidden_states, condition_image_tensor,
                              added_time_ids, disable_crossview, disable_temporal,
                              crossview_attention_mask)
        # 1. time embeddings: emb = time_embedding(sin(t)) [+ add_embedding(sin(ids))]
        tsin = torch.empty(N, pk["te"][0].w.shape[1], device=dev, dtype=dt)
        _ops.sinusoid(timesteps.flatten().float().contiguous(), tsin.shape[1], tsin, True, 0.0)
        hm = gemm(tsin, pk["te"][0], act=_lib.ACT_SILU)
        if cd["aug"] is not None:
            emb = gemm(hm, pk["te"][1], epilogue=_lib.EPI_RESID, resid=cd["aug"])
        else:
            emb = gemm(hm, pk["te"][1], epilogue=_lib.EPI_F32)
        emb16 = torch.empty(emb.shape, device=dev, dtype=dt)
        _ops.act_cast(emb, emb16, _lib.ACT_SILU)
        # every ResBlock's time_emb_proj(SiLU(emb)) in one GEMM
        temb_all = gemm(emb16, pk["temb"], epilogue=_lib.EPI_F32)
        # 2. conv_in on channels-last 16-bit input
        x = torch.zeros(N, 1, H, W, pk["cin_p"], device=dev, dtype=dt)
        x[..., :Cin] = sample.reshape(N, Cin, H, W).permute(0, 2, 3, 1).unsqueeze(1)
        h = conv(x, pk["conv_in"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        residuals = list(cd["residuals"])
        if residuals:
            _ops.axpy(residuals.pop(0), h)
        skips = [h]
        cH, cW = H, W
        for i, (blk, bp) in enumerate(zip(self.down_blocks, pk["down"])):
            h, outs, cH, cW = self._run_block(blk, bp, h, N, cH, cW, temb_all, geo, cd,
                                              ("down", i))
            if residuals:
                h = h.clone() if (outs and outs[-1] is h) else h
                _ops.axpy(residuals.pop(0), h)
                outs = outs[:-1] + [h]
            skips += outs
        h, _, cH, cW = self._run_block(self.mid_block, pk["mid"], h, N, cH, cW, temb_all, geo,
                                       cd, ("mid", 0))
        for i, (blk, bp) in enumerate(zip(self.up_blocks, pk["up"])):
            k = len(blk.resnets)
            res, skips = skips[-k:], skips[:-k]
            h, _, cH, cW = self._run_block(blk, bp, h, N, cH, cW, temb_all, geo, cd,
                                           ("up", i), skips=res)
        a = self._gn(h, N, cH, cW, pk["norm_out"], True)
        y = conv(a, pk["conv_out"], kernel=(1, 3, 3), epilogue=_lib.EPI_F32)
        out = y.view(N, cH, cW, -1)[..., :self.out_channels].permute(0, 3, 1, 2)\
            .reshape(B, T, V, self.out_channels, cH, cW).contiguous()
        out = out.to(sample.dtype if sample.dtype.is_floating_point else torch.float32)
        if should_add_dim:
            out = out.squeeze(2)
        if return_dict:
            return {"noise_pred": out}
        # the reference returns ((sample,), up_feature_list, down_feature_list) (:826-833)
        return (out,), [], []
