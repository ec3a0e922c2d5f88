"""CTSD-3.x MMDiT with cross-view / temporal grafts — H100-native mirror of reference
src/dwm/models/crossview_temporal_dit.py:105-630 (`DiTCrossviewTemporalConditionModel`,
a subclass of diffusers `SD3Transformer2DModel`).

Same constructor kwargs (the JSON config keys), same `forward` signature and return
value, same state_dict key names (SURVEY.md Appendix B) — but the forward is a fixed
sequence of `opendwm_b200` kernel launches over pre-packed 16-bit weights:

  * every Linear (incl. patchify conv, AdaLN linears, FFNs, q/k/v/out) is the wgmma
    GEMM with a fused epilogue (bias, GELU, GEGLU, per-head RMSNorm, gate*x+residual,
    AlphaBlender);
  * LayerNorm + AdaLN modulation emit the next GEMM operand in one pass;
  * the joint / cross-view / temporal attentions gather their token groups in place
    (no permuted copies; the reference materialises two per block);
  * everything that does not depend on latents/timestep (context_embedder, pooled-text
    embedding, view / frame index embeddings, ImageAdapter residuals, blend alphas) is
    computed once per condition set and cached (the reference recomputes it every
    step, crossview_temporal_dit.py:422-423,459-462,528-568);
  * no host synchronisation inside the forward (the reference does 25 `.item()`s).

With `shard=(rank, world, group)` the frame axis T is sharded across GPUs: cross-view
blocks stay local, temporal blocks all-gather the post-norm K,V of their frames.
"""
from typing import Optional

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops

from .. import _compat
from . import adapters as _adapters
from .crossview_temporal import (
    AlphaBlender, ParamGroup, VTSelfAttentionBlock, make_attention, make_feed_forward,
    sharded_crossview_qkv_attend, sharded_temporal_qkv_attend)
from .packing import (
    FP8, Operand, fp32, fp8_bytes_saved, gemm, layernorm, pack_linear, requantize)


def _sincos_2d(embed_dim, grid_size, base_size, device):
    """2-D sin-cos table of diffusers PatchEmbed (get_2d_sincos_pos_embed),
    computed in float64 on `device`."""
    g = torch.arange(grid_size, dtype=torch.float64, device=device) / \
        (grid_size / base_size)
    gw, gh = torch.meshgrid(g, g, indexing="xy")  # w varies fastest

    def one(pos, dim):
        omega = torch.arange(dim // 2, dtype=torch.float64, device=device)
        omega = 1.0 / 10000 ** (omega / (dim / 2.0))
        out = pos.reshape(-1)[:, None] * omega[None]
        return torch.cat([torch.sin(out), torch.cos(out)], dim=1)

    emb = torch.cat([one(gw, embed_dim // 2), one(gh, embed_dim // 2)], dim=1)
    return emb.float().unsqueeze(0)


class _PatchEmbed(torch.nn.Module):
    def __init__(self, sample_size, patch_size, in_channels, embed_dim,
                 pos_embed_max_size):
        super().__init__()
        self.patch_size = patch_size
        self.pos_embed_max_size = pos_embed_max_size
        self.proj = torch.nn.Conv2d(
            in_channels, embed_dim, patch_size, patch_size, bias=True)
        dev = self.proj.weight.device
        self.register_buffer("pos_embed", _sincos_2d(
            embed_dim, pos_embed_max_size, sample_size // patch_size,
            dev if dev.type != "meta" else "cpu"), persistent=True)

    def cropped(self, height, width):
        m = self.pos_embed_max_size
        top, left = (m - height) // 2, (m - width) // 2
        pe = self.pos_embed.reshape(1, m, m, -1)
        return pe[0, top:top + height, left:left + width, :]\
            .reshape(height * width, -1).float().contiguous()


def _mlp(in_dim, hidden, out_dim):
    m = ParamGroup()
    m.linear_1 = torch.nn.Linear(in_dim, hidden)
    m.linear_2 = torch.nn.Linear(hidden, out_dim)
    return m


class _JointBlock(torch.nn.Module):
    """Parameter layout of diffusers JointTransformerBlock (SURVEY Appendix B)."""

    def __init__(self, dim, heads, head_dim, context_pre_only, qk_norm, dual):
        super().__init__()
        self.context_pre_only = context_pre_only
        self.dual = dual
        self.norm1 = ParamGroup()
        self.norm1.linear = torch.nn.Linear(dim, (9 if dual else 6) * dim)
        self.norm1_context = ParamGroup()
        self.norm1_context.linear = torch.nn.Linear(
            dim, (2 if context_pre_only else 6) * dim)
        self.attn = make_attention(
            dim, heads, head_dim, bias=True, qk_norm=qk_norm, eps=1e-6,
            added_kv_proj_dim=dim, context_pre_only=context_pre_only)
        if dual:
            self.attn2 = make_attention(
                dim, heads, head_dim, bias=True, qk_norm=qk_norm, eps=1e-6)
        self.ff = make_feed_forward(dim, activation_fn="gelu-approximate")
        if not context_pre_only:
            self.ff_context = make_feed_forward(
                dim, activation_fn="gelu-approximate")


class DiTCrossviewTemporalConditionModel(_compat.SD3Transformer2DModelMarker):

    def __init__(
        self,
        sample_size: int = 128,
        patch_size: int = 2,
        in_channels: int = 16,
        num_layers: int = 18,
        attention_head_dim: int = 64,
        num_attention_heads: int = 18,
        joint_attention_dim: int = 4096,
        caption_projection_dim: int = 1152,
        pooled_projection_dim: int = 2048,
        out_channels: int = 16,
        pos_embed_max_size: int = 96,
        dual_attention_layers=(),
        qk_norm: Optional[str] = None,
        projection_class_embeddings_input_dim: int = None,
        condition_image_adapter_config: Optional[dict] = None,
        enable_crossview: bool = False,
        enable_temporal: bool = False,
        crossview_attention_type: str = None,
        temporal_attention_type: str = None,
        merge_factor: float = 2, merge_strategy="learned_with_images",
        crossview_block_layers: Optional[list] = None,
        temporal_block_layers: Optional[list] = None,
        crossview_gradient_checkpointing: bool = False,
        temporal_gradient_checkpointing: bool = False,
        mixer_type: str = "AlphaBlender",
        perspective_modeling_type: str = "",
        disable_view_emb_on_temporal_module: bool = False,
        qk_norm_on_additional_modules=None,
        mask_module=None,
        compute_dtype=None,
        gemm_dtype=None,
    ):
        """gemm_dtype=torch.float8_e4m3fn runs the linears inside the joint and the
        cross-view / temporal blocks as E4M3 GEMMs (per-row activation and per-channel weight
        scales); None keeps every GEMM 16-bit."""
        super().__init__()
        if gemm_dtype not in (None, torch.float8_e4m3fn):
            raise ValueError(
                "gemm_dtype must be None or torch.float8_e4m3fn, got {!r}".format(gemm_dtype))
        if attention_head_dim != 64:
            raise NotImplementedError("kernels are built for head_dim 64")
        if mixer_type != "AlphaBlender":
            raise NotImplementedError(
                "mixer_type {} (all shipped CTSD configs use AlphaBlender)"
                .format(mixer_type))
        if mask_module is not None:
            raise NotImplementedError(
                "mask_module is training-only (MaskGWM) and out of scope")
        if perspective_modeling_type not in ("", "implicit"):
            raise NotImplementedError(
                "perspective_modeling_type {}".format(perspective_modeling_type))
        inner_dim = attention_head_dim * num_attention_heads
        if caption_projection_dim != inner_dim:
            raise ValueError("caption_projection_dim must equal the inner dim")
        self.config = dict(
            sample_size=sample_size, patch_size=patch_size,
            in_channels=in_channels, num_layers=num_layers,
            attention_head_dim=attention_head_dim,
            num_attention_heads=num_attention_heads,
            joint_attention_dim=joint_attention_dim,
            caption_projection_dim=caption_projection_dim,
            pooled_projection_dim=pooled_projection_dim,
            out_channels=out_channels, pos_embed_max_size=pos_embed_max_size,
            dual_attention_layers=tuple(dual_attention_layers), qk_norm=qk_norm)
        self.inner_dim = inner_dim
        self.heads = num_attention_heads
        self.patch_size = patch_size
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.compute_dtype = compute_dtype
        self.gemm_dtype = gemm_dtype
        self.gradient_checkpointing = False
        self.crossview_gradient_checkpointing = crossview_gradient_checkpointing
        self.temporal_gradient_checkpointing = temporal_gradient_checkpointing
        self.disable_view_emb_on_temporal_module = \
            disable_view_emb_on_temporal_module

        # ---- members inherited from SD3Transformer2DModel in the reference ----
        self.pos_embed = _PatchEmbed(
            sample_size, patch_size, in_channels, inner_dim, pos_embed_max_size)
        self.time_text_embed = ParamGroup()
        self.time_text_embed.timestep_embedder = _mlp(256, inner_dim, inner_dim)
        self.time_text_embed.text_embedder = _mlp(
            pooled_projection_dim, inner_dim, inner_dim)
        self.context_embedder = torch.nn.Linear(
            joint_attention_dim, caption_projection_dim)
        self.transformer_blocks = torch.nn.ModuleList([
            _JointBlock(inner_dim, num_attention_heads, attention_head_dim,
                        i == num_layers - 1, qk_norm,
                        i in dual_attention_layers)
            for i in range(num_layers)])
        self.norm_out = ParamGroup()
        self.norm_out.linear = torch.nn.Linear(inner_dim, 2 * inner_dim)
        self.proj_out = torch.nn.Linear(
            inner_dim, patch_size * patch_size * out_channels)

        # ---- OpenDWM additions (crossview_temporal_dit.py:143-215) ----
        self.condition_image_adapter = None \
            if condition_image_adapter_config is None else \
            _adapters.ImageAdapter(**condition_image_adapter_config)
        self.perspective_modeling_type = perspective_modeling_type
        if perspective_modeling_type == "implicit":
            self.view_embedding = _mlp(
                projection_class_embeddings_input_dim, inner_dim, inner_dim)
        self.enable_crossview = enable_crossview
        self.crossview_attention_type = crossview_attention_type
        self.crossview_block_layers = crossview_block_layers
        if enable_crossview:
            n = len(crossview_block_layers)
            self.view_pos_embeds = torch.nn.ModuleList(
                [_mlp(inner_dim, inner_dim * 4, inner_dim) for _ in range(n)])
            self.crossview_transformer_blocks = torch.nn.ModuleList([
                VTSelfAttentionBlock(
                    inner_dim, inner_dim, num_attention_heads,
                    attention_head_dim, qk_norm=qk_norm_on_additional_modules)
                for _ in range(n)])
            self.view_mixers = torch.nn.ModuleList([
                AlphaBlender(merge_factor, merge_strategy=merge_strategy)
                for _ in range(n)])
        self.enable_temporal = enable_temporal
        self.temporal_attention_type = temporal_attention_type
        self.temporal_block_layers = temporal_block_layers
        if enable_temporal:
            n = len(temporal_block_layers)
            self.time_pos_embeds = torch.nn.ModuleList(
                [_mlp(inner_dim, inner_dim * 4, inner_dim) for _ in range(n)])
            self.temporal_transformer_blocks = torch.nn.ModuleList([
                VTSelfAttentionBlock(
                    inner_dim, inner_dim, num_attention_heads,
                    attention_head_dim, qk_norm=qk_norm_on_additional_modules)
                for _ in range(n)])
            self.time_mixers = torch.nn.ModuleList([
                AlphaBlender(merge_factor, merge_strategy=merge_strategy)
                for _ in range(n)])
        self.depth_net = None
        self.mask_module = None

        self._pk = None          # packed weights (16-bit; E4M3 + scales with gemm_dtype)
        self._ws = {}            # workspaces keyed by shape
        self._cond_key = None
        self._cond = None
        self.shard = None        # opendwm_b200.sharding.ShardPlan (frame-axis sharding)

    # -- nn.Module plumbing the pipeline relies on ---------------------------------
    def enable_gradient_checkpointing(self):
        self.gradient_checkpointing = True  # inference path: nothing to checkpoint

    def _apply(self, fn, *args, **kwargs):
        self._pk, self._cond_key, self._cond = None, None, None
        self._ws = {}
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, state_dict, strict: bool = True, assign=False):
        self._pk, self._cond_key, self._cond = None, None, None
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    # -- weight packing --------------------------------------------------------------
    def _dtype(self):
        if self.compute_dtype is not None:
            return self.compute_dtype
        pd = self.proj_out.weight.dtype
        return pd if pd in (torch.float16, torch.bfloat16) else torch.bfloat16

    @torch.no_grad()
    def _pack(self):
        dev = self.proj_out.weight.device
        if dev.type != "cuda":
            raise RuntimeError(
                "DiTCrossviewTemporalConditionModel runs on CUDA (sm_90a) only; "
                "there is no CPU fallback. Move the model to the GPU first.")
        dt = self._dtype()
        D = self.inner_dim
        fp8 = self.gemm_dtype is not None
        pk = {"dtype": dt, "fp8": fp8}
        # 16-bit in either precision: the embedders, the AdaLN linears and proj_out; E4M3
        # with fp8: the linears of the joint and cross-view / temporal blocks
        te = self.time_text_embed
        pk["patch"], pk["t1"], pk["t2"], pk["p1"], pk["p2"], pk["ctx"] = (
            pack_linear(m.weight, m.bias, dt, dev) for m in (
                self.pos_embed.proj, te.timestep_embedder.linear_1,
                te.timestep_embedder.linear_2, te.text_embedder.linear_1,
                te.text_embedder.linear_2, self.context_embedder))

        # all AdaLN linears act on the same SiLU(temb): one concatenated GEMM
        mod_w, mod_b, off = [], [], 0
        blocks = []
        for blk in self.transformer_blocks:
            b = {"dual": blk.dual, "last": blk.context_pre_only}
            for key, m in (("mod", blk.norm1.linear),
                           ("cmod", blk.norm1_context.linear)):
                mod_w.append(m.weight.detach())
                mod_b.append(m.bias.detach())
                b[key] = (off, m.weight.shape[0])
                off += m.weight.shape[0]
            at = blk.attn
            b["qkv"] = pack_linear(
                torch.cat([at.to_q.weight, at.to_k.weight, at.to_v.weight]),
                torch.cat([at.to_q.bias, at.to_k.bias, at.to_v.bias]), dt, dev, fp8)
            b["cqkv"] = pack_linear(
                torch.cat([at.add_q_proj.weight, at.add_k_proj.weight, at.add_v_proj.weight]),
                torch.cat([at.add_q_proj.bias, at.add_k_proj.bias, at.add_v_proj.bias]),
                dt, dev, fp8)
            b["qk_norm"] = at.qk_norm == "rms_norm"
            if b["qk_norm"]:
                b["nq"], b["nk"] = fp32(at.norm_q.weight), fp32(at.norm_k.weight)
                b["ncq"], b["nck"] = fp32(at.norm_added_q.weight), \
                    fp32(at.norm_added_k.weight)
            b["out"] = pack_linear(at.to_out[0].weight, at.to_out[0].bias, dt, dev, fp8)
            if not blk.context_pre_only:
                b["cout"], b["cff1"], b["cff2"] = (
                    pack_linear(m.weight, m.bias, dt, dev, fp8) for m in (
                        at.to_add_out, blk.ff_context.net[0].proj, blk.ff_context.net[2]))
            if blk.dual:
                a2 = blk.attn2
                b["qkv2"] = pack_linear(
                    torch.cat([a2.to_q.weight, a2.to_k.weight, a2.to_v.weight]),
                    torch.cat([a2.to_q.bias, a2.to_k.bias, a2.to_v.bias]), dt, dev, fp8)
                if b["qk_norm"]:
                    b["nq2"], b["nk2"] = fp32(a2.norm_q.weight), fp32(a2.norm_k.weight)
                b["out2"] = pack_linear(a2.to_out[0].weight, a2.to_out[0].bias, dt, dev, fp8)
            b["ff1"], b["ff2"] = (pack_linear(m.weight, m.bias, dt, dev, fp8)
                                  for m in (blk.ff.net[0].proj, blk.ff.net[2]))
            blocks.append(b)
        mod_w.append(self.norm_out.linear.weight.detach())
        mod_b.append(self.norm_out.linear.bias.detach())
        pk["final_mod"] = (off, 2 * D)
        off += 2 * D
        pk["mod"] = pack_linear(torch.cat(mod_w), torch.cat(mod_b), dt, dev)
        pk["mod_total"] = off
        pk["blocks"] = blocks
        pk["proj_out"] = pack_linear(self.proj_out.weight, self.proj_out.bias, dt, dev)
        if self.perspective_modeling_type == "implicit":
            pk["ve1"], pk["ve2"] = (pack_linear(m.weight, m.bias, dt, dev) for m in (
                self.view_embedding.linear_1, self.view_embedding.linear_2))
        if self.enable_crossview:
            pk["cv"] = [b.pack(dt, dev, fp8) for b in self.crossview_transformer_blocks]
            pk["vpe"] = [tuple(pack_linear(lin.weight, lin.bias, dt, dev)
                               for lin in (m.linear_1, m.linear_2))
                         for m in self.view_pos_embeds]
        if self.enable_temporal:
            pk["tp"] = [b.pack(dt, dev, fp8) for b in self.temporal_transformer_blocks]
            pk["tpe"] = [tuple(pack_linear(lin.weight, lin.bias, dt, dev)
                               for lin in (m.linear_1, m.linear_2))
                         for m in self.time_pos_embeds]
        # weight bytes the E4M3 copies save against 16-bit ones (scales included)
        pk["fp8_bytes_saved"] = fp8_bytes_saved(pk)
        self._pk = pk
        return pk

    # -- workspaces --------------------------------------------------------------------
    def _workspace(self, N, S, L, dev, dt):
        key = (N, S, L, dt)
        ws = self._ws.get(key)
        if ws is not None:
            return ws
        D, pk = self.inner_dim, self._pk
        p2c = self.patch_size ** 2 * self.in_channels

        def e(*shape, dtype=dt):
            return torch.empty(*shape, device=dev, dtype=dtype)

        ws = {
            "patch16": e(N * S, p2c),
            "x": e(N * S, D, dtype=torch.float32),
            "y": e(N * S, D, dtype=torch.float32),
            "c": e(N * L, D, dtype=torch.float32),
            "a16": e(N * S, D), "a16b": e(N * S, D), "ac16": e(N * L, D),
            "g16": e(N * S, 4 * D), "gc16": e(N * L, 4 * D),
            "qkv_j": e(N * (S + L), 3 * D), "qkv_s": e(N * S, 3 * D),
            "o16": e(N * S, D), "oc16": e(N * L, D),
            "tsin": e(N, 256), "th": e(N, D),
            "temb": e(N, D, dtype=torch.float32), "temb_silu": e(N, D),
            "mod": e(N, pk["mod_total"], dtype=torch.float32),
            "tokens": e(N * S, self.patch_size ** 2 * self.out_channels,
                        dtype=torch.float32),
        }
        # GEMM operands: the LayerNorm outputs (a, ab sample rows, ac context rows) and the
        # E4M3 buffers the 16-bit GEMM outputs are requantized into (q sample rows, qc
        # context rows; None in 16 bit)
        if pk["fp8"]:
            ws["a"], ws["ab"], ws["ac"], ws["q"], ws["qc"] = (
                Operand(e(rows, cols, dtype=FP8), e(rows, dtype=torch.float32))
                for rows, cols in ((N * S, D), (N * S, D), (N * L, D), (N * S, 4 * D),
                                   (N * L, 4 * D)))
        else:
            ws["a"], ws["ab"], ws["ac"] = Operand(ws["a16"]), Operand(ws["a16b"]), \
                Operand(ws["ac16"])
            ws["q"] = ws["qc"] = None
        self._ws = {key: ws}  # keep a single live workspace
        return ws

    # -- step-invariant condition cache ---------------------------------------------------
    @staticmethod
    def _tkey(t):
        return None if t is None else \
            (t.data_ptr(), tuple(t.shape), t.dtype, t._version)

    def _mlp_run(self, a16, l1, l2, resid=None):
        h = gemm(a16, l1, act=_lib.ACT_SILU)
        return gemm(h, l2, epilogue=_lib.EPI_RESID if resid is not None else _lib.EPI_F32,
                    resid=resid)

    @torch.no_grad()
    def _conditions(self, B, T, V, Hp, Wp, t_offset, T_total,
                    encoder_hidden_states, pooled_projections,
                    condition_image_tensor, added_time_ids, disable_crossview,
                    disable_temporal, crossview_attention_mask, v_offset=0, V_total=None):
        V_total = V if V_total is None else V_total
        key = (B, T, V, Hp, Wp, t_offset, T_total, v_offset, V_total,
               self._tkey(encoder_hidden_states), self._tkey(pooled_projections),
               self._tkey(condition_image_tensor), self._tkey(added_time_ids),
               self._tkey(disable_crossview), self._tkey(disable_temporal),
               self._tkey(crossview_attention_mask))
        if key == self._cond_key:
            return self._cond
        # the key holds addresses: keep the keyed tensors alive with the cache entry, so the
        # caching allocator cannot hand the same address to a different condition set
        refs = (encoder_hidden_states, pooled_projections, condition_image_tensor,
                added_time_ids, disable_crossview, disable_temporal, crossview_attention_mask)
        if self.__dict__.pop("_ring_shift", False) and self._ring_applicable(
                B, T, V, Hp, Wp, t_offset, T_total, condition_image_tensor, v_offset, V_total):
            cd = self._conditions_shifted(
                B, T, V, Hp, Wp, t_offset, T_total, encoder_hidden_states, pooled_projections,
                condition_image_tensor, added_time_ids, disable_crossview, disable_temporal,
                crossview_attention_mask, v_offset, V_total)
            self._cond_key, self._cond, self._cond_refs = key, cd, refs
            return cd
        pk, dt, D = self._pk, self._pk["dtype"], self.inner_dim
        dev = encoder_hidden_states.device
        N, S = B * T * V, Hp * Wp
        cd = {}
        ehs = encoder_hidden_states.flatten(0, 2)
        L = ehs.shape[1]
        cd["L"] = L
        cd["c0"] = gemm(ehs.reshape(N * L, -1).to(dt).contiguous(), pk["ctx"],
                        epilogue=_lib.EPI_F32)
        cd["text_emb"] = self._mlp_run(
            pooled_projections.flatten(0, 2).to(dt).contiguous(),
            pk["p1"], pk["p2"])
        cd["pos"] = self.pos_embed.cropped(Hp, Wp).to(dev)

        view_cam = None
        if self.perspective_modeling_type == "implicit":
            ids = added_time_ids.flatten().float().contiguous()
            sn = torch.empty(ids.numel(), 256, device=dev, dtype=dt)
            _ops.sinusoid(ids, 256, sn, True, 0.0)
            view_cam = self._mlp_run(sn.view(N, -1), pk["ve1"], pk["ve2"])

        def index_table(count, mlps):
            idx = torch.arange(count, device=dev, dtype=torch.float32)
            sn = torch.empty(count, D, device=dev, dtype=dt)
            _ops.sinusoid(idx, D, sn, True, 0.0)
            return [self._mlp_run(sn, l1, l2) for l1, l2 in mlps]

        item_t = (torch.arange(T, device=dev) + t_offset).view(1, T, 1)\
            .expand(B, T, V).reshape(-1)
        # a view shard holds views v_offset ... v_offset + V - 1 of V_total: its view index
        # embeddings are rows of the table over all views
        item_v = (torch.arange(V, device=dev) + v_offset).view(1, 1, V)\
            .expand(B, T, V).reshape(-1)
        cd["_geom"] = (B, T, V, Hp, Wp, t_offset, T_total, v_offset, V_total)
        cd["_view_cam"] = view_cam
        if self.enable_temporal:
            tabs = index_table(T_total, pk["tpe"])
            cd["_tabs_t"] = tabs
            cd["temb_tab"] = []
            for tab in tabs:
                e = tab[item_t]
                if self.enable_crossview and view_cam is not None and \
                        not self.disable_view_emb_on_temporal_module:
                    e = e + view_cam
                cd["temb_tab"].append(e.contiguous())
            dis = disable_temporal if disable_temporal is not None else \
                torch.zeros(B, dtype=torch.bool, device=dev)
            cd["t_alpha"] = [m.batch_alpha(B, dis.flatten().to(dev), dev)
                             for m in self.time_mixers]
        if self.enable_crossview:
            tabs = index_table(V_total, pk["vpe"])
            cd["_tabs_v"] = tabs
            cd["vemb_tab"] = []
            for tab in tabs:
                e = tab[item_v]
                if view_cam is not None:
                    e = e + view_cam
                cd["vemb_tab"].append(e.contiguous())
            dis = disable_crossview if disable_crossview is not None else \
                torch.zeros(B, dtype=torch.bool, device=dev)
            cd["v_alpha"] = [m.batch_alpha(B, dis.flatten().to(dev), dev)
                             for m in self.view_mixers]
            cd["mask"] = None if crossview_attention_mask is None else \
                crossview_attention_mask.to(device=dev).ne(0).to(torch.uint8)\
                .contiguous()
        cd["residuals"] = []
        if self.condition_image_adapter is not None and \
                condition_image_tensor is not None:
            cd["residuals"] = self.condition_image_adapter.token_features(
                condition_image_tensor.to(dev), dt)
        self._cond_key, self._cond, self._cond_refs = key, cd, refs
        return cd

    # -- streaming ring update of the step-invariant cache (opt-in, SURVEY.md §8(f)2) -----------
    def _ring_applicable(self, B, T, V, Hp, Wp, t_offset, T_total, image, v_offset, V_total):
        """T frames from t_offset of a T_total-frame window: the whole window on one GPU, or
        a frame and / or view shard (`ShardPlan`) of it."""
        old = self._cond
        return old is not None and T > 1 and \
            old.get("_geom") == (B, T, V, Hp, Wp, t_offset, T_total, v_offset, V_total) and \
            (image is None or image.shape[1] == T)

    def _conditions_shifted(self, B, T, V, Hp, Wp, t_offset, T_total, ehs, pooled, image, ids,
                            dis_cv, dis_t, mask, v_offset, V_total):
        """The FIFO moved on by one frame: every per-item entry of the cached condition set is
        the old one shifted by a frame, only the last frame's entries (context embedding, pooled
        text MLP, camera embedding, ImageAdapter residuals) are computed.  The index-embedding
        sums are re-formed because a frame's time index changes with its queue slot.

        A frame shard shifts the same way: its new last slot is window frame
        t_offset + T - 1, computed from the shard's own conditions, so no exchange is needed."""
        old = self._cond
        saved = (self._cond_key, self._cond)
        self._cond_key = None
        one = lambda t: None if t is None else t[:, T - 1:]          # noqa: E731
        cd1 = self._conditions(B, 1, V, Hp, Wp, t_offset + T - 1, T_total, one(ehs), one(pooled),
                               one(image), one(ids), dis_cv, dis_t, mask, v_offset, V_total)
        self._cond_key, self._cond = saved

        def shift(o, n):
            if o is None:
                return None
            rows = o.shape[0] // (B * T)            # rows per (batch, frame): V * rows per item
            o4 = o.view(B, T, rows, o.shape[1])
            return torch.cat([o4[:, 1:], n.view(B, 1, rows, o.shape[1])], 1)\
                .reshape(o.shape).contiguous()
        cd = dict(old)
        cd["c0"] = shift(old["c0"], cd1["c0"])
        cd["text_emb"] = shift(old["text_emb"], cd1["text_emb"])
        view_cam = cd["_view_cam"] = shift(old["_view_cam"], cd1["_view_cam"])
        dev = cd["c0"].device
        item_t = (torch.arange(T, device=dev) + t_offset).view(1, T, 1)\
            .expand(B, T, V).reshape(-1)
        item_v = (torch.arange(V, device=dev) + v_offset).view(1, 1, V).expand(B, T, V).reshape(-1)
        if self.enable_temporal:
            cd["temb_tab"] = []
            for tab in old["_tabs_t"]:
                e = tab[item_t]
                if self.enable_crossview and view_cam is not None and \
                        not self.disable_view_emb_on_temporal_module:
                    e = e + view_cam
                cd["temb_tab"].append(e.contiguous())
            cd["t_alpha"] = cd1["t_alpha"]
        if self.enable_crossview:
            cd["vemb_tab"] = []
            for tab in old["_tabs_v"]:
                e = tab[item_v]
                if view_cam is not None:
                    e = e + view_cam
                cd["vemb_tab"].append(e.contiguous())
            cd["v_alpha"] = cd1["v_alpha"]
            cd["mask"] = cd1["mask"]
        cd["residuals"] = [shift(o, n) for o, n in zip(old["residuals"], cd1["residuals"])]
        return cd

    # -- attention regroupings (crossview_temporal_dit.py:289-315, 335-361) -----------------
    def _crossview_attend(self, B, T, V, Hp, Wp, mask):
        S, D, heads = Hp * Wp, self.inner_dim, self.heads
        kind = self.crossview_attention_type
        if kind == "rowwise":      # (bt v) (h w) c -> (bt h) (v w) c
            def attend(qkv, out):
                _ops.attention(qkv, out, D=D, heads=heads,
                               group_dims=[B * T, Hp], group_strides=[V * S, Wp],
                               seq=V * Wp, inner=Wp, stride_outer=S,
                               stride_inner=1, mask=mask, mask_div=T)
        elif kind == "full":       # all tokens of the V views of one frame
            if mask is not None:
                raise NotImplementedError(
                    "crossview 'full' with a view mask is not produced by the "
                    "CTSD pipeline")

            def attend(qkv, out):
                _ops.attention(qkv, out, D=D, heads=heads, group_dims=[B * T],
                               group_strides=[V * S], seq=V * S)
        else:
            # mirrors `raise f"Not support ..."` (a TypeError) at
            # crossview_temporal_dit.py:317-318; "fuse"/"adj_fuse" need
            # crossview_attention_index which get_conditions never provides.
            raise TypeError("Not support {}".format(kind))
        return attend

    def _temporal_attend(self, B, T, V, Hp, Wp):
        S, D, heads = Hp * Wp, self.inner_dim, self.heads
        kind = self.temporal_attention_type
        if kind == "full":         # (b t v) hw c -> (b v) (t hw) c
            def attend(qkv, out):
                _ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V],
                               group_strides=[T * V * S, S], seq=T * S, inner=S,
                               stride_outer=V * S, stride_inner=1)
        elif kind == "rowwise":    # (b t v) (h w) c -> (b v h) (t w) c
            def attend(qkv, out):
                _ops.attention(qkv, out, D=D, heads=heads, group_dims=[B, V, Hp],
                               group_strides=[T * V * S, S, Wp], seq=T * Wp,
                               inner=Wp, stride_outer=V * S, stride_inner=1)
        else:                      # "pointwise": (b t v) hw c -> (b v hw) t c
            def attend(qkv, out):
                _ops.attention(qkv, out, D=D, heads=heads,
                               group_dims=[B, V * S], group_strides=[T * V * S, 1],
                               seq=T, inner=1, stride_outer=V * S, stride_inner=0)
        return attend

    def _temporal_qkv_attend_sharded(self, B, T_loc, V, Hp, Wp, ws):
        """Frame-sharded temporal attention (`sharded_temporal_qkv_attend`) with its buffers
        kept in the step workspace for the input geometry."""
        plan = self.shard
        S, D, heads = Hp * Wp, self.inner_dim, self.heads
        T = plan.T
        rows = B * T_loc * V * S
        rows_full = B * T * V * S
        dt, dev = ws["a16"].dtype, ws["a16"].device
        if ws.get("kv_geom") != (rows, rows_full):
            ws["kv_geom"] = (rows, rows_full)
            ws["q_loc"] = torch.empty(rows, D, device=dev, dtype=dt)
            ws["peer_kv"] = None
            if plan.use_peer_scatter:
                from opendwm_b200.sharding import PeerKV
                ws["peer_kv"] = PeerKV(plan, rows_full, 2 * D, dt, dev)
            else:
                ws["kv_loc"] = torch.empty(rows, 2 * D, device=dev, dtype=dt)
                ws["kv_all"] = torch.empty(rows_full, 2 * D, device=dev, dtype=dt)
        return sharded_temporal_qkv_attend(
            plan, self.temporal_attention_type, B, T_loc, V, Hp, Wp, D, heads, ws["q_loc"],
            peer_kv=ws["peer_kv"], kv_loc=ws.get("kv_loc"), kv_all=ws.get("kv_all"))

    def _crossview_qkv_attend_sharded(self, B, T, V_loc, Hp, Wp, ws, mask):
        """Row-wise cross-view attention of a view shard (`sharded_crossview_qkv_attend`): local
        query views against the K,V of all views, gathered over the view group, with its
        buffers kept in the step workspace for the input geometry."""
        plan = self.shard
        if self.crossview_attention_type != "rowwise":
            raise NotImplementedError(
                "crossview {!r} attention under a view shard: only 'rowwise' (the CTSD "
                "configs) is sharded".format(self.crossview_attention_type))
        S, D, heads = Hp * Wp, self.inner_dim, self.heads
        rows, rows_full = B * T * V_loc * S, B * T * plan.V * S
        dt, dev = ws["a16"].dtype, ws["a16"].device
        if ws.get("cv_geom") != (rows, rows_full):
            ws["cv_geom"] = (rows, rows_full)
            ws["cv_q_loc"] = torch.empty(rows, D, device=dev, dtype=dt)
            ws["cv_peer_kv"] = None
            if plan.use_peer_scatter:
                from opendwm_b200.sharding import PeerKV
                ws["cv_peer_kv"] = PeerKV(plan, rows_full, 2 * D, dt, dev, axis="v")
            else:
                ws["cv_kv_loc"] = torch.empty(rows, 2 * D, device=dev, dtype=dt)
                ws["cv_kv_all"] = torch.empty(rows_full, 2 * D, device=dev, dtype=dt)
        return sharded_crossview_qkv_attend(
            plan, B * T, Hp, Wp, D, heads, ws["cv_q_loc"], mask, T,
            peer_kv=ws["cv_peer_kv"], kv_loc=ws.get("cv_kv_loc"), kv_all=ws.get("cv_kv_all"))

    # -- one JointTransformerBlock ----------------------------------------------------------
    def _joint_block(self, b, ws, N, S, L, residual):
        D, heads = self.inner_dim, self.heads
        x, c, mod = ws["x"], ws["c"], ws["mod"]
        c_src = ws.pop("c_in", None)          # first block: context read from the cache
        c_src = c if c_src is None else c_src
        qkv, o16, oc16 = ws["qkv_j"], ws["o16"], ws["oc16"]
        a, ab, ac, q, qc = ws["a"], ws["ab"], ws["ac"], ws["q"], ws["qc"]
        o, _ = b["mod"]
        m = [mod[:, o + i * D:o + (i + 1) * D] for i in range(9 if b["dual"] else 6)]
        shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = m[:6]
        co, _ = b["cmod"]
        if b["last"]:   # AdaLayerNormContinuous: (scale, shift)
            c_scale_msa, c_shift_msa = mod[:, co:co + D], mod[:, co + D:co + 2 * D]
        else:
            cm = [mod[:, co + i * D:co + (i + 1) * D] for i in range(6)]
            c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, \
                c_gate_mlp = cm
        kw = {}
        if b["dual"]:
            kw = dict(shift2=m[6], scale2=m[7], out2=ab)
        if residual is not None:   # hidden_states += condition residual (:491-494)
            kw.update(add_full=residual, sum_out=x)
        layernorm(x, a, eps=1e-6, rows_per_item=S, shift=shift_msa, scale=scale_msa, **kw)
        layernorm(c_src, ac, eps=1e-6, rows_per_item=L, shift=c_shift_msa, scale=c_scale_msa)
        if b["qk_norm"]:
            gemm(a, b["qkv"], epilogue=_lib.EPI_QKNORM, out=qkv,
                 rows_per_item=S, out_item_stride=S + L, out_row_offset=0,
                 q_norm_weight=b["nq"], k_norm_weight=b["nk"], qk_region=D,
                 eps=1e-6)
            gemm(ac, b["cqkv"], epilogue=_lib.EPI_QKNORM, out=qkv,
                 rows_per_item=L, out_item_stride=S + L, out_row_offset=S,
                 q_norm_weight=b["ncq"], k_norm_weight=b["nck"],
                 qk_region=D, eps=1e-6)
        else:
            gemm(a, b["qkv"], out=qkv, rows_per_item=S,
                 out_item_stride=S + L, out_row_offset=0)
            gemm(ac, b["cqkv"], out=qkv, rows_per_item=L,
                 out_item_stride=S + L, out_row_offset=S)
        # joint attention over [sample ; context] tokens of each view-frame
        _ops.attention(qkv, o16, D=D, heads=heads, group_dims=[N],
                       group_strides=[S + L], seq=S + L, out_group_strides=[S],
                       out_stride_outer=0, out_stride_inner=1, split=S, out2=oc16)
        gemm(requantize(o16, q), b["out"], epilogue=_lib.EPI_RESID, resid=x, out=x,
             gate=gate_msa, rows_per_item=S)
        if b["dual"]:
            q2 = ws["qkv_s"]
            if b["qk_norm"]:
                gemm(ab, b["qkv2"], epilogue=_lib.EPI_QKNORM, out=q2,
                     q_norm_weight=b["nq2"], k_norm_weight=b["nk2"],
                     qk_region=D, eps=1e-6)
            else:
                gemm(ab, b["qkv2"], out=q2)
            _ops.attention(q2, o16, D=D, heads=heads, group_dims=[N],
                           group_strides=[S], seq=S)
            gemm(requantize(o16, q), b["out2"], epilogue=_lib.EPI_RESID, resid=x, out=x,
                 gate=m[8], rows_per_item=S)
        layernorm(x, a, eps=1e-6, rows_per_item=S, shift=shift_mlp, scale=scale_mlp)
        gemm(a, b["ff1"], act=_lib.ACT_GELU_TANH, out=ws["g16"])
        gemm(requantize(ws["g16"], q), b["ff2"], epilogue=_lib.EPI_RESID, resid=x, out=x,
             gate=gate_mlp, rows_per_item=S)
        if not b["last"]:
            gemm(requantize(oc16, qc), b["cout"], epilogue=_lib.EPI_RESID, resid=c_src,
                 out=c, gate=c_gate_msa, rows_per_item=L)
            layernorm(c, ac, eps=1e-6, rows_per_item=L, shift=c_shift_mlp, scale=c_scale_mlp)
            gemm(ac, b["cff1"], act=_lib.ACT_GELU_TANH, out=ws["gc16"])
            gemm(requantize(ws["gc16"], qc), b["cff2"], epilogue=_lib.EPI_RESID, resid=c,
                 out=c, gate=c_gate_mlp, rows_per_item=L)

    # -- forward -------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_tokens(
        self, sample, timestep, encoder_hidden_states, pooled_projections,
        condition_image_tensor=None, disable_crossview=None,
        disable_temporal=None, crossview_attention_mask=None,
        added_time_ids=None, t_offset=0, T_total=None, cfg_repeat=1, v_offset=0, V_total=None
    ):
        """Runs the noise-predict forward and returns the proj_out tokens
        fp32 [B*T*V*S, p*p*C] (column = (py*p+px)*C + c) plus the geometry; the
        fused CFG/Euler kernel and `forward` un-patchify from this.
        `cfg_repeat=2`: `sample` / `timestep` hold ONE copy of the batch and stand for
        `torch.cat([x, x])` (reference ctsd.py:2058-2063) — the patchify and timestep kernels
        write both halves, no concatenated copy is materialised.
        A frame / view shard of a ShardPlan (`self.shard`) passes the frames from t_offset of
        T_total and the views from v_offset of V_total it holds."""
        if self._pk is None:
            self._pack()
        pk = self._pk
        dt, D, P = pk["dtype"], self.inner_dim, self.patch_size
        if not sample.is_cuda:
            raise RuntimeError("DiTCrossviewTemporalConditionModel needs CUDA "
                               "tensors; there is no CPU fallback.")
        B, T, V, C, H, W = sample.shape
        B *= cfg_repeat
        Hp, Wp = H // P, W // P
        N, S = B * T * V, Hp * Wp
        T_total = T if T_total is None else T_total
        cd = self._conditions(
            B, T, V, Hp, Wp, t_offset, T_total, encoder_hidden_states,
            pooled_projections, condition_image_tensor, added_time_ids,
            disable_crossview, disable_temporal, crossview_attention_mask, v_offset, V_total)
        L = cd["L"]
        ws = self._workspace(N, S, L, sample.device, dt)

        # K1: patchify conv + cropped pos-embed
        x_in = sample.reshape(N // cfg_repeat, C, H, W)
        if x_in.dtype != torch.float32 or not x_in.is_contiguous():
            x_in = x_in.float().contiguous()
        n1 = (N // cfg_repeat) * S
        for r in range(cfg_repeat):
            _ops.patchify(x_in, P, ws["patch16"][r * n1:(r + 1) * n1])
        gemm(ws["patch16"], pk["patch"], epilogue=_lib.EPI_RESID, resid=cd["pos"],
             resid_row_mod=S, out=ws["x"])
        # K3: temb = timestep_embedder(sinusoid(t)) + text_embedder(pooled)
        t_in = timestep.flatten()
        if t_in.dtype != torch.float32 or not t_in.is_contiguous():
            t_in = t_in.float().contiguous()
        for r in range(cfg_repeat):
            _ops.sinusoid(t_in, 256, ws["tsin"][r * t_in.numel():(r + 1) * t_in.numel()],
                          True, 0.0)
        gemm(ws["tsin"], pk["t1"], act=_lib.ACT_SILU, out=ws["th"])
        gemm(ws["th"], pk["t2"], epilogue=_lib.EPI_RESID, resid=cd["text_emb"], out=ws["temb"])
        _ops.act_cast(ws["temb"], ws["temb_silu"], _lib.ACT_SILU)
        # every AdaLN modulation of the forward in one GEMM
        gemm(ws["temb_silu"], pk["mod"], epilogue=_lib.EPI_F32, out=ws["mod"])
        # the context stream starts as the (cached, read-only) embedded text: block 0 reads
        # cd["c0"] and writes ws["c"], so no per-step copy of it is made
        ws["c_in"] = cd["c0"]

        residuals = list(cd["residuals"])
        cv_attend = self._crossview_attend(B, T, V, Hp, Wp, cd.get("mask")) \
            if self.enable_crossview else None
        cv_sharded = None
        if self.enable_crossview and self.shard is not None and self.shard.v_ways > 1:
            cv_sharded = self._crossview_qkv_attend_sharded(B, T, V, Hp, Wp, ws, cd.get("mask"))
        tp_attend = self._temporal_attend(B, T, V, Hp, Wp) \
            if self.enable_temporal else None
        tp_sharded = None
        if self.enable_temporal and self.shard is not None and \
                self.shard.t_ways > 1:
            tp_sharded = self._temporal_qkv_attend_sharded(B, T, V, Hp, Wp, ws)
        trace = getattr(self, "_trace", None)     # parity diagnostics only
        for i, b in enumerate(pk["blocks"]):
            res = residuals.pop(0) if residuals else None
            self._joint_block(b, ws, N, S, L, res)
            if trace is not None:
                trace(("joint", i), ws["x"])
            if self.enable_temporal and i in self.temporal_block_layers:
                k = self.temporal_block_layers.index(i)
                self.temporal_transformer_blocks[k].run(
                    pk["tp"][k], ws["x"], cd["temb_tab"][k], S, ws, tp_attend,
                    cd["t_alpha"][k], T * V * S, qkv_attend=tp_sharded)
                if trace is not None:
                    trace(("temporal", i), ws["x"])
            if self.enable_crossview and i in self.crossview_block_layers:
                k = self.crossview_block_layers.index(i)
                self.crossview_transformer_blocks[k].run(
                    pk["cv"][k], ws["x"], cd["vemb_tab"][k], S, ws, cv_attend,
                    cd["v_alpha"][k], T * V * S, qkv_attend=cv_sharded)
                if trace is not None:
                    trace(("crossview", i), ws["x"])

        # K8: AdaLayerNormContinuous (scale, shift) + proj_out
        fo, _ = pk["final_mod"]
        _ops.layernorm(ws["x"], ws["a16"], eps=1e-6, rows_per_item=S,
                       scale=ws["mod"][:, fo:fo + D],
                       shift=ws["mod"][:, fo + D:fo + 2 * D])
        gemm(ws["a16"], pk["proj_out"], epilogue=_lib.EPI_F32, out=ws["tokens"])
        return ws["tokens"], (B, T, V, Hp, Wp)

    def forward(
        self,
        sample: torch.FloatTensor,
        timestep: torch.LongTensor = None,
        frustum_bev_residuals: torch.Tensor = None,
        encoder_hidden_states: torch.FloatTensor = None,
        pooled_projections: torch.FloatTensor = None,
        condition_image_tensor: torch.Tensor = None,
        disable_crossview: torch.BoolTensor = None,
        disable_temporal: torch.BoolTensor = None,
        crossview_attention_mask: torch.Tensor = None,
        crossview_attention_index: torch.Tensor = None,
        camera_intrinsics: torch.Tensor = None,
        camera_transforms: torch.Tensor = None,
        camera_intrinsics_norm: torch.Tensor = None,
        camera2referego: torch.Tensor = None,
        added_time_ids: torch.Tensor = None,
        noise: torch.Tensor = None,
        return_dict: bool = False
    ):
        if noise is not None:
            raise NotImplementedError(
                "`noise` drives the training-only mask module (out of scope)")
        should_add_dim = len(sample.shape) < 6
        if should_add_dim:   # crossview_temporal_dit.py:392-403
            sample = sample.unsqueeze(2)
            timestep = timestep.unsqueeze(2)
            if condition_image_tensor is not None:
                condition_image_tensor = condition_image_tensor.unsqueeze(2)
            if encoder_hidden_states is not None:
                encoder_hidden_states = encoder_hidden_states.unsqueeze(2)
            if disable_temporal is not None:
                disable_temporal = disable_temporal.unsqueeze(2)
            if pooled_projections is not None:
                pooled_projections = pooled_projections.unsqueeze(2)
            if added_time_ids is not None and added_time_ids.dim() < 4:
                added_time_ids = added_time_ids.unsqueeze(2)
        tokens, (B, T, V, Hp, Wp) = self.forward_tokens(
            sample, timestep, encoder_hidden_states, pooled_projections,
            condition_image_tensor, disable_crossview, disable_temporal,
            crossview_attention_mask, added_time_ids)
        P, C = self.patch_size, self.out_channels
        # un-patchify: pure data movement ("nhwpqc->nchpwq", :603-621)
        out = tokens.view(B * T * V, Hp, Wp, P, P, C)\
            .permute(0, 5, 1, 3, 2, 4).reshape(B, T, V, C, Hp * P, Wp * P)
        out = out.to(sample.dtype if sample.dtype.is_floating_point
                     else torch.float32)
        result = [out]
        if should_add_dim:
            out = out.squeeze(2)
        if return_dict:
            return {"noise_pred": out}
        # the reference returns the sequence length twice as filler (Appendix D)
        return result, T, T
