"""CLIP and T5-v1.1 text encoders on the sm_90a kernels.

Native counterparts of the `transformers` models the CTSD pipelines encode prompts with
(`CLIPTextModel`, `CLIPTextModelWithProjection`, `T5EncoderModel`), loaded from the same
`text_encoder*/` directories.  Each is a pre-LN transformer over a 77-token prompt: an fp32
residual stream, 16-bit GEMM operands written by the norms, and the step's kernels
(`ops.embed`, `ops.layernorm` / `ops.rmsnorm`, `packing.gemm` with fused epilogues,
`ops.attention` with CLIP's causal mask or T5's relative-position bias).

Every kernel computes a row (a token, or a prompt's attention) from that row's inputs alone, in
an order that does not depend on the batch, so a prompt's outputs are the same bits whatever it
is batched with.  The encoders therefore run each distinct id row once and scatter the results
back: a CFG streaming frame of 6 views holds at most 7 distinct prompts, not 12.

The call surface is the one `text_conditions.encode_sd3` / `encode_clip_hidden` use:
`enc(ids, output_hidden_states=True)` returns an output with `[0]` (text_embeds with a
projection, else last_hidden_state) and `.hidden_states`, of which only [-2] and [-1] are
materialised (the others are None); `.dtype` is the dtype the outputs are returned in (the
`torch_dtype` the transformers model would have been loaded with) and `.device` the GPU.
"""
import json
import math
import os

import torch

from opendwm_b200 import lib as _lib
from opendwm_b200 import ops as _ops
from dwm.models.packing import Linear, fp32, gemm, pack_linear

HEAD_DIM = 64


class EncoderOutput:
    """transformers-style output: `out[0]`, `out.last_hidden_state`, `out.hidden_states`,
    `out.text_embeds` (CLIP with projection)."""

    def __init__(self, last_hidden_state, hidden_states=None, text_embeds=None):
        self.last_hidden_state = last_hidden_state
        self.hidden_states = hidden_states
        self.text_embeds = text_embeds

    def __getitem__(self, i):
        return tuple(t for t in (self.text_embeds, self.last_hidden_state, self.hidden_states)
                     if t is not None)[i]


def _load_weights(directory):
    """State dict of a `save_pretrained` directory: model.safetensors, or the shards a
    model.safetensors.index.json names."""
    from safetensors.torch import load_file
    single = os.path.join(directory, "model.safetensors")
    index = os.path.join(directory, "model.safetensors.index.json")
    if os.path.exists(single):
        return load_file(single)
    if os.path.exists(index):
        with open(index) as f:
            shards = sorted(set(json.load(f)["weight_map"].values()))
        sd = {}
        for s in shards:
            sd.update(load_file(os.path.join(directory, s)))
        return sd
    raise NotImplementedError(
        "{} holds no model.safetensors / model.safetensors.index.json: the native text "
        "encoders load safetensors weights only".format(directory))


class _NativeEncoder:
    def __init__(self, config, device, compute_dtype, dtype):
        self.check_config(config)
        self.config = config
        self.device = torch.device(device)
        self.compute_dtype = compute_dtype
        self.dtype = dtype
        self.p = None

    @classmethod
    def from_pretrained(cls, path, subfolder=None, device="cuda", torch_dtype=None, **kw):
        """From `path[/subfolder]` (config.json + safetensors).  torch_dtype is the dtype of the
        returned states, as `transformers.from_pretrained(torch_dtype=...)` would give them."""
        d = path if subfolder is None else os.path.join(path, subfolder)
        config = cls.config_class().from_pretrained(d)
        if torch_dtype is not None:
            kw["dtype"] = torch_dtype
        enc = cls(config, device=device, **kw)
        enc.load_state_dict(_load_weights(d))
        return enc

    def __call__(self, input_ids, output_hidden_states=False, **_):
        if input_ids.dim() != 2:
            raise ValueError("input_ids must be [batch, seq]")
        ids = input_ids.detach().to("cpu", torch.int64)
        vocab = self.p["tok"].shape[0]
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= vocab):
            raise ValueError("token ids must lie in [0, {})".format(vocab))
        uniq, inv = torch.unique(ids, dim=0, return_inverse=True)
        out = self._forward(uniq, output_hidden_states)
        inv = inv.to(self.device)
        pick = lambda t: None if t is None else t.index_select(0, inv).to(self.dtype)  # noqa: E731
        hs = None
        if output_hidden_states:
            n = out["layers"] + 1
            hs = (None,) * (n - 2) + (pick(out["h_m2"]), pick(out["h_m1"]))
        return EncoderOutput(pick(out["last"]), hs, pick(out.get("text_embeds")))


def _linear(sd, name, dtype, device, bias=True):
    return pack_linear(sd[name + ".weight"], sd.get(name + ".bias") if bias else None, dtype,
                       device)


def _cat_linear(sd, names, dtype, device, bias=True):
    w = torch.cat([sd[n + ".weight"] for n in names])
    b = torch.cat([sd[n + ".bias"] for n in names]) if bias else None
    return pack_linear(w, b, dtype, device)


class NativeCLIPTextModel(_NativeEncoder):
    """transformers.CLIPTextModel (`hidden_act` "quick_gelu" or "gelu", head_dim 64): causal
    self-attention without a padding mask, as the pipeline calls it; `[0]` is the
    final-normed last_hidden_state.  The GEMM operands are compute_dtype: by default dtype
    when that is 16-bit, else fp16."""
    with_projection = False

    def __init__(self, config, device="cuda", dtype=torch.float32, compute_dtype=None):
        if compute_dtype is None:
            compute_dtype = dtype if dtype in (torch.float16, torch.bfloat16) else torch.float16
        super().__init__(config, device, compute_dtype, dtype)

    @staticmethod
    def config_class():
        import transformers
        return transformers.CLIPTextConfig

    @staticmethod
    def check_config(c):
        if c.hidden_size % c.num_attention_heads or \
                c.hidden_size // c.num_attention_heads != HEAD_DIM:
            raise NotImplementedError("native CLIP needs head_dim {}, got {} / {}".format(
                HEAD_DIM, c.hidden_size, c.num_attention_heads))
        if c.hidden_act not in ("quick_gelu", "gelu"):
            raise NotImplementedError("native CLIP supports hidden_act quick_gelu / gelu, not "
                                      "{}".format(c.hidden_act))
        if c.hidden_size > 2048 or c.intermediate_size % 32:
            raise NotImplementedError("native CLIP needs hidden_size <= 2048 and "
                                      "intermediate_size % 32 == 0")

    def load_state_dict(self, sd):
        """From a transformers CLIPTextModel(WithProjection) state dict."""
        c, dt, dev, pre = self.config, self.compute_dtype, self.device, "text_model."
        e = pre + "embeddings."
        p = {"tok": fp32(sd[e + "token_embedding.weight"].to(dev)),
             "pos": fp32(sd[e + "position_embedding.weight"].to(dev)), "layers": []}
        norm = lambda n: (fp32(sd[n + ".weight"].to(dev)), fp32(sd[n + ".bias"].to(dev)))  # noqa
        for i in range(c.num_hidden_layers):
            L = pre + "encoder.layers.{}.".format(i)
            a = L + "self_attn."
            p["layers"].append({
                "ln1": norm(L + "layer_norm1"), "ln2": norm(L + "layer_norm2"),
                "qkv": _cat_linear(sd, [a + "q_proj", a + "k_proj", a + "v_proj"], dt, dev),
                "out": _linear(sd, a + "out_proj", dt, dev),
                "fc1": _linear(sd, L + "mlp.fc1", dt, dev),
                "fc2": _linear(sd, L + "mlp.fc2", dt, dev)})
        p["final"] = norm(pre + "final_layer_norm")
        if self.with_projection:
            p["proj"] = _linear(sd, "text_projection", dt, dev, bias=False)
        self.p = p
        return self

    def _eos_positions(self, ids):
        """transformers' pooling row: argmax(ids) for the legacy eos_token_id 2, else the first
        eos_token_id."""
        if self.config.eos_token_id == 2:
            return ids.to(torch.int).argmax(-1)
        return (ids.to(torch.int) == self.config.eos_token_id).int().argmax(-1)

    def _forward(self, ids, hidden):
        c, p, dt = self.config, self.p, self.compute_dtype
        n, S = ids.shape
        if S > p["pos"].shape[0]:
            raise ValueError("{} tokens > max_position_embeddings {}".format(S, p["pos"].shape[0]))
        D, M, L = c.hidden_size, n * S, len(p["layers"])
        dev = self.device
        x = torch.empty(M, D, device=dev)
        _ops.embed(ids.reshape(-1).to(dev), p["tok"], x, pos=p["pos"], seq=S)
        a16 = torch.empty(M, D, device=dev, dtype=dt)
        o16 = torch.empty(M, D, device=dev, dtype=dt)
        act = _lib.ACT_QUICK_GELU if c.hidden_act == "quick_gelu" else _lib.ACT_GELU_ERF
        res = {"layers": L, "h_m2": None, "h_m1": None}
        for i, b in enumerate(p["layers"]):
            if hidden and i == L - 1:
                res["h_m2"] = x.clone()
            _ops.layernorm(x, a16, weight=b["ln1"][0], bias=b["ln1"][1], eps=c.layer_norm_eps)
            qkv = gemm(a16, b["qkv"])
            _ops.attention(qkv, o16, D=D, heads=c.num_attention_heads, group_dims=[n],
                           group_strides=[S], seq=S, scale=HEAD_DIM ** -0.5, causal=True)
            gemm(o16, b["out"], epilogue=_lib.EPI_RESID, resid=x, out=x)
            _ops.layernorm(x, a16, weight=b["ln2"][0], bias=b["ln2"][1], eps=c.layer_norm_eps)
            gemm(gemm(a16, b["fc1"], act=act), b["fc2"], epilogue=_lib.EPI_RESID, resid=x, out=x)
        if hidden:
            res["h_m1"] = x
        last = _ops.layernorm(x, torch.empty(M, D, device=dev, dtype=dt),
                              weight=p["final"][0], bias=p["final"][1], eps=c.layer_norm_eps)
        res["last"] = last.view(n, S, D)
        if hidden:
            res["h_m2"], res["h_m1"] = res["h_m2"].view(n, S, D), res["h_m1"].view(n, S, D)
        if "proj" in p:
            rows = torch.arange(n) * S + self._eos_positions(ids)
            pooled = last.index_select(0, rows.to(dev))
            res["text_embeds"] = gemm(pooled, p["proj"], epilogue=_lib.EPI_F32)
        return res


class NativeCLIPTextModelWithProjection(NativeCLIPTextModel):
    """transformers.CLIPTextModelWithProjection: `[0]` is text_embeds, the projection of the
    final-normed EOS row."""
    with_projection = True


def relative_position_buckets(seq, num_buckets=32, max_distance=128):
    """int64 [seq, seq] bucket of key j for query i, by transformers'
    T5Attention._relative_position_bucket (bidirectional, float32 log), on the CPU."""
    ctx = torch.arange(seq, dtype=torch.long)[:, None]
    rel = torch.arange(seq, dtype=torch.long)[None, :] - ctx
    num_buckets //= 2
    buckets = (rel > 0).to(torch.long) * num_buckets
    rel = torch.abs(rel)
    max_exact = num_buckets // 2
    is_small = rel < max_exact
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, rel, large)


class NativeT5EncoderModel(_NativeEncoder):
    """transformers.T5EncoderModel for T5 v1.1 (feed_forward_proj "gated-gelu", d_kv 64):
    unscaled scores plus the relative-position bias of block 0, shared by every block; RMSNorms
    (T5LayerNorm) before each sub-layer and at the end; `[0]` is last_hidden_state.

    The GEMM operands are bf16 whatever the pipeline dtype: T5 v1.1's activations overflow
    fp16 (transformers keeps `wo` in fp32 for that reason).  The residual stream and the
    returned states are computed in fp32."""

    def __init__(self, config, device="cuda", dtype=torch.float32, compute_dtype=torch.bfloat16):
        if compute_dtype != torch.bfloat16:
            raise NotImplementedError("native T5 runs bf16 operands (fp16 overflows)")
        super().__init__(config, device, torch.bfloat16, dtype)
        self._bias = {}

    @staticmethod
    def config_class():
        import transformers
        return transformers.T5Config

    @staticmethod
    def check_config(c):
        if c.d_kv != HEAD_DIM:
            raise NotImplementedError("native T5 needs d_kv {}, got {}".format(HEAD_DIM, c.d_kv))
        if c.feed_forward_proj != "gated-gelu":
            raise NotImplementedError("native T5 supports feed_forward_proj gated-gelu (T5 v1.1), "
                                      "not {}".format(c.feed_forward_proj))
        if c.d_ff % 128 or c.d_model % 4:
            raise NotImplementedError("native T5 needs d_ff % 128 == 0 and d_model % 4 == 0")

    def load_state_dict(self, sd):
        """From a transformers T5EncoderModel state dict."""
        c, dt, dev = self.config, self.compute_dtype, self.device
        tok = sd.get("shared.weight", sd.get("encoder.embed_tokens.weight"))
        p = {"tok": fp32(tok.to(dev)), "layers": []}
        for i in range(c.num_layers):
            B = "encoder.block.{}.layer.".format(i)
            a, f = B + "0.SelfAttention.", B + "1.DenseReluDense."
            wi = torch.cat([sd[f + "wi_1.weight"], sd[f + "wi_0.weight"]]).to(dev)
            p["layers"].append({
                "ln0": fp32(sd[B + "0.layer_norm.weight"].to(dev)),
                "ln1": fp32(sd[B + "1.layer_norm.weight"].to(dev)),
                "qkv": _cat_linear(sd, [a + "q", a + "k", a + "v"], dt, dev, bias=False),
                "o": _linear(sd, a + "o", dt, dev, bias=False),
                "wi": Linear(_ops.pack_geglu(wi)[0].to(dt).contiguous()),
                "wo": _linear(sd, f + "wo", dt, dev, bias=False)})
        p["rel"] = fp32(sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]
                        .to(dev))
        p["final"] = fp32(sd["encoder.final_layer_norm.weight"].to(dev))
        self.p, self._bias = p, {}
        return self

    def position_bias(self, seq):
        """fp32 [heads, seq, seq]: relative_attention_bias gathered by the bucket table, once per
        sequence length."""
        if seq not in self._bias:
            c = self.config
            idx = relative_position_buckets(seq, c.relative_attention_num_buckets,
                                            c.relative_attention_max_distance).to(self.device)
            self._bias[seq] = self.p["rel"][idx].permute(2, 0, 1).contiguous()
        return self._bias[seq]

    def _forward(self, ids, hidden):
        c, p, dt = self.config, self.p, self.compute_dtype
        n, S = ids.shape
        D, M, L, dev = c.d_model, n * S, len(p["layers"]), self.device
        inner = c.num_heads * HEAD_DIM
        x = torch.empty(M, D, device=dev)
        _ops.embed(ids.reshape(-1).to(dev), p["tok"], x)
        bias = self.position_bias(S)
        a16 = torch.empty(M, D, device=dev, dtype=dt)
        o16 = torch.empty(M, inner, device=dev, dtype=dt)
        res = {"layers": L, "h_m2": None}
        for i, b in enumerate(p["layers"]):
            if hidden and i == L - 1:
                res["h_m2"] = x.clone().view(n, S, D)
            _ops.rmsnorm(x, b["ln0"], a16, eps=c.layer_norm_epsilon)
            qkv = gemm(a16, b["qkv"])
            _ops.attention(qkv, o16, D=inner, heads=c.num_heads, group_dims=[n],
                           group_strides=[S], seq=S, scale=1.0, bias=bias)
            gemm(o16, b["o"], epilogue=_lib.EPI_RESID, resid=x, out=x)
            _ops.rmsnorm(x, b["ln1"], a16, eps=c.layer_norm_epsilon)
            g16 = gemm(a16, b["wi"], epilogue=_lib.EPI_GEGLU_TANH)
            gemm(g16, b["wo"], epilogue=_lib.EPI_RESID, resid=x, out=x)
        last = _ops.rmsnorm(x, p["final"], torch.empty(M, D, device=dev),
                            eps=c.layer_norm_epsilon).view(n, S, D)
        res["last"] = last
        res["h_m1"] = last          # transformers' T5 hidden_states[-1] is the final-normed state
        return res
