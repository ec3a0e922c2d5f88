"""The native text encoders (dwm.models.text_encoders) without a GPU: config refusals, loading
tiny head_dim-64 CLIP-L / CLIP-G / SD-2.1 CLIP / T5 from `save_pretrained` directories (T5 also
from a sharded safetensors index) onto the CPU with weights equal to the source, T5's bucket
table against transformers', and `load_text_encoders(native=...)` routing.  (The pipeline
constructor's `native_text_encoders` key is exercised on the GPU, where the pipeline runs.)"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

CPU = torch.device("cpu")


def clip_config(hidden=128, heads=2, act="quick_gelu", proj=64, layers=2, eos=2):
    import transformers
    return transformers.CLIPTextConfig(
        vocab_size=300, hidden_size=hidden, intermediate_size=2 * hidden, projection_dim=proj,
        num_hidden_layers=layers, num_attention_heads=heads, max_position_embeddings=77,
        hidden_act=act, bos_token_id=298, eos_token_id=eos, pad_token_id=eos)


def t5_config(d_kv=64, ff="gated-gelu", layers=2):
    import transformers
    return transformers.T5Config(vocab_size=300, d_model=128, d_kv=d_kv, d_ff=256,
                                 num_layers=layers, num_heads=2, feed_forward_proj=ff)


def test_config_refusals():
    from dwm.models import text_encoders as te
    with pytest.raises(NotImplementedError, match="head_dim"):
        te.NativeCLIPTextModel(clip_config(hidden=96, heads=2), device=CPU)
    with pytest.raises(NotImplementedError, match="hidden_act"):
        te.NativeCLIPTextModel(clip_config(act="relu"), device=CPU)
    with pytest.raises(NotImplementedError, match="d_kv"):
        te.NativeT5EncoderModel(t5_config(d_kv=32), device=CPU)
    with pytest.raises(NotImplementedError, match="feed_forward_proj"):
        te.NativeT5EncoderModel(t5_config(ff="relu"), device=CPU)
    with pytest.raises(NotImplementedError, match="bf16"):
        te.NativeT5EncoderModel(t5_config(), device=CPU, compute_dtype=torch.float16)
    for act in ("quick_gelu", "gelu"):
        te.NativeCLIPTextModelWithProjection(clip_config(act=act), device=CPU)
    te.NativeT5EncoderModel(t5_config(), device=CPU)


def test_non_safetensors_weights_are_refused(tmp_path):
    import transformers
    from dwm.models import text_encoders as te
    torch.manual_seed(0)
    m = transformers.CLIPTextModel(clip_config())
    m.config.save_pretrained(str(tmp_path))
    torch.save(m.state_dict(), str(tmp_path / "pytorch_model.bin"))
    with pytest.raises(NotImplementedError, match="safetensors"):
        te.NativeCLIPTextModel.from_pretrained(str(tmp_path), device=CPU)


def _check_clip(nat, ref, with_proj, compute_dtype):
    sd = ref.state_dict()
    p = nat.p
    assert torch.equal(p["tok"], sd["text_model.embeddings.token_embedding.weight"].float())
    assert torch.equal(p["pos"], sd["text_model.embeddings.position_embedding.weight"].float())
    for i, b in enumerate(p["layers"]):
        a = "text_model.encoder.layers.{}.self_attn.".format(i)
        qkv = torch.cat([sd[a + n + "_proj.weight"] for n in "qkv"])
        assert b["qkv"].w.dtype == compute_dtype
        assert torch.equal(b["qkv"].w, qkv.to(compute_dtype))
        assert torch.equal(b["qkv"].b, torch.cat([sd[a + n + "_proj.bias"] for n in "qkv"]).float())
        f = "text_model.encoder.layers.{}.mlp.".format(i)
        assert torch.equal(b["fc2"].w, sd[f + "fc2.weight"].to(compute_dtype))
    assert ("proj" in p) == with_proj
    if with_proj:
        assert torch.equal(p["proj"].w, sd["text_projection.weight"].to(compute_dtype))
        assert p["proj"].b is None


def _check_t5(nat, ref):
    from opendwm_b200 import ops
    sd = ref.state_dict()
    p = nat.p
    assert torch.equal(p["tok"], sd["shared.weight"].float())
    for i, b in enumerate(p["layers"]):
        f = "encoder.block.{}.layer.1.DenseReluDense.".format(i)
        wi = ops.pack_geglu(torch.cat([sd[f + "wi_1.weight"], sd[f + "wi_0.weight"]]))[0]
        assert torch.equal(b["wi"].w, wi.to(torch.bfloat16))
        # packed blocks: [128 value rows (wi_1) | 128 gate rows (wi_0)]
        assert torch.equal(b["wi"].w[:128], sd[f + "wi_1.weight"][:128].to(torch.bfloat16))
        assert torch.equal(b["wi"].w[128:256], sd[f + "wi_0.weight"][:128].to(torch.bfloat16))
        assert torch.equal(b["ln1"], sd["encoder.block.{}.layer.1.layer_norm.weight".format(i)])
    assert torch.equal(p["rel"], sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])
    assert torch.equal(p["final"], sd["encoder.final_layer_norm.weight"])


@pytest.mark.parametrize("kind", ["clip_l", "clip_g", "sd21", "t5", "t5_sharded"])
def test_load_from_save_pretrained(tmp_path, kind):
    import transformers
    from dwm.models import text_encoders as te
    torch.manual_seed(5)
    d = str(tmp_path / kind)
    if kind.startswith("t5"):
        ref = transformers.T5EncoderModel(t5_config()).eval()
        ref.save_pretrained(d, max_shard_size="200KB" if kind == "t5_sharded" else "5GB")
        assert os.path.exists(os.path.join(d, "model.safetensors.index.json")) == \
            (kind == "t5_sharded")
        nat = te.NativeT5EncoderModel.from_pretrained(d, device=CPU)
        _check_t5(nat, ref)
        # also from the in-memory state dict
        _check_t5(te.NativeT5EncoderModel(ref.config, device=CPU).load_state_dict(ref.state_dict()), ref)
        return
    cls, ncls = {"clip_l": (transformers.CLIPTextModelWithProjection,
                            te.NativeCLIPTextModelWithProjection),
                 "clip_g": (transformers.CLIPTextModelWithProjection,
                            te.NativeCLIPTextModelWithProjection),
                 "sd21": (transformers.CLIPTextModel, te.NativeCLIPTextModel)}[kind]
    act = "quick_gelu" if kind == "clip_l" else "gelu"
    ref = cls(clip_config(act=act, hidden=128 if kind != "clip_g" else 192,
                          heads=2 if kind != "clip_g" else 3)).eval()
    ref.save_pretrained(d)
    nat = ncls.from_pretrained(d, device=CPU, torch_dtype=torch.float16)
    assert nat.dtype == torch.float16 and nat.compute_dtype == torch.float16
    _check_clip(nat, ref, kind != "sd21", torch.float16)
    nat = ncls(ref.config, device=CPU).load_state_dict(ref.state_dict())
    assert nat.dtype == torch.float32 and nat.compute_dtype == torch.float16
    _check_clip(nat, ref, kind != "sd21", torch.float16)


def test_bucket_table_matches_transformers():
    from transformers.models.t5.modeling_t5 import T5Attention
    from dwm.models.text_encoders import relative_position_buckets
    for seq in range(1, 301):
        ctx = torch.arange(seq, dtype=torch.long)[:, None]
        mem = torch.arange(seq, dtype=torch.long)[None, :]
        want = T5Attention._relative_position_bucket(mem - ctx, bidirectional=True,
                                                     num_buckets=32, max_distance=128)
        got = relative_position_buckets(seq, 32, 128)
        assert got.dtype == want.dtype and torch.equal(got, want), seq


def test_eos_rule():
    from dwm.models import text_encoders as te
    ids = torch.tensor([[298, 5, 7, 2, 2, 2], [298, 9, 299, 4, 299, 299]])
    legacy = te.NativeCLIPTextModel(clip_config(eos=2), device=CPU)
    assert legacy._eos_positions(ids).tolist() == [0, 2]          # argmax(ids)
    new = te.NativeCLIPTextModel(clip_config(eos=299), device=CPU)
    assert new._eos_positions(ids).tolist() == [0, 2]             # first eos_token_id
    ids2 = torch.tensor([[298, 5, 299, 3, 299]])
    assert new._eos_positions(ids2).tolist() == [2]
    assert legacy._eos_positions(ids2).tolist() == [2]


def _save_sd3_dir(root):
    """tokenizer*/ and text_encoder*/ of a tiny head_dim-64 SD-3.5 checkpoint (the CLIP byte
    tokenizer stands in for all three tokenizers)."""
    import transformers
    from common import tiny_text_stack
    tok = tiny_text_stack()[0]
    n = len(tok)
    cfg = lambda h, act: transformers.CLIPTextConfig(  # noqa: E731
        vocab_size=n, hidden_size=h, intermediate_size=2 * h, projection_dim=64,
        num_hidden_layers=2, num_attention_heads=h // 64, max_position_embeddings=77,
        hidden_act=act, bos_token_id=n - 2, eos_token_id=n - 1, pad_token_id=n - 1)
    torch.manual_seed(11)
    encs = [transformers.CLIPTextModelWithProjection(cfg(128, "quick_gelu")).eval(),
            transformers.CLIPTextModelWithProjection(cfg(192, "gelu")).eval(),
            transformers.T5EncoderModel(transformers.T5Config(
                vocab_size=n, d_model=128, d_kv=64, d_ff=256, num_layers=2, num_heads=2,
                feed_forward_proj="gated-gelu")).eval()]
    for i, e in enumerate(encs):
        e.save_pretrained(os.path.join(root, "text_encoder" + ("_%d" % (i + 1) if i else "")))
    for sub in ("tokenizer", "tokenizer_2"):
        tok.save_pretrained(os.path.join(root, sub))
    return tok, encs


def test_native_routing(tmp_path, monkeypatch):
    import transformers
    from dwm.models import text_encoders as te
    from dwm.pipelines import text_conditions as tc
    root = str(tmp_path)
    tok, encs = _save_sd3_dir(root)
    # tokenizer_3 is read by T5TokenizerFast; stand in with the CLIP tokenizer
    monkeypatch.setattr(transformers.T5TokenizerFast, "from_pretrained",
                        classmethod(lambda cls, *a, **k: tok))
    l_encs, l_toks = tc.load_text_encoders(True, root, CPU, {"torch_dtype": torch.float16},
                                           native=True)
    assert [type(e) for e in l_encs] == [te.NativeCLIPTextModelWithProjection,
                                         te.NativeCLIPTextModelWithProjection,
                                         te.NativeT5EncoderModel]
    assert all(e.dtype == torch.float16 for e in l_encs) and len(l_toks) == 3
    ref_encs, _ = tc.load_text_encoders(True, root, CPU, {}, native=False)
    assert [type(e).__name__ for e in ref_encs] == [
        "CLIPTextModelWithProjection", "CLIPTextModelWithProjection", "T5EncoderModel"]
    enc21, _ = tc.load_text_encoders(False, root, CPU, {}, native=True)
    assert type(enc21) is te.NativeCLIPTextModel

