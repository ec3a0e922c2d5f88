"""The native text encoders against transformers on the same weights, and the pipeline on them.

Accuracy: transformers in fp32 is the reference; the bound is 1.5 x the noise floor this file
measures, transformers itself in the same 16-bit dtype against fp32 (fp16 for CLIP, bf16 for
T5, whose activations overflow fp16), with the metric max|y - y_ref| / max|y_ref|.  Checked:
hidden_states[-2] and the pooled text_embeds of CLIP-L / CLIP-G, T5's last_hidden_state and the
SD-2.1 CLIP's last_hidden_state, at tiny head_dim-64 widths and with 2 layers at the real
widths.  Batch invariance: a prompt's outputs are the same bits alone, in a batch of 12 and in
a batch of 192 with repeats."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

VOCAB = 1000
EOS, BOS = VOCAB - 1, VOCAB - 2

# name -> (kind, hidden, heads, ff, act / None, projection)
CONFIGS = {
    "clip_l_tiny": ("clip_proj", 128, 2, 256, "quick_gelu", 64),
    "clip_g_tiny": ("clip_proj", 192, 3, 384, "gelu", 64),
    "sd21_tiny": ("clip", 128, 2, 256, "gelu", None),
    "t5_tiny": ("t5", 128, 2, 256, None, None),
    "clip_l": ("clip_proj", 768, 12, 3072, "quick_gelu", 768),
    "clip_g": ("clip_proj", 1280, 20, 5120, "gelu", 1280),
    "sd21": ("clip", 1024, 16, 4096, "gelu", None),
    "t5_xxl": ("t5", 4096, 64, 10240, None, None),
}


def build_pair(name, layers=2, seed=0):
    """(transformers fp32 model on cuda, native model on the same weights)."""
    import transformers
    from dwm.models import text_encoders as te
    kind, d, h, ff, act, proj = CONFIGS[name]
    torch.manual_seed(seed)
    if kind == "t5":
        cfg = transformers.T5Config(vocab_size=VOCAB, d_model=d, d_kv=64, d_ff=ff,
                                    num_layers=layers, num_heads=h,
                                    feed_forward_proj="gated-gelu")
        with torch.device("cuda"):
            ref = transformers.T5EncoderModel(cfg).eval()
        nat = te.NativeT5EncoderModel(cfg)
    else:
        cfg = transformers.CLIPTextConfig(
            vocab_size=VOCAB, hidden_size=d, intermediate_size=ff, projection_dim=proj or d,
            num_hidden_layers=layers, num_attention_heads=h, max_position_embeddings=77,
            hidden_act=act, bos_token_id=BOS, eos_token_id=EOS, pad_token_id=EOS)
        cls = transformers.CLIPTextModelWithProjection if kind == "clip_proj" \
            else transformers.CLIPTextModel
        ncls = te.NativeCLIPTextModelWithProjection if kind == "clip_proj" \
            else te.NativeCLIPTextModel
        with torch.device("cuda"):
            ref = cls(cfg).eval()
        nat = ncls(cfg)
    nat.load_state_dict(ref.state_dict())
    return ref, nat


def prompt_ids(n, seed=0, seq=77):
    """n token rows shaped like tokenizer output: BOS, words, EOS, EOS padding."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((n, seq), EOS, dtype=torch.long)
    for i in range(n):
        L = int(torch.randint(1, seq - 1, (1,), generator=g))
        ids[i, 0] = BOS
        ids[i, 1:L] = torch.randint(0, BOS, (L - 1,), generator=g)
    return ids.cuda()


def outputs(kind, out):
    """The states the pipeline reads, by encoder kind."""
    if kind == "clip_proj":
        return {"hidden_states[-2]": out.hidden_states[-2], "text_embeds": out[0]}
    return {"last_hidden_state": out[0]}


def rel(y, ref):
    return ((y.double() - ref.double()).abs().max() / ref.double().abs().max()).item()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_native_encoder_matches_transformers(name):
    kind = CONFIGS[name][0]
    ref, nat = build_pair(name)
    ids = prompt_ids(6, seed=len(name))
    with torch.no_grad():
        want = outputs(kind, ref(ids, output_hidden_states=True))
        half = copy.deepcopy(ref).to(torch.bfloat16 if kind == "t5" else torch.float16)
        floor = outputs(kind, half(ids, output_hidden_states=True))
        del half
    got = outputs(kind, nat(ids, output_hidden_states=True))
    for k in want:
        assert got[k].shape == want[k].shape and got[k].dtype == torch.float32
        noise = rel(floor[k], want[k])
        err = rel(got[k], want[k])
        print("{} {}: native {:.3g}, transformers 16-bit {:.3g}".format(name, k, err, noise))
        assert err <= 1.5 * noise, (name, k, err, noise)


@pytest.mark.parametrize("name", ["clip_l", "clip_g", "sd21", "t5_xxl"])
def test_batch_invariance(name):
    """A prompt's states are bit-identical alone, in 12 distinct prompts and in 192 rows with
    repeats; the kernels also run the 12 distinct prompts as one batch without the
    deduplication."""
    kind = CONFIGS[name][0]
    _, nat = build_pair(name, layers=2, seed=1)
    ids12 = prompt_ids(12, seed=7)
    ids192 = ids12[torch.randint(0, 12, (192,), generator=torch.Generator().manual_seed(1))]
    ids192[0] = ids12[3]
    alone = outputs(kind, nat(ids12[3:4], output_hidden_states=True))
    in12 = outputs(kind, nat(ids12, output_hidden_states=True))
    in192 = outputs(kind, nat(ids192, output_hidden_states=True))
    raw = nat._forward(ids12.cpu(), True)     # 12 distinct rows in one launch sequence
    for k in alone:
        assert torch.equal(alone[k][0], in12[k][3]), k
        assert torch.equal(alone[k][0], in192[k][0]), k
        for j in range(192):
            assert torch.equal(in192[k][j], in12[k][int((ids12 == ids192[j]).all(1).nonzero())])
    raw_k = {"hidden_states[-2]": raw["h_m2"], "text_embeds": raw.get("text_embeds"),
             "last_hidden_state": raw["last"]}
    for k in alone:
        assert torch.equal(alone[k][0], raw_k[k][3].float()), k


T5_TINY_D = 384     # >= CLIP-L + CLIP-G widths (128 + 192): the CLIP states are padded to it


def _save_tiny_sd3(root):
    """A checkpoint directory with tiny head_dim-64 CLIP-L / CLIP-G / T5 (SD-3.5 layout) and an
    SD-2.1 CLIP under sd21/; the CLIP byte tokenizer stands in for every tokenizer."""
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
                vocab_size=n, d_model=T5_TINY_D, d_kv=64, d_ff=256, num_layers=2, num_heads=2,
                feed_forward_proj="gated-gelu")).eval()]
    for i, e in enumerate(encs):
        e.save_pretrained(os.path.join(root, "text_encoder" + ("_%d" % (i + 1) if i else "")))
    for sub in ("tokenizer", "tokenizer_2", "tokenizer_3"):
        tok.save_pretrained(os.path.join(root, sub))
    sd21 = os.path.join(root, "sd21")
    tok.save_pretrained(os.path.join(sd21, "tokenizer"))
    transformers.CLIPTextModel(cfg(128, "gelu")).eval().save_pretrained(
        os.path.join(sd21, "text_encoder"))
    return tok


@pytest.fixture
def t5_tok_is_clip(monkeypatch):
    """tokenizer_3 is a saved CLIP tokenizer here (no sentencepiece model offline)."""
    import transformers
    monkeypatch.setattr(transformers.T5TokenizerFast, "from_pretrained",
                        classmethod(lambda cls, p, subfolder=None, **k:
                                    transformers.CLIPTokenizer.from_pretrained(p, subfolder=subfolder)))


@pytest.mark.parametrize("case", ["dit_flat_cfg", "dit_nested_masked_cfg", "unet_nested"])
def test_get_conditions_native_vs_transformers(tmp_path, t5_tok_is_clip, case):
    """text_conditions (the text branch of get_conditions: nested prompts, CFG "" copies,
    condition masks; SD-3 and SD-2.1 layouts) on the native encoders, within 1.5 x the noise
    floor of transformers' 16-bit conditions."""
    from common import TEXT_CASES
    from dwm.pipelines.text_conditions import load_text_encoders, text_conditions
    is_dit, prompts, mask, cfg, _ = TEXT_CASES[case]
    root = str(tmp_path)
    _save_tiny_sd3(root)
    path = root if is_dit else os.path.join(root, "sd21")
    dev = torch.device("cuda")
    ref_encs, toks = load_text_encoders(is_dit, path, dev, {})
    nat_encs, _ = load_text_encoders(is_dit, path, dev, {}, native=True)

    def run(encs):
        with torch.no_grad():
            return text_conditions(is_dit, encs, toks, prompts, 4, 3, dev, torch.float32, mask,
                                   cfg)
    want = run(ref_encs)
    if is_dit:
        half = [copy.deepcopy(e).to(dt) for e, dt in
                zip(ref_encs, (torch.float16, torch.float16, torch.bfloat16))]
    else:
        half = copy.deepcopy(ref_encs).to(torch.float16)
    floor = run(half)
    got = run(nat_encs)
    for i in range(2 if is_dit else 1):
        assert got[i].shape == want[i].shape
        err, noise = rel(got[i], want[i]), rel(floor[i], want[i])
        print(case, i, err, noise)
        assert err <= 1.5 * noise, (case, i, err, noise)
    if not is_dit:
        assert got[1] is None


@pytest.mark.parametrize("interval", [1, 2])
def test_streaming_loop_on_native_encoders(tmp_path, t5_tok_is_clip, interval):
    """The streaming loop encodes each frame's prompts (every `text_prompt_interval`-th frame)
    on the native encoders that the constructor loads for native_text_encoders."""
    from common import CONDITION_COMMON, TINY, condition_batch
    from dwm.functional import take_sequence_clip
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    from dwm.models import text_encoders as te
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    root = str(tmp_path)
    _save_tiny_sd3(root)
    tiny = dict(TINY, joint_attention_dim=T5_TINY_D, pooled_projection_dim=128)
    torch.manual_seed(0)
    m = DiTCrossviewTemporalConditionModel(**tiny, compute_dtype=torch.float16).cuda()
    T, V, n = 4, 3, 6
    common = dict(CONDITION_COMMON, added_time_ids="fps_camera_transforms_action",
                  camera_ego_sensor_indices=[1, 2, 3], native_text_encoders=True)
    inf = {"guidance_scale": 2.0, "inference_steps": 3 * T, "sequence_length_per_iteration": T,
           "text_prompt_interval": interval,
           "autoregression_data_exception_for_take_sequence": ["crossview_mask"],
           "autoregression_condition_exception_for_take_sequence": [
               "disable_crossview", "disable_temporal", "crossview_attention_mask",
               "camera_intrinsics_norm", "camera2referego"]}
    pipe = StreamingCrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {}, inf,
                                        root, m, model_dtype=torch.float16)
    assert [type(e) for e in pipe.text_encoders] == [
        te.NativeCLIPTextModelWithProjection, te.NativeCLIPTextModelWithProjection,
        te.NativeT5EncoderModel]
    calls = []
    for e in pipe.text_encoders:
        fwd = e._forward
        e._forward = lambda ids, h, fwd=fwd: calls.append(ids.shape[0]) or fwd(ids, h)
    batch = condition_batch(T=n, V=V, hw=(64, 96), text_dim=T5_TINY_D, pooled_dim=128)
    del batch["text_embeddings"], batch["pooled_text_embeddings"]
    pipe.reset_streaming((1, T, V, 16, 8, 12), "pt")
    for i in range(n):
        f = {k: v if k == "crossview_mask" else take_sequence_clip(v, i, i + 1)
             for k, v in batch.items()}
        f["clip_text"] = [[["front %d" % i, "left %d" % i, "right"]]]
        pipe.send_frame_condition(f)
        ehs = pipe.conditions["encoder_hidden_states"]
        assert torch.isfinite(ehs).all()
        # CFG: the "" prompt plus this frame's distinct prompts, once per encoder
        if i % interval == 0:
            assert calls[-3:] == [4, 4, 4], calls
        elif interval > 1:
            assert torch.equal(ehs[:, -1], ehs[:, -2])
    assert len(calls) == 3 * len(range(0, n, interval))
    assert pipe.latents is not None and torch.isfinite(pipe.latents).all()
