"""Text encoding on the transformers encoders vs the native ones (dwm.models.text_encoders), in
one process, at the published widths with seeded random weights.

Arms, on the same weights:
  * transformers: CLIPTextModelWithProjection (CLIP-L, CLIP-G), T5EncoderModel (T5-v1.1-XXL) and
    CLIPTextModel (the SD-2.1 OpenCLIP-H), in fp16 as `load_text_encoders` loads them with
    torch_dtype=fp16, T5's `wo` kept in fp32 as `from_pretrained` keeps it
    (T5EncoderModel._keep_in_fp32_modules);
  * native: the same state dicts loaded into the native encoders (CLIP fp16 operands, T5 bf16),
    which encode each distinct prompt once.
Workloads (77 tokens per prompt; ids pre-built):
  * frame:  one north-star streaming frame, 6 views + 6 CFG "" copies (12 prompts, 7 distinct);
  * window: a 16-frame x 6-view window with CFG (192 prompts; 96 distinct view-frame prompts
    plus "");
  * sd21:   config 2's SD-2.1 encode, 12 prompts (6 views + CFG "").
Each round times every arm once per workload with CUDA events (encoders on pre-built ids, then
the whole `text_conditions` call with the tokenizer), alternating the arms; the medians and the
round-to-round spread (max / min) are reported, with the algorithmic FLOP of each workload
(2 x MAC of the linears and attention) and the TFLOP/s achieved, counted over all prompts
(what the transformers arm computes) and over the distinct prompts (what the native arm
computes; `native_tflops_distinct` is its arithmetic rate).
Prints one JSON line with the card name and power limit read in the same run.

Usage: python tools/text_encoder_bench.py [--rounds 3] [--warmup 1] [--layers-scale 1.0]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from fp8_bench import card  # noqa: E402

SEQ = 77
# name -> (kind, layers, hidden, heads, ff, act, projection, vocab)
ENCODERS = {
    "clip_l": ("clip_proj", 12, 768, 12, 3072, "quick_gelu", 768, 49408),
    "clip_g": ("clip_proj", 32, 1280, 20, 5120, "gelu", 1280, 49408),
    "t5_xxl": ("t5", 24, 4096, 64, 10240, None, None, 32128),
    "sd21": ("clip", 23, 1024, 16, 4096, "gelu", None, 49408),
}


def flop_per_prompt(name):
    kind, layers, d, heads, ff, _, proj, _ = ENCODERS[name]
    inner = heads * 64
    lin = 4 * d * inner + (3 if kind == "t5" else 2) * d * ff
    attn = 2 * SEQ * inner
    return 2 * (SEQ * layers * (lin + attn) + (d * proj if proj else 0))


def build(name, layers_scale):
    import transformers
    from dwm.models import text_encoders as te
    kind, layers, d, heads, ff, act, proj, vocab = ENCODERS[name]
    layers = max(1, round(layers * layers_scale))
    torch.manual_seed(list(ENCODERS).index(name))
    if kind == "t5":
        cfg = transformers.T5Config(vocab_size=vocab, d_model=d, d_kv=64, d_ff=ff,
                                    num_layers=layers, num_heads=heads,
                                    feed_forward_proj="gated-gelu")
        cls, ncls = transformers.T5EncoderModel, te.NativeT5EncoderModel
    else:
        cfg = transformers.CLIPTextConfig(
            vocab_size=vocab, hidden_size=d, intermediate_size=ff, projection_dim=proj or d,
            num_hidden_layers=layers, num_attention_heads=heads, max_position_embeddings=SEQ,
            hidden_act=act, bos_token_id=49406, eos_token_id=49407, pad_token_id=49407)
        cls = transformers.CLIPTextModelWithProjection if kind == "clip_proj" \
            else transformers.CLIPTextModel
        ncls = te.NativeCLIPTextModelWithProjection if kind == "clip_proj" \
            else te.NativeCLIPTextModel
    with torch.device("cuda"):
        ref = cls._from_config(cfg, dtype=torch.float16).eval().requires_grad_(False)
    for mod in getattr(cls, "_keep_in_fp32_modules", None) or []:
        for n, m in ref.named_modules():
            if n.split(".")[-1] == mod:
                m.float()
    nat = ncls(cfg, dtype=torch.float16).load_state_dict(ref.state_dict())
    return ref, nat


def prompts(n_distinct, views=6):
    return ["camera {} of frame {}, a street at dusk with parked cars".format(i % views, i // views)
            for i in range(n_distinct)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--layers-scale", type=float, default=1.0,
                    help="fraction of each encoder's layers (1.0 = the published depth)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "text_encoder_bench needs a GPU"
    from common import tiny_text_stack
    from dwm.pipelines.text_conditions import _ids, flatten_prompts, text_conditions
    tok = tiny_text_stack()[0]      # byte-level CLIP tokenizer; ids index every vocabulary
    encs = {n: build(n, args.layers_scale) for n in ENCODERS}
    dev = torch.device("cuda")
    frame = [[prompts(6)]]                       # [B][T=1][V]
    window = [[[p for p in prompts(96)[6 * t:6 * t + 6]] for t in range(16)]]
    work = {"frame": (True, frame), "window": (True, window), "sd21": (False, frame)}

    def arm_encoders(arm, is_dit):
        i = 0 if arm == "transformers" else 1
        if is_dit:
            return [encs[n][i] for n in ("clip_l", "clip_g", "t5_xxl")]
        return encs["sd21"][i]

    def run_encoders(is_dit, e, ids):
        if is_dit:
            e[0](ids, output_hidden_states=True)
            e[1](ids, output_hidden_states=True)
            e[2](ids)
        else:
            e(ids)

    def run_conditions(is_dit, e, clip_text):
        toks = [tok, tok, tok] if is_dit else tok
        text_conditions(is_dit, e, toks, clip_text, 1 if clip_text is frame else 16, 6, dev,
                        torch.float16, None, True)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    times = {}
    with torch.no_grad():
        for r in range(args.warmup + args.rounds):
            for wname, (is_dit, clip_text) in work.items():
                flat, _ = flatten_prompts(clip_text, None, True)
                ids = _ids(tok, flat, SEQ).to(dev)
                for arm in (("transformers", "native") if r % 2 == 0 else ("native", "transformers")):
                    e = arm_encoders(arm, is_dit)
                    t_enc = timed(lambda: run_encoders(is_dit, e, ids))
                    t_all = timed(lambda: run_conditions(is_dit, e, clip_text))
                    if r >= args.warmup:
                        times.setdefault((wname, arm, "encoders"), []).append(t_enc)
                        times.setdefault((wname, arm, "text_conditions"), []).append(t_all)
        # the two arms' states on the frame workload, against each other
        flat, _ = flatten_prompts(frame, None, True)
        ids = _ids(tok, flat, SEQ).to(dev)
        agree = {}
        for n in ENCODERS:
            ref, nat = encs[n]
            a, b = ref(ids, output_hidden_states=True), nat(ids, output_hidden_states=True)
            key = "hidden_states[-2]" if ENCODERS[n][0] == "clip_proj" else "last_hidden_state"
            ya, yb = (a.hidden_states[-2], b.hidden_states[-2]) if key != "last_hidden_state" \
                else (a[0], b[0])
            agree[n] = {key: float((ya.float() - yb.float()).abs().max() / ya.float().abs().max())}
    result = {"card": card(), "rounds": args.rounds, "layers_scale": args.layers_scale,
              "workloads": {}}
    for wname, (is_dit, clip_text) in work.items():
        flat, _ = flatten_prompts(clip_text, None, True)
        names = ("clip_l", "clip_g", "t5_xxl") if is_dit else ("sd21",)
        flop = len(flat) * sum(flop_per_prompt(n) for n in names) * args.layers_scale
        w = {"prompts": len(flat), "distinct": len(set(flat)), "tflop": round(flop / 1e12, 2),
             "tflop_distinct": round(flop * len(set(flat)) / len(flat) / 1e12, 2)}
        for arm in ("transformers", "native"):
            for what in ("encoders", "text_conditions"):
                t = times[(wname, arm, what)]
                med = statistics.median(t)
                w["{}_{}_ms".format(arm, what)] = round(med, 2)
                w["{}_{}_spread".format(arm, what)] = round(max(t) / min(t), 3)
                if what == "encoders":
                    w["{}_tflops".format(arm)] = round(flop / (med * 1e9), 1)
        w["native_tflops_distinct"] = round(w["tflop_distinct"] * 1e3 / w["native_encoders_ms"], 1)
        w["speedup_encoders"] = round(w["transformers_encoders_ms"] / w["native_encoders_ms"], 2)
        w["speedup_text_conditions"] = round(
            w["transformers_text_conditions_ms"] / w["native_text_conditions_ms"], 2)
        result["workloads"][wname] = w
    result["frame_states_rel_diff"] = agree
    print(json.dumps(result))


if __name__ == "__main__":
    main()
