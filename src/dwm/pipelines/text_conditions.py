"""Prompt -> text-condition tensors for `CrossviewTemporalSD.get_conditions`.

The text encoders are callers of the hot path (SURVEY.md §8 A13): by default they run through
Hugging Face `transformers`, exactly as in the reference
(src/dwm/pipelines/ctsd.py:39-83 `flatten_clip_text`, :176-253 the text branch of
`get_conditions`, :744-805 the SD-3 prompt encoders, :886-948 loading).  This module is the
thin adapter that lets reference-style batches (`clip_text` = nested prompt lists) drive the
H100 pipeline when the encoder weights are present; batches that carry pre-encoded
`text_embeddings` / `pooled_text_embeddings` bypass it.  With `native=True` the same calls run
on dwm.models.text_encoders (the sm_90a kernels).
"""
import os

import torch


def flatten_prompts(clip_text, text_condition_mask=None,
                    do_classifier_free_guidance: bool = False):
    """Nested prompt lists ([B], [B][T][V], ...) -> (flat prompt list, shape).  Masked-out
    prompts become "" (the unconditional prompt); with CFG an all-"" copy of the whole
    structure is put in front, which doubles the leading dimension of `shape`."""
    leaves = []

    def walk(node, mask):
        if isinstance(node, str):
            keep = mask is None or (isinstance(mask, bool) and mask)
            leaves.append(node if keep else "")
            return []
        shapes = [walk(child, None if mask is None else
                       (mask[i] if isinstance(mask, list) else mask))
                  for i, child in enumerate(node)]
        return [len(node)] + (shapes[-1] if shapes else [])
    shape = walk(clip_text, text_condition_mask)
    if isinstance(clip_text, str):
        shape = []
    if do_classifier_free_guidance:
        leaves = [""] * len(leaves) + leaves
        if shape:
            shape = [2 * shape[0]] + shape[1:]
    return leaves, shape


def _ids(tokenizer, prompts, max_length, **kw):
    return tokenizer(prompts, padding="max_length", max_length=max_length, truncation=True,
                     return_tensors="pt", **kw).input_ids


@torch.no_grad()
def encode_clip_hidden(text_encoder, tokenizer, prompts, device):
    """SD-2.1: last hidden state of the CLIP text model (reference :186-191)."""
    ids = _ids(tokenizer, prompts, tokenizer.model_max_length)
    return text_encoder(ids.to(device))[0]


@torch.no_grad()
def encode_sd3(text_encoders, tokenizers, prompts, device, t5_max_length: int = 77,
               joint_attention_dim: int = 4096):
    """SD-3 / 3.5: [CLIP-L | CLIP-G] penultimate hidden states, zero-padded to the T5 width
    and followed along the sequence by the T5 states; pooled = concatenated CLIP projections
    (reference :205-236, :744-805)."""
    hidden, pooled = [], []
    for enc, tok in zip(text_encoders[:2], tokenizers[:2]):
        out = enc(_ids(tok, prompts, 77).to(enc.device), output_hidden_states=True)
        pooled.append(out[0])
        hidden.append(out.hidden_states[-2].to(dtype=enc.dtype, device=enc.device))
    clip = torch.cat(hidden, dim=-1)
    t5_enc, t5_tok = text_encoders[-1], tokenizers[-1]
    if t5_enc is None:
        t5 = torch.zeros((len(prompts), t5_max_length, joint_attention_dim), device=device,
                         dtype=torch.float16)
    else:
        t5 = t5_enc(_ids(t5_tok, prompts, t5_max_length, add_special_tokens=True)
                    .to(device))[0].to(dtype=t5_enc.dtype, device=device)
    clip = torch.nn.functional.pad(clip, (0, t5.shape[-1] - clip.shape[-1]))
    return torch.cat([clip, t5], dim=-2), torch.cat(pooled, dim=-1)


def text_conditions(is_dit: bool, text_encoder, tokenizer, clip_text, sequence_length: int,
                    view_count: int, device, dtype, text_condition_mask=None,
                    do_classifier_free_guidance: bool = False):
    """-> (encoder_hidden_states [B', T, V, L, C], pooled [B', T, V, P] or None)."""
    prompts, shape = flatten_prompts(clip_text, text_condition_mask,
                                     do_classifier_free_guidance)
    if is_dit:
        states, pooled = encode_sd3(text_encoder, tokenizer, prompts, device)
    else:
        states, pooled = encode_clip_hidden(text_encoder, tokenizer, prompts, device), None

    def spread(t):
        if t is None:
            return None
        if len(shape) == 1:      # one prompt per sample, shared by all frames and views
            t = t[:, None, None].expand(-1, sequence_length, view_count,
                                        *t.shape[1:]).contiguous()
        else:
            t = t.unflatten(0, shape)
        return t.to(dtype=dtype)
    return spread(states), (spread(pooled) if is_dit else None)


def load_text_encoders(is_dit: bool, path: str, device, load_args: dict, native: bool = False):
    """(text_encoder(s), tokenizer(s)) from a diffusers-layout checkpoint directory, or None
    when it does not hold them (then conditions must come pre-encoded).  native=True loads the
    encoders as dwm.models.text_encoders (the sm_90a kernels, from safetensors weights, with
    load_args' torch_dtype as the dtype of the states they return); tokenizers stay
    transformers on the CPU."""
    import transformers

    def has(sub):
        return path is not None and os.path.isdir(os.path.join(path, sub))
    if not has("tokenizer") or not has("text_encoder"):
        return None
    if native:
        from dwm.models import text_encoders as te
        dtype = load_args.get("torch_dtype", load_args.get("dtype"))

        def load(cls, sub):
            return cls.from_pretrained(path, subfolder=sub, device=device, torch_dtype=dtype)
        clip, clip_proj, t5 = (te.NativeCLIPTextModel, te.NativeCLIPTextModelWithProjection,
                               te.NativeT5EncoderModel)
    else:
        frozen = lambda m: m.requires_grad_(False).eval()   # noqa: E731

        def load(cls, sub):
            return frozen(cls.from_pretrained(path, subfolder=sub, **load_args)).to(device)
        clip, clip_proj, t5 = (transformers.CLIPTextModel,
                               transformers.CLIPTextModelWithProjection,
                               transformers.T5EncoderModel)
    if not is_dit:
        tok = transformers.CLIPTokenizer.from_pretrained(path, subfolder="tokenizer")
        return load(clip, "text_encoder"), tok
    toks = [transformers.CLIPTokenizer.from_pretrained(path, subfolder="tokenizer"),
            transformers.CLIPTokenizer.from_pretrained(path, subfolder="tokenizer_2"),
            transformers.T5TokenizerFast.from_pretrained(path, subfolder="tokenizer_3")]
    encs = [load(clip_proj, sub) for sub in ("text_encoder", "text_encoder_2")]
    encs.append(load(t5, "text_encoder_3") if has("text_encoder_3") else None)
    return encs, toks
