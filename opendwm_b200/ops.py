"""Thin torch-tensor front end of the C ABI: validates shapes/dtypes, passes raw
device pointers + the current CUDA stream.  PyTorch only owns the memory."""
import ctypes

import torch

from . import lib as _l


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return _l.DWM_BF16
    if t.dtype == torch.float16:
        return _l.DWM_F16
    raise TypeError("expected a bf16/fp16 tensor, got {}".format(t.dtype))


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    if _prof is not None:
        _prof["launches"] += 1
    return torch.cuda.current_stream().cuda_stream


_prof = None


def profile_begin():
    """Starts counting kernel launches and timing every dwm_b200_linear launch with a
    CUDA event pair on the launching stream (used by bench.py's roofline figure)."""
    global _prof
    _prof = {"launches": 0, "events": []}


def profile_end():
    """Stops profiling; call after a stream synchronize.  Returns
    {"launches": n, "linear": [{"ms", "flops", "shape", "epilogue"}, ...]}."""
    global _prof
    p, _prof = _prof, None
    out = {"launches": p["launches"], "linear": []}
    for e0, e1, flops, shape, epi in p["events"]:
        out["linear"].append({"ms": e0.elapsed_time(e1), "flops": flops,
                              "shape": shape, "epilogue": epi})
    return out


def _f32(t, name):
    if t is not None:
        if t.dtype != torch.float32 or not t.is_cuda:
            raise TypeError("{} must be a cuda fp32 tensor".format(name))
        if t.stride(-1) != 1:
            raise ValueError("{} must be contiguous in its last dim".format(name))
    return t


def _rows2d(t, name):
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError("{} must be 2-D with contiguous rows".format(name))
    return t


FP8 = torch.float8_e4m3fn


def _cdiv(a, b):
    return (a + b - 1) // b


def _need(t, name, rows, cols):
    """t must cover [rows, cols] (a 1-D t: cols elements)."""
    if t is None:
        return
    have = (1, t.shape[0]) if t.dim() == 1 else (t.shape[0], t.shape[1])
    if have[0] < rows or have[1] < cols:
        raise ValueError("{} is {}, the epilogue addresses [{}, {}]".format(
            name, list(t.shape), rows, cols))


def _check_fp32_epilogue(rows, cols, bias, resid, resid_rows, blend_x, alpha, rows_per_batch):
    """Extents of the fp32 operands every fused epilogue reads."""
    _need(bias, "bias", 1, cols)
    _need(resid, "resid", resid_rows, cols)
    _need(blend_x, "blend_x", rows, cols)
    if blend_x is not None and alpha is not None:
        _need(alpha, "alpha", 1, _cdiv(rows, rows_per_batch) if rows_per_batch > 0 else 1)


def _check_linear_extents(M, N, epilogue, out, bias, rows_per_item, out_item_stride,
                          out_row_offset, resid, resid_row_mod, gate, blend_x, alpha,
                          rows_per_batch):
    """Every row the epilogue of dwm_b200_linear reads or writes lies inside its tensor."""
    items = _cdiv(M, rows_per_item) if rows_per_item > 0 else 1
    if epilogue in (_l.EPI_RESID, _l.EPI_F32):
        out_rows = M
    else:
        if out_row_offset < 0:
            raise ValueError("out_row_offset must be >= 0")
        if rows_per_item > 0:
            if out_item_stride < rows_per_item:
                raise ValueError("out_item_stride {} < rows_per_item {}: items would share "
                                 "output rows".format(out_item_stride, rows_per_item))
            last = items - 1
            out_rows = last * out_item_stride + (M - last * rows_per_item)
        else:
            out_rows = M
        out_rows += out_row_offset
    if out.shape[0] < out_rows:
        raise ValueError("out has {} rows, the epilogue writes {}".format(out.shape[0], out_rows))
    if resid_row_mod > 0:
        resid_rows = min(resid_row_mod, M)
    else:
        resid_rows = items if resid_row_mod < 0 else M
    _check_fp32_epilogue(M, N, bias, resid, resid_rows, blend_x, alpha, rows_per_batch)
    _need(gate, "gate", items, N)


def linear(a, w, bias=None, *, epilogue=_l.EPI_STORE, act=_l.ACT_NONE,
           out=None, rows_per_item=0, out_item_stride=0, out_row_offset=0,
           q_norm_weight=None, k_norm_weight=None, qk_region=0, eps=1e-6,
           qk_norm_regions=0, peer_out=None, resid=None, resid_row_mod=0, gate=None, blend_x=None, alpha=None,
           rows_per_batch=0, a_scale=None, w_scale=None, out_dtype=None):
    """out = epilogue(a @ w.T).  a [M,K], w [N,K] 16-bit; see include/dwm_b200.h.
    FP8: a and w float8_e4m3fn with fp32 row scales a_scale [M] and w_scale [N]
    (quantize_rows / quantize_weight_rows); out_dtype (bf16 / fp16) is the type of the
    16-bit outputs and is required."""
    _rows2d(a, "a")
    _rows2d(w, "w")
    if not (a.is_cuda and w.is_cuda):
        raise RuntimeError("dwm_b200 kernels need CUDA tensors (no CPU fallback)")
    if a.dtype != w.dtype:
        raise TypeError("a and w dtypes differ: {} vs {}".format(a.dtype, w.dtype))
    M, K = a.shape
    N, K2 = w.shape
    if K != K2:
        raise ValueError("K mismatch: a {} vs w {}".format(K, K2))
    fp8 = a.dtype == FP8
    if fp8:
        if a_scale is None or w_scale is None:
            raise ValueError("FP8 operands need a_scale and w_scale")
        for t, n, name in ((a_scale, M, "a_scale"), (w_scale, N, "w_scale")):
            _f32(t, name)
            if t.dim() != 1 or t.numel() != n:
                raise ValueError("{} must be fp32 [{}]".format(name, n))
        if out_dtype not in (torch.bfloat16, torch.float16):
            raise TypeError("FP8 operands need out_dtype bf16 or fp16, got {}".format(out_dtype))
        out16 = out_dtype
    else:
        if a_scale is not None or w_scale is not None:
            raise ValueError("a_scale / w_scale go with float8_e4m3fn operands")
        if out_dtype not in (None, a.dtype):
            raise TypeError("16-bit operands write their own dtype, not {}".format(out_dtype))
        out16 = a.dtype
    out_cols = N // 2 if epilogue in (_l.EPI_GEGLU, _l.EPI_GEGLU_TANH) else N
    if out is None:
        if epilogue in (_l.EPI_RESID, _l.EPI_F32):
            out = torch.empty((M, out_cols), device=a.device, dtype=torch.float32)
        else:
            out = torch.empty((M, out_cols), device=a.device, dtype=out16)
    _rows2d(out, "out")
    want = torch.float32 if epilogue in (_l.EPI_RESID, _l.EPI_F32) else out16
    if out.dtype != want:
        raise TypeError("out dtype {} != {}".format(out.dtype, want))
    if out.shape[1] < out_cols:
        raise ValueError("out has {} columns, need {}".format(out.shape[1], out_cols))
    _check_linear_extents(M, N, epilogue, out, bias, rows_per_item, out_item_stride,
                          out_row_offset, resid, resid_row_mod, gate, blend_x, alpha,
                          rows_per_batch)
    args = _l.LinearArgs()
    args.M, args.N, args.K = M, N, K
    args.A, args.lda = a.data_ptr(), a.stride(0)
    args.W, args.ldw = w.data_ptr(), w.stride(0)
    args.bias = _ptr(_f32(bias, "bias"))
    if fp8:
        args.dtype, args.out_dtype = _l.DWM_E4M3, _dt(torch.empty(0, dtype=out16))
        args.a_scale, args.w_scale = a_scale.data_ptr(), w_scale.data_ptr()
    else:
        args.dtype = args.out_dtype = _dt(a)
    args.epilogue, args.act = epilogue, act
    args.out, args.ldo = out.data_ptr(), out.stride(0)
    args.rows_per_item = rows_per_item
    args.out_item_stride = out_item_stride
    args.out_row_offset = out_row_offset
    args.q_norm_weight = _ptr(_f32(q_norm_weight, "q_norm_weight"))
    args.k_norm_weight = _ptr(_f32(k_norm_weight, "k_norm_weight"))
    args.qk_region = qk_region
    args.eps = eps
    args.qk_norm_regions = qk_norm_regions
    if resid is not None:
        _rows2d(_f32(resid, "resid"), "resid")
        args.resid, args.ldr = resid.data_ptr(), resid.stride(0)
    args.resid_row_mod = resid_row_mod
    if gate is not None:
        _rows2d(_f32(gate, "gate"), "gate")
        args.gate, args.gate_ld = gate.data_ptr(), gate.stride(0)
    if blend_x is not None:
        _rows2d(_f32(blend_x, "blend_x"), "blend_x")
        args.blend_x, args.ldx = blend_x.data_ptr(), blend_x.stride(0)
    args.alpha = _ptr(_f32(alpha, "alpha"))
    args.rows_per_batch = rows_per_batch
    if peer_out:
        # raw device pointers of the peers' buffers (same layout / pitch as `out`)
        if len(peer_out) > 8:
            raise ValueError("at most 8 peer buffers")
        for i, ptr in enumerate(peer_out):
            args.peer_out[i] = int(ptr)
        args.n_peer_out = len(peer_out)
    if _prof is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = _l.load().dwm_b200_linear(ctypes.byref(args), _stream())
        e1.record()
        _prof["events"].append((e0, e1, 2.0 * M * N * K, (M, N, K), epilogue))
    else:
        rc = _l.load().dwm_b200_linear(ctypes.byref(args), _stream())
    _l.check(rc, "dwm_b200_linear")
    return out


def quantize_rows(x, out=None, scale=None):
    """Row-wise E4M3 quantization of a bf16 / fp16 / fp32 [M, K] tensor (rows contiguous):
    returns (out float8_e4m3fn [M, K], scale fp32 [M]) with x[m] ~= out[m] * scale[m];
    see dwm_b200_quantize_rows for the exact recipe."""
    _rows2d(x, "x")
    if not x.is_cuda:
        raise RuntimeError("dwm_b200 kernels need CUDA tensors (no CPU fallback)")
    M, K = x.shape
    if out is None:
        out = torch.empty(M, K, device=x.device, dtype=FP8)
    if scale is None:
        scale = torch.empty(M, device=x.device, dtype=torch.float32)
    _rows2d(out, "out")
    _f32(scale, "scale")
    if out.dtype != FP8 or out.shape[0] != M or out.shape[1] < K or scale.numel() != M:
        raise ValueError("quantize_rows: out must be float8_e4m3fn [M, >= K], scale fp32 [M]")
    _l.check(_l.load().dwm_b200_quantize_rows(
        x.data_ptr(), M, K, x.stride(0), _code(x.dtype), out.data_ptr(), out.stride(0),
        scale.data_ptr(), _stream()), "dwm_b200_quantize_rows")
    return out, scale


def quantize_weight_rows(w):
    """nn.Linear weight [N, K] (any float dtype, on the GPU) -> (w8 float8_e4m3fn [N, K],
    fp32 scale [N]), one scale per output channel, quantized from fp32."""
    return quantize_rows(w.detach().float().contiguous())


def pack_geglu(weight: torch.Tensor, bias=None, block=128):
    """Re-orders a diffusers GEGLU projection (rows [0,F) value, [F,2F) gate,
    FeedForward net.0.proj) into blocks [128 value | 128 gate] so one 256-column
    GEMM tile holds matching value/gate columns.  T5's gated GELU packs the same way
    from cat([wi_1, wi_0]) (value wi_1, gate wi_0) for EPI_GEGLU_TANH."""
    two_f = weight.shape[0]
    f = two_f // 2
    if f % block:
        raise ValueError("GEGLU inner dim {} not a multiple of {}".format(f, block))
    idx = torch.arange(two_f, device=weight.device).view(2, f // block, block)
    idx = idx.permute(1, 0, 2).reshape(-1)
    w = weight.index_select(0, idx).contiguous()
    b = None if bias is None else bias.index_select(0, idx).contiguous()
    return w, b


def _code(dtype):
    if dtype == torch.bfloat16:
        return _l.DWM_BF16
    if dtype == torch.float16:
        return _l.DWM_F16
    if dtype == torch.float32:
        return _l.DWM_F32
    raise TypeError("unsupported dtype {}".format(dtype))


def attention(qkv, out, *, D, heads, group_dims, group_strides, seq, inner=None,
              stride_outer=0, stride_inner=1, out_group_strides=None,
              out_stride_outer=None, out_stride_inner=None, split=0, out2=None,
              mask=None, mask_div=1, scale=None, kv=None, k_col=0, v_col=0,
              kv_group_strides=None, seq_kv=None, inner_kv=None,
              kv_stride_outer=0, kv_stride_inner=1, mask_q_offset=0, causal=False, bias=None):
    """Gathered multi-head attention over the fused q|k|v buffer (or a separate
    key/value buffer `kv`); see dwm_attention_args in include/dwm_b200.h.  Text encoders:
    `causal` (CLIP) or `bias` fp32 [heads, seq, seq] added to the scaled scores (T5), on
    contiguous sequences."""
    _rows2d(qkv, "qkv")
    _rows2d(out, "out")
    if not qkv.is_cuda:
        raise RuntimeError("dwm_b200 kernels need CUDA tensors (no CPU fallback)")
    a = _l.AttentionArgs()
    a.qkv, a.ld, a.D = qkv.data_ptr(), qkv.stride(0), D
    a.heads, a.head_dim, a.dtype = heads, D // heads, _dt(qkv)
    gd = list(group_dims) + [1] * (3 - len(group_dims))
    gs = list(group_strides) + [0] * (3 - len(group_strides))
    ogs = gs if out_group_strides is None else \
        list(out_group_strides) + [0] * (3 - len(out_group_strides))
    for i in range(3):
        a.group_dims[i], a.group_strides[i], a.out_group_strides[i] = \
            gd[i], gs[i], ogs[i]
    a.seq, a.inner = seq, seq if inner is None else inner
    a.stride_outer, a.stride_inner = stride_outer, stride_inner
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    a.out_stride_outer = stride_outer if out_stride_outer is None \
        else out_stride_outer
    a.out_stride_inner = stride_inner if out_stride_inner is None \
        else out_stride_inner
    a.split = split
    if out2 is not None:
        _rows2d(out2, "out2")
        a.out2, a.ldo2 = out2.data_ptr(), out2.stride(0)
    if mask is not None:
        if mask.dtype != torch.uint8 or mask.dim() != 3 or not mask.is_contiguous():
            raise TypeError("mask must be a contiguous uint8 [B, n, n] tensor")
        a.mask, a.mask_div, a.n_outer = mask.data_ptr(), mask_div, mask.shape[-1]
    a.mask_q_offset = mask_q_offset
    a.scale = (D // heads) ** -0.5 if scale is None else scale
    if kv is not None:
        _rows2d(kv, "kv")
        if kv.dtype != qkv.dtype:
            raise TypeError("kv dtype differs from q dtype")
        a.kv, a.ld_kv, a.k_col, a.v_col = kv.data_ptr(), kv.stride(0), k_col, v_col
        kgs = list(kv_group_strides) + [0] * (3 - len(kv_group_strides))
        for i in range(3):
            a.kv_group_strides[i] = kgs[i]
        a.seq_kv = seq if seq_kv is None else seq_kv
        a.inner_kv = a.seq_kv if inner_kv is None else inner_kv
        a.kv_stride_outer, a.kv_stride_inner = kv_stride_outer, kv_stride_inner
    if causal or bias is not None:
        if bias is not None:
            _f32(bias, "bias")
            if tuple(bias.shape) != (heads, seq, seq) or not bias.is_contiguous():
                raise ValueError("bias must be contiguous fp32 [heads, seq, seq] = [{}, {}, {}], "
                                 "got {}".format(heads, seq, seq, list(bias.shape)))
        _l.check(_l.load().dwm_b200_attention_text(ctypes.byref(a), int(bool(causal)),
                                                   _ptr(bias), _stream()),
                 "dwm_b200_attention_text")
        return out
    _l.check(_l.load().dwm_b200_attention(ctypes.byref(a), _stream()),
             "dwm_b200_attention")
    return out


def layernorm(x, out, *, weight=None, bias=None, eps=1e-5, add_item=None,
              add_full=None, rows_per_item=0, sum_out=None, shift=None,
              scale=None, shift2=None, scale2=None, out2=None, out_scale=None,
              out2_scale=None):
    """LayerNorm (+adds, +AdaLN modulation) of an fp32 stream into 16-bit out, or into
    float8_e4m3fn out (and out2) with fp32 row scales out_scale [M] (out2_scale [M])."""
    _rows2d(_f32(x, "x"), "x")
    _rows2d(out, "out")
    a = _l.LayerNormArgs()
    a.M, a.D = x.shape
    a.x, a.ldx = x.data_ptr(), x.stride(0)
    if add_item is not None:
        _rows2d(_f32(add_item, "add_item"), "add_item")
        a.add_item, a.add_item_ld = add_item.data_ptr(), add_item.stride(0)
    if add_full is not None:
        _rows2d(_f32(add_full, "add_full"), "add_full")
        a.add_full, a.add_full_ld = add_full.data_ptr(), add_full.stride(0)
    a.rows_per_item = rows_per_item
    if sum_out is not None:
        _rows2d(_f32(sum_out, "sum_out"), "sum_out")
        a.sum_out, a.ld_sum = sum_out.data_ptr(), sum_out.stride(0)
    a.weight, a.bias, a.eps = _ptr(_f32(weight, "weight")), _ptr(_f32(bias, "bias")), eps
    mod_ld = None
    for name, t in (("shift", shift), ("scale", scale), ("shift2", shift2),
                    ("scale2", scale2)):
        if t is not None:
            _rows2d(_f32(t, name), name)
            if mod_ld is not None and t.stride(0) != mod_ld:
                raise ValueError("modulation tensors must share a row pitch")
            mod_ld = t.stride(0)
            setattr(a, name, t.data_ptr())
    a.mod_ld = mod_ld or 0
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    if out2 is not None:
        _rows2d(out2, "out2")
        a.out2, a.ldo2 = out2.data_ptr(), out2.stride(0)
    if out.dtype == FP8:
        if out_scale is None or (out2 is not None and (out2_scale is None or out2.dtype != FP8)):
            raise ValueError("FP8 layernorm output needs out_scale (and an FP8 out2 with out2_scale)")
        for t, name in ((out_scale, "out_scale"), (out2_scale, "out2_scale")):
            if t is not None and _f32(t, name).numel() != a.M:
                raise ValueError("{} must be fp32 [M]".format(name))
        a.dtype = _l.DWM_E4M3
        a.out_scale, a.out2_scale = out_scale.data_ptr(), _ptr(out2_scale)
    else:
        if out_scale is not None or out2_scale is not None:
            raise ValueError("out_scale / out2_scale go with a float8_e4m3fn out")
        a.dtype = _dt(out)
    _l.check(_l.load().dwm_b200_layernorm(ctypes.byref(a), _stream()),
             "dwm_b200_layernorm")
    return out


def rmsnorm(x, weight, out, eps=1e-6):
    """T5LayerNorm of an fp32 [M, D] stream: out = weight * x * rsqrt(mean(x^2) + eps), out
    bf16 / fp16 (the GEMM operand) or fp32."""
    _rows2d(_f32(x, "x"), "x")
    _rows2d(out, "out")
    _f32(weight, "weight")
    M, D = x.shape
    if weight.numel() != D or tuple(out.shape[:1]) != (M,) or out.shape[1] < D:
        raise ValueError("rmsnorm: weight must be [D] and out [M, >= D]")
    _l.check(_l.load().dwm_b200_rmsnorm(
        x.data_ptr(), M, D, x.stride(0), weight.data_ptr(), float(eps), out.data_ptr(),
        out.stride(0), _code(out.dtype), _stream()), "dwm_b200_rmsnorm")
    return out


def embed(ids, tok, out, pos=None, seq=None):
    """out[m] = tok[ids[m]] (+ pos[m % seq]): the token / position embedding of a text
    encoder into its fp32 residual stream out [M, D]; ids int64 [M] on the GPU."""
    _f32(tok, "tok")
    _f32(pos, "pos")
    _rows2d(_f32(out, "out"), "out")
    if ids.dtype != torch.int64 or ids.dim() != 1 or not ids.is_contiguous() or not ids.is_cuda:
        raise TypeError("ids must be a contiguous cuda int64 [M] tensor")
    M, D = out.shape
    if ids.numel() != M or tok.dim() != 2 or tok.shape[1] != D or not tok.is_contiguous():
        raise ValueError("embed: ids [M], tok [vocab, D] and out [M, D] must agree")
    seq = M if seq is None else seq
    if pos is not None and (tuple(pos.shape[1:]) != (D,) or pos.shape[0] < seq or
                            not pos.is_contiguous()):
        raise ValueError("embed: pos must be contiguous [>= seq, D]")
    _l.check(_l.load().dwm_b200_embed(
        ids.data_ptr(), M, seq, tok.data_ptr(), tok.shape[0], _ptr(pos), D, out.data_ptr(),
        out.stride(0), _stream()), "dwm_b200_embed")
    return out


def act_cast(x, out, act=_l.ACT_NONE):
    _f32(x, "x")
    if not x.is_contiguous() or not out.is_contiguous():
        raise ValueError("act_cast needs contiguous tensors")
    _l.check(_l.load().dwm_b200_act_cast(
        x.data_ptr(), out.data_ptr(), x.numel(), act, _dt(out), _stream()),
        "dwm_b200_act_cast")
    return out


def sinusoid(t, channels, out, flip_sin_to_cos=True, downscale_freq_shift=0.0):
    _f32(t, "t")
    _rows2d(out, "out")
    _l.check(_l.load().dwm_b200_sinusoid(
        t.data_ptr(), t.numel(), channels, int(flip_sin_to_cos),
        float(downscale_freq_shift), out.data_ptr(), out.stride(0), _dt(out),
        _stream()), "dwm_b200_sinusoid")
    return out


def patchify(x, patch, out):
    _f32(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise ValueError("x must be contiguous [items, C, H, W]")
    _rows2d(out, "out")
    n, c, h, w = x.shape
    _l.check(_l.load().dwm_b200_patchify(
        x.data_ptr(), n, c, h, w, patch, out.data_ptr(), out.stride(0),
        _dt(out), _stream()), "dwm_b200_patchify")
    return out


def cfg_euler_step(tokens, latents, idx, sigmas, *, cfg, guidance_scale, patch,
                   in_range=None, noise_pred=None, round_dtype=torch.float32):
    _rows2d(_f32(tokens, "tokens"), "tokens")
    _f32(latents, "latents")
    _f32(sigmas, "sigmas")
    if latents.dim() != 6 or not latents.is_contiguous():
        raise ValueError("latents must be contiguous [B,T,V,C,H,W]")
    if idx.dtype != torch.int32 or not idx.is_contiguous():
        raise TypeError("idx must be contiguous int32 [B,T,V]")
    if in_range is not None and (in_range.dtype != torch.uint8 or
                                 in_range.numel() != latents.shape[1]):
        raise TypeError("in_range must be uint8 [T]")
    B, T, V, C, H, W = latents.shape
    _l.check(_l.load().dwm_b200_cfg_euler_step(
        tokens.data_ptr(), tokens.stride(0), cfg, float(guidance_scale),
        B, T, V, C, H, W, patch, idx.data_ptr(), sigmas.data_ptr(),
        sigmas.numel(), _ptr(in_range), latents.data_ptr(), _ptr(noise_pred),
        _code(round_dtype), _stream()), "dwm_b200_cfg_euler_step")
    return latents


def euler_step_by_indices(model_output, sample, idx, sigmas, round_dtype=torch.float32):
    """sample (fp32, in place) += dsigma[idx] * model_output; idx int32 over the
    leading dims of sample."""
    _f32(model_output, "model_output")
    _f32(sample, "sample")
    _f32(sigmas, "sigmas")
    if not (model_output.is_contiguous() and sample.is_contiguous() and idx.is_contiguous()):
        raise ValueError("euler_step_by_indices needs contiguous tensors")
    if idx.dtype != torch.int32:
        raise TypeError("idx must be int32")
    n = sample.numel()
    if idx.numel() == 0 or n % idx.numel():
        raise ValueError("sample has {} elements, not a multiple of idx's {}".format(
            n, idx.numel()))
    inner = n // idx.numel()
    _l.check(_l.load().dwm_b200_euler_step_by_indices(
        model_output.data_ptr(), sample.data_ptr(), n, inner, idx.data_ptr(),
        sigmas.data_ptr(), sigmas.numel(), _code(round_dtype), _stream()),
        "dwm_b200_euler_step_by_indices")
    return sample


def pack_conv_weight(weight: torch.Tensor, dtype, pad_out_to=None, pad_in_to=None):
    """torch Conv3d/Conv2d weight [O, I, (kt,) kh, kw] -> tap-major [kt*kh*kw, O', I']
    (optionally zero-padding O / I)."""
    if weight.dim() == 4:
        weight = weight.unsqueeze(2)
    o, i, kt, kh, kw = weight.shape
    w = weight.detach().permute(2, 3, 4, 0, 1).reshape(kt * kh * kw, o, i)
    op = pad_out_to or o
    ip = pad_in_to or i
    if op != o or ip != i:
        wp = torch.zeros(kt * kh * kw, op, ip, device=w.device, dtype=w.dtype)
        wp[:, :o, :i] = w
        w = wp
    return w.to(dtype).contiguous()


def pack_conv_weight_fp8(weight: torch.Tensor):
    """torch Conv3d/Conv2d weight [O, I, (kt,) kh, kw] (on the GPU) -> (E4M3 tap-major
    [kt*kh*kw, O, I], fp32 scale [O]).  Each output channel has ONE scale, the amax over all
    of its taps and input channels: the [O, taps*I] view is quantized row-wise from fp32, then
    stored tap-major like pack_conv_weight."""
    if weight.dim() == 4:
        weight = weight.unsqueeze(2)
    o, i, kt, kh, kw = weight.shape
    rows = weight.detach().float().permute(0, 2, 3, 4, 1).reshape(o, kt * kh * kw * i)
    q, s = quantize_rows(rows.contiguous())
    return q.view(o, kt * kh * kw, i).transpose(0, 1).contiguous(), s


def conv(x, weight, bias=None, *, kernel, epilogue=_l.EPI_F32, act=_l.ACT_NONE,
         out=None, resid=None, resid_rows_per_item=0, blend_x=None, alpha=None,
         rows_per_batch=0, a_scale=None, w_scale=None):
    """x: 16-bit channels-last [nb, tp, h, w, c_in]; weight: tap-major
    [kt*kh*kw, c_out, c_in]; returns [nb*(tp-kt+1)*h*w, c_out].
    FP8: x and weight float8_e4m3fn with a_scale fp32 [nb] (one per volume,
    groupnorm_silu_e4m3 / spatialnorm_silu_e4m3) and w_scale fp32 [c_out]
    (pack_conv_weight_fp8); RESID, or F32 with c_out % 128 == 0."""
    if x.dim() != 5 or not x.is_contiguous() or not weight.is_contiguous():
        raise ValueError("conv: x must be contiguous [nb, tp, h, w, c]")
    if not x.is_cuda:
        raise RuntimeError("dwm_b200 kernels need CUDA tensors (no CPU fallback)")
    kt, kh, kw = kernel
    nb, tp, h, w, c_in = x.shape
    taps, c_out, c_in2 = weight.shape
    if taps != kt * kh * kw or c_in2 != c_in or weight.dtype != x.dtype:
        raise ValueError("conv: weight shape/dtype mismatch")
    fp8 = x.dtype == FP8
    if fp8:
        if a_scale is None or w_scale is None:
            raise ValueError("conv: FP8 operands need a_scale and w_scale")
        if epilogue != _l.EPI_RESID and (epilogue != _l.EPI_F32 or c_out % 128):
            raise ValueError("conv: FP8 operands need the RESID epilogue, or F32 with "
                             "c_out % 128 == 0; got epilogue {} with c_out {}".format(
                                 epilogue, c_out))
        for t, n, name in ((a_scale, nb, "a_scale"), (w_scale, c_out, "w_scale")):
            _f32(t, name)
            if t.dim() != 1 or t.numel() != n:
                raise ValueError("{} must be fp32 [{}]".format(name, n))
    elif a_scale is not None or w_scale is not None:
        raise ValueError("conv: a_scale / w_scale go with float8_e4m3fn operands")
    rows = nb * (tp - kt + 1) * h * w
    want = x.dtype if epilogue == _l.EPI_STORE else torch.float32
    if out is None:
        out = torch.empty(rows, c_out, device=x.device, dtype=want)
    _rows2d(out, "out")
    if out.dtype != want or out.shape[0] < rows or out.shape[1] < c_out:
        raise TypeError("conv: bad out tensor")
    if epilogue != _l.EPI_RESID and (resid is not None or blend_x is not None):
        raise ValueError("conv: resid / blend_x need the RESID epilogue")
    if resid_rows_per_item:
        resid_rows = _cdiv(rows, resid_rows_per_item)
    else:
        resid_rows = rows
    _check_fp32_epilogue(rows, c_out, bias, resid, resid_rows, blend_x, alpha, rows_per_batch)
    a = _l.ConvArgs()
    a.x, a.nb, a.tp, a.h, a.w, a.c_in = x.data_ptr(), nb, tp, h, w, c_in
    a.weight, a.kt, a.kh, a.kw, a.c_out = weight.data_ptr(), kt, kh, kw, c_out
    a.bias = _ptr(_f32(bias, "bias"))
    a.dtype, a.epilogue, a.act = _l.DWM_E4M3 if fp8 else _dt(x), epilogue, act
    if fp8:
        a.a_scale, a.w_scale = a_scale.data_ptr(), w_scale.data_ptr()
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    if resid is not None:
        _rows2d(_f32(resid, "resid"), "resid")
        a.resid, a.ldr = resid.data_ptr(), resid.stride(0)
        if resid_rows_per_item:
            a.resid_per_item, a.rows_per_item = 1, resid_rows_per_item
    if blend_x is not None:
        _rows2d(_f32(blend_x, "blend_x"), "blend_x")
        a.blend_x, a.ldx = blend_x.data_ptr(), blend_x.stride(0)
        a.alpha, a.rows_per_batch = _f32(alpha, "alpha").data_ptr(), rows_per_batch
    _l.check(_l.load().dwm_b200_conv(ctypes.byref(a), _stream()), "dwm_b200_conv")
    return out


def groupnorm_stats(x, groups, sums=None):
    """x fp32 channels-last [nb, T, H, W, C] -> double [nb, groups, 2] (sum, sum sq)."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    if sums is None:
        sums = torch.empty(nb, groups, 2, device=x.device, dtype=torch.float64)
    _l.check(_l.load().dwm_b200_groupnorm_stats(
        x.data_ptr(), nb, T * H * W, C, groups, sums.data_ptr(), _stream()),
        "dwm_b200_groupnorm_stats")
    return sums


def _check_gn_operands(sums, gamma, beta, nb, C, groups):
    """GroupNorm statistics double [nb, groups, 2] and affine parameters fp32 [>= C]."""
    if sums.dtype != torch.float64 or not sums.is_contiguous() or \
            tuple(sums.shape) != (nb, groups, 2):
        raise ValueError("sums must be contiguous float64 [{}, {}, 2]".format(nb, groups))
    for t, name in ((gamma, "gamma"), (beta, "beta")):
        _f32(t, name)
        if t.numel() < C:
            raise ValueError("{} has {} elements, the kernel reads {}".format(name, t.numel(), C))


def spatialnorm_silu(x, sums, gamma, beta, out, *, groups, eps=1e-6, zy=None,
                     zb=None, out_t0=0, silu=True):
    """x fp32 [nb,T,H,W,C]; out 16-bit [nb,out_T,H,W,C]; zy/zb fp32 [nb,Tz,hz,wz,C]."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    if out.dim() != 5 or not out.is_contiguous() or out.shape[0] != nb or out.shape[2:] != x.shape[2:]:
        raise ValueError("out must be contiguous [nb, out_T, H, W, C]")
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    Tz, hz, wz = _spatial_mod(zy, zb, nb, C)
    _l.check(_l.load().dwm_b200_spatialnorm_silu(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(),
        _ptr(zy), _ptr(zb), Tz, hz, wz, int(silu), out.data_ptr(), out.shape[1],
        out_t0, _dt(out), _stream()), "dwm_b200_spatialnorm_silu")
    return out


def _spatial_mod(zy, zb, nb, C):
    """(Tz, hz, wz) of the SpatialNorm3D modulation zy / zb fp32 [nb, Tz, hz, wz, C] (zeros
    without one)."""
    if (zy is None) != (zb is None):
        raise ValueError("zy and zb go together")
    if zy is None:
        return 0, 0, 0
    for t, name in ((zy, "zy"), (zb, "zb")):
        _f32(t, name)
        if t.dim() != 5 or not t.is_contiguous() or t.shape[0] != nb or t.shape[4] != C:
            raise ValueError("{} must be contiguous fp32 [nb, Tz, hz, wz, C]".format(name))
    if zb.shape != zy.shape:
        raise ValueError("zy and zb shapes differ")
    return tuple(zy.shape[1:4])


def spatialnorm_silu_e4m3(x, sums, gamma, beta, out, scale, *, groups, eps=1e-6, zy=None,
                          zb=None, out_t0=0, silu=True, tail_in=None, tail_out=None):
    """SpatialNorm3D(+SiLU) of x fp32 [nb,T,H,W,C] (zy / zb as in spatialnorm_silu) into E4M3
    out [nb,out_T,H,W,C] (frames [out_t0, out_t0+T)) with one fp32 scale per volume in
    scale [nb].  tail_in (16-bit [nb,2,H,W,C]): the previous chunk's causal-conv cache, covered
    by the volume's amax and quantized into frames out_t0-2, out_t0-1.  tail_out (same
    layout and dtype, may be tail_in): receives the operand's last two frames in 16 bit."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    for t, name in ((out, "out"), (scale, "scale"), (sums, "sums"), (gamma, "gamma"),
                    (beta, "beta"), (zy, "zy"), (zb, "zb"), (tail_in, "tail_in"),
                    (tail_out, "tail_out")):
        if t is not None and t.device != x.device:
            raise RuntimeError("spatialnorm_silu_e4m3: {} is on {}, x on {} (every operand on "
                               "x's GPU; no CPU fallback)".format(name, t.device, x.device))
    if out.dtype != FP8 or out.dim() != 5 or not out.is_contiguous() or \
            out.shape[0] != nb or out.shape[2:] != x.shape[2:]:
        raise ValueError("out must be contiguous float8_e4m3fn [nb, out_T, H, W, C]")
    _f32(scale, "scale")
    if scale.numel() != nb or not scale.is_contiguous():
        raise ValueError("scale must be fp32 [nb]")
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    Tz, hz, wz = _spatial_mod(zy, zb, nb, C)
    tails = [t for t in (tail_in, tail_out) if t is not None]
    for t in tails:
        if t.dtype != tails[0].dtype or t.dim() != 5 or not t.is_contiguous() or \
                tuple(t.shape) != (nb, 2, H, W, C):
            raise ValueError("tail_in / tail_out must be contiguous 16-bit [nb, 2, H, W, C] of "
                             "one dtype")
    _l.check(_l.load().dwm_b200_spatialnorm_silu_e4m3(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(),
        _ptr(zy), _ptr(zb), Tz, hz, wz, int(silu), out.data_ptr(), out.shape[1], out_t0,
        scale.data_ptr(), _ptr(tail_in), _ptr(tail_out), _dt(tails[0]) if tails else 0,
        _stream()), "dwm_b200_spatialnorm_silu_e4m3")
    return out, scale


def groupnorm_silu_e4m3(x, sums, gamma, beta, out, scale, *, groups, eps=1e-6, out_t0=0,
                        silu=True):
    """GroupNorm(+SiLU) of x fp32 [nb,T,H,W,C] into E4M3 out [nb,out_T,H,W,C] (frames
    [out_t0, out_t0+T) only) with one fp32 scale per volume written to scale [nb]."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    if out.dtype != FP8 or out.dim() != 5 or not out.is_contiguous() or \
            out.shape[0] != nb or out.shape[2:] != x.shape[2:]:
        raise ValueError("out must be contiguous float8_e4m3fn [nb, out_T, H, W, C]")
    _f32(scale, "scale")
    if scale.numel() != nb or not scale.is_contiguous():
        raise ValueError("scale must be fp32 [nb]")
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    _l.check(_l.load().dwm_b200_groupnorm_silu_e4m3(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(), int(silu),
        out.data_ptr(), out.shape[1], out_t0, scale.data_ptr(), _stream()),
        "dwm_b200_groupnorm_silu_e4m3")
    return out, scale


def _halo_args(x, out, prev_out, next_out, dtype):
    """Checks a frame shard's operand out [nb, T + 2, H, W, C] and its neighbours' operands
    (None at the ends of the window) -> (prev ptr, prev frames, next ptr, next frames)."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T = x.shape[:2]
    args = []
    for name, t, want_T in (("out", out, T + 2), ("prev_out", prev_out, None),
                            ("next_out", next_out, None)):
        if t is None and name != "out":
            args += [None, 0]
            continue
        if t.dtype != dtype or t.dim() != 5 or not t.is_contiguous() or t.shape[0] != nb or \
                t.shape[2:] != x.shape[2:] or t.shape[1] < 3 or \
                (want_T is not None and t.shape[1] != want_T):
            raise ValueError("{} must be contiguous {} [nb, {}, H, W, C]".format(
                name, dtype, "T + 2" if want_T else "frames + 2"))
        if name != "out":
            args += [t.data_ptr(), t.shape[1]]
    return args


def groupnorm_silu_halo(x, sums, gamma, beta, out, *, groups, stat_frames, prev_out=None,
                        next_out=None, eps=1e-6, silu=True):
    """GroupNorm(+SiLU) of a frame shard x fp32 [nb,T,H,W,C] with statistics `sums` summed over
    the window's `stat_frames` frames, into the shard's 16-bit temporal-conv operand
    out [nb,T+2,H,W,C] (local frames at 1..T); the boundary frames are also stored into the
    neighbours' operands prev_out / next_out, a missing neighbour leaves a zero halo frame."""
    halo = _halo_args(x, out, prev_out, next_out, out.dtype)
    nb, T, H, W, C = x.shape
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    _l.check(_l.load().dwm_b200_groupnorm_silu_halo(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), stat_frames, eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(), int(silu),
        out.data_ptr(), *halo, _dt(out), _stream()), "dwm_b200_groupnorm_silu_halo")
    return out


def groupnorm_silu_e4m3_amax(x, sums, gamma, beta, amax, *, groups, stat_frames, eps=1e-6,
                             silu=True):
    """First E4M3 frame-shard pass: amax fp32 [nb] of the shard's GroupNorm(+SiLU) output, to be
    reduced with MAX over the window's shards before `groupnorm_silu_e4m3_halo`."""
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    _f32(amax, "amax")
    if amax.numel() != nb or not amax.is_contiguous():
        raise ValueError("amax must be fp32 [nb]")
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    _l.check(_l.load().dwm_b200_groupnorm_silu_e4m3_amax(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), stat_frames, eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(), int(silu),
        amax.data_ptr(), _stream()), "dwm_b200_groupnorm_silu_e4m3_amax")
    return amax


def groupnorm_silu_e4m3_halo(x, sums, gamma, beta, amax, out, scale, *, groups, stat_frames,
                             prev_out=None, next_out=None, eps=1e-6, silu=True):
    """Second E4M3 frame-shard pass: quantizes with the window's amax [nb] into
    out float8_e4m3fn [nb,T+2,H,W,C] and scale [nb] (the bytes and scales groupnorm_silu_e4m3
    gives for that amax), halo frames as in `groupnorm_silu_halo`."""
    halo = _halo_args(x, out, prev_out, next_out, FP8)
    nb, T, H, W, C = x.shape
    _check_gn_operands(sums, gamma, beta, nb, C, groups)
    for t, name in ((amax, "amax"), (scale, "scale")):
        _f32(t, name)
        if t.numel() != nb or not t.is_contiguous():
            raise ValueError("{} must be fp32 [nb]".format(name))
    _l.check(_l.load().dwm_b200_groupnorm_silu_e4m3_halo(
        x.data_ptr(), nb, T, H, W, C, groups, sums.data_ptr(), stat_frames, eps,
        _f32(gamma, "gamma").data_ptr(), _f32(beta, "beta").data_ptr(), int(silu),
        amax.data_ptr(), out.data_ptr(), *halo, scale.data_ptr(), _stream()),
        "dwm_b200_groupnorm_silu_e4m3_halo")
    return out, scale


def upsample_nearest(x, compress_time, dtype):
    _f32(x, "x")
    if x.dim() != 5 or not x.is_contiguous():
        raise ValueError("x must be contiguous [nb, T, H, W, C]")
    nb, T, H, W, C = x.shape
    To = T
    if compress_time and T > 1:
        To = 1 + 2 * (T - 1) if T % 2 == 1 else 2 * T
    out = torch.empty(nb, To, 2 * H, 2 * W, C, device=x.device, dtype=dtype)
    _l.check(_l.load().dwm_b200_upsample_nearest(
        x.data_ptr(), nb, T, H, W, C, int(compress_time), out.data_ptr(), _dt(out),
        _stream()), "dwm_b200_upsample_nearest")
    return out


def axpy(x, y, a=1.0):
    """y += a * x (fp32, in place)."""
    _f32(x, "x")
    _f32(y, "y")
    if x.numel() != y.numel() or not (x.is_contiguous() and y.is_contiguous()):
        raise ValueError("axpy needs contiguous tensors of equal size")
    _l.check(_l.load().dwm_b200_axpy(x.data_ptr(), y.data_ptr(), x.numel(), float(a),
                                     _stream()), "dwm_b200_axpy")
    return y


def softmax_rows(x, scale, out):
    """out[r] = softmax(scale * x[r]) — fp32 [rows, cols] (row stride allowed) -> 16-bit."""
    _f32(x, "x")
    if x.dim() != 2 or out.dim() != 2 or x.shape != out.shape or x.stride(1) != 1 or \
            out.stride(1) != 1:
        raise ValueError("softmax_rows needs 2-D row-major tensors of equal shape")
    _l.check(_l.load().dwm_b200_softmax_rows(
        x.data_ptr(), x.shape[0], x.shape[1], x.stride(0), float(scale), out.data_ptr(),
        out.stride(0), _dt(out), _stream()), "dwm_b200_softmax_rows")
    return out


def cfg_ddim_step(pred, latents, timesteps, alphas_cumprod, *, cfg, guidance_scale,
                  step_ratio, final_alpha_cumprod, prediction_type,
                  round_dtype=torch.float32):
    """Fused CFG + DDIM (eta 0) update of fp32 latents [B,T,V,...] in place."""
    _f32(pred, "pred")
    _f32(latents, "latents")
    _f32(alphas_cumprod, "alphas_cumprod")
    if not (pred.is_contiguous() and latents.is_contiguous() and timesteps.is_contiguous()):
        raise ValueError("cfg_ddim_step needs contiguous tensors")
    if timesteps.dtype != torch.int32:
        raise TypeError("timesteps must be int32")
    n_items = timesteps.numel()
    inner = latents.numel() // n_items
    code = {"epsilon": 0, "sample": 1, "v_prediction": 2}[prediction_type]
    _l.check(_l.load().dwm_b200_cfg_ddim_step(
        pred.data_ptr(), cfg, float(guidance_scale), n_items, inner,
        timesteps.data_ptr(), int(step_ratio), alphas_cumprod.data_ptr(),
        alphas_cumprod.numel(), float(final_alpha_cumprod), code, latents.data_ptr(),
        _code(round_dtype), _stream()), "dwm_b200_cfg_ddim_step")
    return latents


def lincomb2(x, y, s0, s1, out):
    """out = s0[item] * x + s1[item] * y with one coefficient pair per item."""
    for t, nme in ((x, "x"), (y, "y"), (s0, "s0"), (s1, "s1"), (out, "out")):
        _f32(t, nme)
        if not t.is_contiguous():
            raise ValueError("lincomb2 needs contiguous tensors")
    n = x.numel()
    if y.numel() != n or out.numel() != n or s1.numel() != s0.numel() or n % s0.numel():
        raise ValueError("lincomb2: x {}, y {}, out {} must match and split into the {} items "
                         "of s0 / s1 ({})".format(n, y.numel(), out.numel(), s0.numel(), s1.numel()))
    _l.check(_l.load().dwm_b200_lincomb2(
        x.data_ptr(), y.data_ptr(), s0.data_ptr(), s1.data_ptr(), n, n // s0.numel(),
        out.data_ptr(), _stream()), "dwm_b200_lincomb2")
    return out


def cfg_dpmpp_step(pred, latents, x0_prev, row, *, cfg, guidance_scale=1.0):
    """Fused CFG combine + DPM-Solver++ (midpoint, order <= 2) step, in place on fp32 latents
    and the x0 history x0_prev (both n elements).  pred: fp32 [cfg * n], unconditional half
    first; row: fp32 [6] device tensor (c_x, c_m, k_s, k_0, k_1, order).  The CFG weights are
    fp32(1 - guidance_scale) and fp32(guidance_scale)."""
    for t, nme in ((pred, "pred"), (latents, "latents"), (x0_prev, "x0_prev"), (row, "row")):
        _f32(t, nme)
        if not t.is_contiguous():
            raise ValueError("cfg_dpmpp_step needs contiguous tensors")
    n = latents.numel()
    if cfg not in (1, 2) or pred.numel() != cfg * n or x0_prev.numel() != n or row.numel() != 6:
        raise ValueError("cfg_dpmpp_step: pred {} must be cfg ({}) x latents {}, x0_prev {} "
                         "match latents, row {} hold 6 values".format(
                             pred.numel(), cfg, n, x0_prev.numel(), row.numel()))
    g = float(guidance_scale)
    _l.check(_l.load().dwm_b200_cfg_dpmpp_step(
        pred.data_ptr(), cfg, 1.0 - g, g, n, row.data_ptr(), latents.data_ptr(),
        x0_prev.data_ptr(), _stream()), "dwm_b200_cfg_dpmpp_step")
    return latents
