"""The C-ABI shared library loads without a GPU and exports every entry point that
include/dwm_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    with open(os.path.join(ROOT, "include", "dwm_b200.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dwm_b200_\w+)\s*\(", text)))


def test_header_symbols_exported_and_bound():
    from opendwm_b200 import lib
    names = _declared()
    assert len(names) >= 10
    handle = lib.load()
    raw = ctypes.CDLL(lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), "library does not export " + n
        assert n in lib.SYMBOLS, "ctypes binding missing for " + n
        assert getattr(handle, n).restype is lib.SYMBOLS[n][0]
    assert set(lib.SYMBOLS) == set(names)
    assert b"sm_90a" in handle.dwm_b200_version()


def test_struct_layouts_match_header_field_order():
    from opendwm_b200 import lib
    with open(os.path.join(ROOT, "include", "dwm_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    for cname, st in (("dwm_linear_args", lib.LinearArgs),
                      ("dwm_attention_args", lib.AttentionArgs),
                      ("dwm_layernorm_args", lib.LayerNormArgs),
                      ("dwm_conv_args", lib.ConvArgs)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), text, re.S).group(1)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            names = decl.split(",")
            first = names[0].split()[-1]
            for n in [first] + [x.strip() for x in names[1:]]:
                fields.append(n.lstrip("*").split("[")[0])
        assert fields == [f[0] for f in st._fields_], cname


# Fake, 16-byte aligned device addresses: without a CUDA device a call that passes every
# argument check stops at tensor-map encoding, so nothing is ever dereferenced or launched.
_BASE = 1 << 32


def _addr(i, misalign=0):
    return _BASE + i * (1 << 24) + misalign


def _linear_args(**kw):
    """A well-formed RESID call (gate, blend, per-item rows) and the fields in `kw`."""
    from opendwm_b200 import lib
    a = lib.LinearArgs()
    a.M, a.N, a.K = 512, 256, 64
    a.A, a.lda, a.W, a.ldw = _addr(0), 64, _addr(1), 64
    a.bias, a.dtype, a.out_dtype = _addr(2), lib.DWM_BF16, lib.DWM_BF16
    a.epilogue, a.out, a.ldo = lib.EPI_RESID, _addr(3), 256
    a.rows_per_item = 128
    a.resid, a.ldr = _addr(4), 256
    a.gate, a.gate_ld = _addr(5), 1536
    a.blend_x, a.ldx, a.alpha, a.rows_per_batch = _addr(6), 260, _addr(7), 256
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _conv_args(**kw):
    from opendwm_b200 import lib
    a = lib.ConvArgs()
    a.x, a.nb, a.tp, a.h, a.w, a.c_in = _addr(0), 2, 3, 8, 14, 64
    a.weight, a.kt, a.kh, a.kw, a.c_out = _addr(1), 1, 3, 3, 128
    a.bias, a.dtype, a.epilogue = _addr(2), lib.DWM_BF16, lib.EPI_RESID
    a.out, a.ldo = _addr(3), 128
    a.resid, a.ldr, a.resid_per_item, a.rows_per_item = _addr(4), 132, 1, 8 * 14
    a.blend_x, a.ldx, a.alpha, a.rows_per_batch = _addr(5), 128, _addr(6), 3 * 8 * 14
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(fn, args):
    import ctypes
    from opendwm_b200 import lib
    rc = getattr(lib.load(), fn)(ctypes.byref(args), None)
    return rc, lib.load().dwm_b200_last_error().decode()


def _no_device():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible: these calls use fake device addresses")


def _linear_breaks():
    from opendwm_b200 import lib
    peers = (ctypes.c_void_p * 8)(_addr(8), _addr(9, 8))
    return [
        ("bias+4", dict(bias=_addr(2, 4)), "16-byte aligned"),
        ("bias+8 STORE", dict(bias=_addr(2, 8), epilogue=lib.EPI_STORE, resid=None, gate=None,
                              blend_x=None, rows_per_item=0), "16-byte aligned"),
        ("resid+4", dict(resid=_addr(4, 4)), "16-byte aligned"),
        ("gate+8", dict(gate=_addr(5, 8)), "16-byte aligned"),
        ("blend_x+12", dict(blend_x=_addr(6, 12)), "16-byte aligned"),
        ("ldr 257", dict(ldr=257), "multiples of 4"),
        ("gate_ld 1538", dict(gate_ld=1538), "multiples of 4"),
        ("ldx 258", dict(ldx=258), "multiples of 4"),
        ("peer_out[1]+8", dict(epilogue=lib.EPI_STORE, resid=None, gate=None, blend_x=None,
                               rows_per_item=0, peer_out=peers, n_peer_out=2), "peer_out\\[1\\]"),
        ("STORE items collapse", dict(epilogue=lib.EPI_STORE, resid=None, gate=None, blend_x=None,
                                      out_item_stride=0), "out_item_stride 0 < rows_per_item 128"),
        ("QKNORM items overlap", dict(epilogue=lib.EPI_QKNORM, resid=None, gate=None, blend_x=None,
                                      q_norm_weight=_addr(10), k_norm_weight=_addr(11),
                                      qk_region=64, out_item_stride=127),
         "out_item_stride 127 < rows_per_item 128"),
    ]


def _conv_breaks():
    from opendwm_b200 import lib
    no_resid = dict(resid=None, resid_per_item=0, rows_per_item=0, blend_x=None, alpha=None)
    return [
        ("bias+4", dict(bias=_addr(2, 4)), "16-byte aligned"),
        ("resid+8", dict(resid=_addr(4, 8)), "16-byte aligned"),
        ("blend_x+4", dict(blend_x=_addr(5, 4)), "16-byte aligned"),
        ("ldr 130", dict(ldr=130), "multiples of 4"),
        ("ldx 129", dict(ldx=129), "multiples of 4"),
        ("STORE with resid", dict(epilogue=lib.EPI_STORE), "need epilogue DWM_EPI_RESID"),
        ("F32 with blend_x", dict(no_resid, epilogue=lib.EPI_F32, blend_x=_addr(5), alpha=_addr(6)),
         "need epilogue DWM_EPI_RESID"),
        ("STORE resid_per_item", dict(no_resid, epilogue=lib.EPI_STORE, resid_per_item=1,
                                      rows_per_item=112), "need epilogue DWM_EPI_RESID"),
        ("blend_x without alpha", dict(alpha=None), "blend_x without alpha"),
        ("resid_per_item without rows", dict(rows_per_item=0), "resid_per_item needs rows_per_item"),
    ]


def test_linear_argument_checks():
    """dwm_b200_linear rejects every misaligned fp32 operand, every fp32 pitch that is not whole
    16-byte rows and every row remap that folds items onto each other; each call breaks one
    rule of an otherwise well-formed call, which itself passes every check."""
    import pytest
    _no_device()
    rc, msg = _call("dwm_b200_linear", _linear_args())
    assert rc < 0 and "cuTensorMapEncodeTiled" in msg, msg
    failed = []
    for name, kw, want in _linear_breaks():
        rc, msg = _call("dwm_b200_linear", _linear_args(**kw))
        if not (rc < 0 and re.search(want, msg)):
            failed.append((name, rc, msg))
    if failed:
        pytest.fail("accepted or wrong message: %r" % failed)


def test_conv_argument_checks():
    """dwm_b200_conv: the same alignment and pitch rules, and residual / blend operands only with
    the RESID epilogue (a 16-bit store given rows_per_item would write every item onto the
    first item's rows)."""
    import pytest
    _no_device()
    rc, msg = _call("dwm_b200_conv", _conv_args())
    assert rc < 0 and "cuTensorMapEncodeTiled" in msg, msg
    failed = []
    for name, kw, want in _conv_breaks():
        rc, msg = _call("dwm_b200_conv", _conv_args(**kw))
        if not (rc < 0 and re.search(want, msg)):
            failed.append((name, rc, msg))
    if failed:
        pytest.fail("accepted or wrong message: %r" % failed)


def _ln_args(**kw):
    """A well-formed BF16 LayerNorm with every optional operand (resident kernel: M < 4096)."""
    from opendwm_b200 import lib
    a = lib.LayerNormArgs()
    a.M, a.D, a.x, a.ldx = 64, 256, _addr(0), 260
    a.add_item, a.add_item_ld, a.rows_per_item = _addr(1), 256, 16
    a.add_full, a.add_full_ld = _addr(2), 264
    a.sum_out, a.ld_sum = _addr(3), 256
    a.weight, a.bias, a.eps = _addr(4), _addr(5), 1e-6
    a.shift, a.scale, a.shift2, a.scale2, a.mod_ld = _addr(6), _addr(7), _addr(8), _addr(9), 1536
    a.out, a.ldo, a.out2, a.ldo2, a.dtype = _addr(10), 256, _addr(11), 260, lib.DWM_BF16
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _ln_breaks():
    from opendwm_b200 import lib
    e4m3 = dict(dtype=lib.DWM_E4M3, out_scale=_addr(12), out2_scale=_addr(13))
    out = [("%s+%d" % (f, m), {f: _addr(i, m)}, "16-byte aligned")
           for i, (f, m) in enumerate((("x", 4), ("add_item", 8), ("add_full", 4), ("sum_out", 12),
                                       ("weight", 4), ("bias", 8), ("shift", 4), ("scale", 8),
                                       ("shift2", 12), ("scale2", 4)))]
    out += [
        ("add_item_ld 258", dict(add_item_ld=258), "multiples of 4"),
        ("add_full_ld 262", dict(add_full_ld=262), "multiples of 4"),
        ("ld_sum 257", dict(ld_sum=257), "multiples of 4"),
        ("ldo2 258 bf16", dict(ldo2=258), "multiples of 4"),
        ("ldo2 258 e4m3", dict(e4m3, ldo2=258), "multiples of 4"),
        ("out+4 bf16", dict(out=_addr(10, 4)), "8-byte aligned"),
        ("out2+2 bf16", dict(out2=_addr(11, 2)), "8-byte aligned"),
        ("out+2 e4m3", dict(e4m3, out=_addr(10, 2)), "4-byte aligned"),
    ]
    return out


def _fn(name, *args):
    from opendwm_b200 import lib
    rc = getattr(lib.load(), name)(*args)
    return rc, lib.load().dwm_b200_last_error().decode()


def _rowop_calls():
    """(entry point, well-formed arguments, [(label, {argument index: value}, message)])."""
    from opendwm_b200 import lib
    A = _addr
    gn = [A(0), 2, 3, 4, 6, 64, 16]   # x, nb, T, H, W, C, groups
    ep = [A(2), A(3)]                 # gamma, beta
    return [
        ("dwm_b200_act_cast", [A(0), A(1), 1001, lib.ACT_SILU, lib.DWM_BF16, None], [
            ("relu", {3: lib.ACT_RELU}, "not implemented"),
            ("act 9", {3: 9}, "not implemented"),
            ("in+8", {0: A(0, 8)}, "aligned"),
            ("out+4", {1: A(1, 4)}, "aligned")]),
        ("dwm_b200_axpy", [A(0), A(1), 1001, 0.5, None], [
            ("x+4", {0: A(0, 4)}, "16-byte aligned"),
            ("y+8", {1: A(1, 8)}, "16-byte aligned")]),
        ("dwm_b200_upsample_nearest", [A(0), 2, 3, 4, 6, 64, 1, A(1), lib.DWM_BF16, None], [
            ("x+8", {0: A(0, 8)}, "aligned"),
            ("out+4", {7: A(1, 4)}, "aligned")]),
        ("dwm_b200_groupnorm_stats", [A(0), 2, 72, 64, 16, A(1), None], [
            ("x+4", {0: A(0, 4)}, "aligned"),
            ("sums+4", {5: A(1, 4)}, "aligned")]),
        ("dwm_b200_spatialnorm_silu",
         gn + [A(1), 1e-6] + ep + [A(4), A(5), 2, 2, 3, 1, A(6), 5, 1, lib.DWM_BF16, None], [
             ("x+4", {0: A(0, 4)}, "aligned"), ("sums+4", {7: A(1, 4)}, "aligned"),
             ("gamma+8", {9: A(2, 8)}, "aligned"), ("beta+4", {10: A(3, 4)}, "aligned"),
             ("zy+4", {11: A(4, 4)}, "aligned"), ("zb+12", {12: A(5, 12)}, "aligned"),
             ("out+4", {17: A(6, 4)}, "aligned")]),
        ("dwm_b200_groupnorm_silu_e4m3",
         gn + [A(1), 1e-6] + ep + [1, A(6), 5, 1, A(7), None], [
             ("x+4", {0: A(0, 4)}, "aligned"), ("gamma+4", {9: A(2, 4)}, "aligned"),
             ("out+2", {12: A(6, 2)}, "aligned")]),
        ("dwm_b200_groupnorm_silu_halo",
         gn + [A(1), 6, 1e-6] + ep + [1, A(6), A(7), 5, A(8), 5, lib.DWM_BF16, None], [
             ("x+4", {0: A(0, 4)}, "aligned"), ("beta+8", {11: A(3, 8)}, "aligned"),
             ("out+4", {13: A(6, 4)}, "aligned"), ("prev_out+4", {14: A(7, 4)}, "aligned"),
             ("next_out+2", {16: A(8, 2)}, "aligned")]),
        ("dwm_b200_groupnorm_silu_e4m3_amax",
         gn + [A(1), 6, 1e-6] + ep + [1, A(6), None], [
             ("x+4", {0: A(0, 4)}, "aligned"), ("sums+4", {7: A(1, 4)}, "aligned")]),
        ("dwm_b200_groupnorm_silu_e4m3_halo",
         gn + [A(1), 6, 1e-6] + ep + [1, A(5), A(6), A(7), 5, A(8), 5, A(9), None], [
             ("gamma+4", {10: A(2, 4)}, "aligned"), ("out+2", {14: A(6, 2)}, "aligned"),
             ("next_out+1", {17: A(8, 1)}, "aligned")]),
    ]


def test_layernorm_argument_checks():
    """dwm_b200_layernorm reads every fp32 operand as float4 and stores four outputs at a time:
    it rejects each misaligned operand and pitch.  A misaligned x used to reach the resident
    kernel as misaligned float4 loads."""
    import pytest
    _no_device()
    rc, msg = _call("dwm_b200_layernorm", _ln_args())
    assert rc < 0 and "cudaGetLastError" in msg, msg
    failed = []
    for name, kw, want in _ln_breaks():
        rc, msg = _call("dwm_b200_layernorm", _ln_args(**kw))
        if not (rc == -1 and re.search(want, msg)):
            failed.append((name, rc, msg))
    if failed:
        pytest.fail("accepted or wrong message: %r" % failed)


def test_rowop_and_groupnorm_argument_checks():
    """act_cast, axpy, upsample_nearest and the GroupNorm entry points reject misaligned
    operands (one broken argument per call), and act_cast an activation it does not implement
    (ReLU used to return its input unchanged).  Each well-formed call passes every check and
    fails only at its first CUDA call."""
    import pytest
    _no_device()
    failed = []
    for fn, args, breaks in _rowop_calls():
        rc, msg = _fn(fn, *args)
        assert rc == -2 and "failed:" in msg, (fn, msg)
        for name, change, want in breaks:
            bad = list(args)
            for i, v in change.items():
                bad[i] = v
            rc, msg = _fn(fn, *bad)
            if not (rc == -1 and re.search(want, msg)):
                failed.append((fn, name, rc, msg))
    if failed:
        pytest.fail("accepted or wrong message: %r" % failed)


def test_errors_without_gpu_are_loud():
    import pytest
    import torch
    from opendwm_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(a, a)
