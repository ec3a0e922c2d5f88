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


def test_errors_without_gpu_are_loud():
    import pytest
    import torch
    from opendwm_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(a, a)
