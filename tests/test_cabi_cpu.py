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


def test_errors_without_gpu_are_loud():
    import pytest
    import torch
    from opendwm_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(a, a)
