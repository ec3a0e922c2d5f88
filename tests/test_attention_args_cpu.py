"""Argument checks of dwm_b200_attention for the view-sharded cross-view call (local query views
with a mask row offset, separate gathered K,V), without a GPU: fake 16-byte aligned device
addresses, so a call that passes every check stops at its first CUDA call and nothing is
dereferenced or launched."""
import ctypes
import re

import pytest
import torch

_BASE = 1 << 32


def _addr(i, misalign=0):
    return _BASE + i * (1 << 24) + misalign


def _crossview_args(**kw):
    """View shard 2 of 6 views (V_loc = 2 from v_offset 2) of the DiT cross-view row-wise
    call: groups (b t, h), query units of Wp = 28 tokens, K,V of all six views."""
    from opendwm_b200 import lib
    B, V, V_loc, Hp, Wp, D = 2, 6, 2, 16, 28, 128
    S = Hp * Wp
    a = lib.AttentionArgs()
    a.qkv, a.ld, a.D, a.heads, a.head_dim, a.dtype = _addr(0), D, D, 2, 64, lib.DWM_BF16
    a.group_dims[0], a.group_dims[1], a.group_dims[2] = B, Hp, 1
    a.group_strides[0], a.group_strides[1] = V_loc * S, Wp
    a.out_group_strides[0], a.out_group_strides[1] = V_loc * S, Wp
    a.seq, a.inner, a.stride_outer, a.stride_inner = V_loc * Wp, Wp, S, 1
    a.out, a.ldo, a.out_stride_outer, a.out_stride_inner = _addr(1), D, S, 1
    a.mask, a.mask_div, a.n_outer, a.mask_q_offset = _addr(2), 1, V, 2
    a.scale = 0.125
    a.kv, a.ld_kv, a.k_col, a.v_col = _addr(3), 2 * D, 0, D
    a.kv_group_strides[0], a.kv_group_strides[1] = V * S, Wp
    a.seq_kv, a.inner_kv, a.kv_stride_outer, a.kv_stride_inner = V * Wp, Wp, S, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(args):
    from opendwm_b200 import lib
    rc = lib.load().dwm_b200_attention(ctypes.byref(args), None)
    return rc, lib.load().dwm_b200_last_error().decode()


BREAKS = [
    ("offset past the mask", dict(mask_q_offset=5), "outside the 6 mask rows"),
    ("last unit past the mask", dict(mask_q_offset=4, seq=3 * 28), "outside the 6 mask rows"),
    ("negative offset", dict(mask_q_offset=-1), "mask_q_offset must be >= 0"),
    ("negative offset, no mask", dict(mask_q_offset=-1, mask=None), "mask_q_offset must be >= 0"),
    ("kv + 8 bytes", dict(kv=_addr(3, 8)), "bad separate kv description"),
    ("ld_kv not whole 16 bytes", dict(ld_kv=2 * 128 + 4), "bad separate kv description"),
    ("k_col not whole 16 bytes", dict(k_col=4), "bad separate kv description"),
    ("v_col not whole 16 bytes", dict(v_col=128 + 2), "bad separate kv description"),
]


def test_view_shard_attention_argument_checks():
    """Each call breaks one rule of the well-formed view-shard call, which itself passes every
    check (with the wgmma kernel and with the mma.sync kernel) and fails only at its first CUDA
    call."""
    from opendwm_b200 import lib
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible: these calls use fake device addresses")
    rejections = "|".join(want for _, _, want in BREAKS)
    try:
        for tc in (1, 0):
            lib.set_option("attn_tc", tc)
            rc, msg = _call(_crossview_args())
            assert rc != 0 and not re.search(rejections, msg), (tc, msg)
            rc, msg = _call(_crossview_args(mask_q_offset=4))     # the last view shard 4, 5
            assert rc != 0 and not re.search(rejections, msg), (tc, msg)
            failed = []
            for name, kw, want in BREAKS:
                rc, msg = _call(_crossview_args(**kw))
                if not (rc < 0 and re.search(want, msg)):
                    failed.append((name, rc, msg))
            assert not failed, "accepted or wrong message: %r" % failed
    finally:
        lib.set_option("attn_tc", -1)


def test_mask_q_offset_is_the_last_field():
    """Appended at the end: callers that zero-initialise the struct keep the unsharded meaning."""
    from opendwm_b200 import lib
    assert lib.AttentionArgs._fields_[-1] == ("mask_q_offset", ctypes.c_int)
    assert lib.AttentionArgs().mask_q_offset == 0
