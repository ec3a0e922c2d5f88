"""dwm_b200_cfg_dpmpp_step (fused CFG + DPM-Solver++ step) rejects malformed arguments before it
launches anything: each call breaks one rule of a well-formed call, which itself passes every
check and fails only at its first CUDA call (no device here)."""
import re

import pytest

from test_cabi_cpu import _addr, _fn, _no_device

N = 1001          # not a multiple of 4 or 256


def _args():
    # pred [2N], cfg, w_uncond, w_cond, n, row [6], latents [N], x0_prev [N], stream
    return [_addr(0), 2, -2.0, 3.0, N, _addr(1), _addr(2), _addr(3), None]


BREAKS = [
    ("null pred", {0: None}, "null"),
    ("null row", {5: None}, "null"),
    ("null latents", {6: None}, "null"),
    ("null x0_prev", {7: None}, "null"),
    ("cfg 0", {1: 0}, "cfg must be 1 or 2"),
    ("cfg 3", {1: 3}, "cfg must be 1 or 2"),
    ("n 0", {4: 0}, "bad n"),
    ("n -5", {4: -5}, "bad n"),
    ("n beyond the grid", {4: 1 << 40}, "bad n"),
    ("pred+2", {0: _addr(0, 2)}, "4-byte aligned"),
    ("row+1", {5: _addr(1, 1)}, "4-byte aligned"),
    ("latents+2", {6: _addr(2, 2)}, "4-byte aligned"),
    ("x0_prev+3", {7: _addr(3, 3)}, "4-byte aligned"),
    ("x0_prev on latents", {7: _addr(2, 4 * (N - 1))}, "must not overlap"),
    ("latents in pred's cond half", {6: _addr(0, 4 * N)}, "must not overlap"),
    ("x0_prev in pred", {7: _addr(0, 4 * 7)}, "must not overlap"),
    ("row in x0_prev", {5: _addr(3, 4 * (N - 2))}, "must not overlap"),
]


def test_cfg_dpmpp_step_argument_checks():
    _no_device()
    rc, msg = _fn("dwm_b200_cfg_dpmpp_step", *_args())
    assert rc == -2 and "failed:" in msg, msg
    # cfg 1 reads only n prediction values: a latents buffer right after them is fine
    ok = _args()
    ok[1], ok[6] = 1, _addr(0, 4 * N)
    rc, msg = _fn("dwm_b200_cfg_dpmpp_step", *ok)
    assert rc == -2 and "failed:" in msg, msg
    failed = []
    for name, change, want in BREAKS:
        bad = _args()
        for i, v in change.items():
            bad[i] = v
        rc, msg = _fn("dwm_b200_cfg_dpmpp_step", *bad)
        if not (rc == -1 and re.search(want, msg)):
            failed.append((name, rc, msg))
    if failed:
        pytest.fail("accepted or wrong message: %r" % failed)
