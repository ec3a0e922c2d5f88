"""The GEMM's TMA-stored 16-bit outputs against float64, and the elements they must not write.

A 16-bit epilogue (STORE, GEGLU, QKNORM, QuickGELU STORE, GEGLU_TANH) without peer outputs
stores its tile from shared memory by TMA, through a tensor map of the output's row layout:
[items, rows_per_item, N] at out_row_offset with item pitch out_item_stride (TmaOut in
gemm_epilogue.cuh).  TMA clips each 64 x 64 box to the item of its first row and to N; the
box's rows in later items, or in a partial last item, are copied by the consumer threads.
Every case here:

  * writes into views of sentinel-filled buffers (test_gemm_conformance_gpu's guard rows and
    columns past N up to ldo): every element outside the result rows x [0, N) (the gap rows of
    a remapped layout, the rows past M) must keep its sentinel bits, every element inside must
    be within the float64 bound of the conformance tests;
  * repeats the call with two peer outputs, which the kernel stores from registers: the same
    bits, so the two store paths round nothing differently;
  * runs every kernel variant the options reach (gemm_2cta x gemm_bn): the same bits.
"""
import pytest
import torch

from test_gemm_conformance_gpu import (
    GEGLU, GEGLU_TANH, GUARD, NONE, QKNORM, QUICK_GELU, SILU, STORE, Epi, _bits, _Options, _sms,
    big_scale, check_output, epilogue_reference, linear_kernel, make_operands, padded_vec,
    poisoned_2d, sentinel_buffer)
from test_fp8_conformance_gpu import _linear_case, _reference

S, L = 448, 154          # the step's sample and context rows per item in the joint q|k|v buffer
D = 1536                 # the step's model width: QKNORM regions, GEGLU's output width 4 D


def _case(name, M, N, K, kind, act=NONE, rpi=0, stride=0, offset=0, out_rows=0, regions=2):
    return (name, dict(M=M, N=N, K=K, kind=kind, act=act, rpi=rpi, stride=stride, offset=offset,
                       out_rows=out_rows, regions=regions))


# (name, call); a list of calls writes one buffer together (the joint q|k|v layout)
CASES = [
    # no items: M not a multiple of 64 (nor of the 128-row tile), N % 64 = 32 and N < one tile
    ("store_M130_N96", [_case("", 130, 96, 80, STORE, act=SILU)]),
    ("store_M1000_N160", [_case("", 1000, 160, 144, STORE)]),
    # items of 100 rows at pitch 130: boundaries inside 64-row boxes, a partial last item of
    # 50 rows (also M not a multiple of 64), a nonzero offset
    ("store_remap_tail_M250_N160", [_case("", 250, 160, 80, STORE, rpi=100, stride=130, offset=7)]),
    ("store_remap_M600_N96_pair", [_case("", 600, 96, 80, STORE, rpi=100, stride=130, offset=3)]),
    # items shorter than a box: one 64-row box spans up to four items
    ("store_remap_short_M100_N96", [_case("", 100, 96, 80, STORE, rpi=20, stride=33, offset=5)]),
    # the step's joint q|k|v buffer, two items: sample rows at 0, context rows at S, pitch S + L
    ("qknorm_joint_step", [
        _case("sample", 2 * S, 3 * D, 80, QKNORM, rpi=S, stride=S + L, offset=0, out_rows=2 * (S + L)),
        _case("context", 2 * L, 3 * D, 80, QKNORM, rpi=L, stride=S + L, offset=S, out_rows=2 * (S + L))]),
    ("store_joint_step", [
        _case("sample", 2 * S, 3 * D, 80, STORE, rpi=S, stride=S + L, offset=0, out_rows=2 * (S + L)),
        _case("context", 2 * L, 3 * D, 80, STORE, rpi=L, stride=S + L, offset=S, out_rows=2 * (S + L))]),
    # FF1 at the step's width (output 4 D), an odd number of 128-row tiles
    ("geglu_step_M600", [_case("", 600, 8 * D, 80, GEGLU)]),
    ("geglu_remap_M300", [_case("", 300, 768, 80, GEGLU, rpi=100, stride=110, offset=3)]),
    ("quick_gelu_remap_M301", [_case("", 301, 352, 80, STORE, act=QUICK_GELU, rpi=77, stride=90, offset=4)]),
    ("geglu_tanh_M616", [_case("", 616, 1536, 144, GEGLU_TANH)]),
]
FP8_CASES = [c for c in CASES if c[0] in ("store_remap_tail_M250_N160", "store_M1000_N160",
                                          "qknorm_joint_step", "geglu_step_M600")]


def _epi(c, g):
    e = Epi(c["kind"], act=c["act"], rows_per_item=c["rpi"], out_item_stride=c["stride"],
            out_row_offset=c["offset"])
    e.bias = padded_vec(torch.randn(c["N"], generator=g) * 0.5)
    if c["kind"] == QKNORM:
        e.qw = (torch.randn(64, generator=g) * 0.2 + 1).cuda()
        e.kw = (torch.randn(64, generator=g) * 0.2 + 1).cuda()
        e.qk_region, e.regions = D, c["regions"]
    return e


def _inputs(calls, dtype, fp8):
    """[(operands, Epi, (ref, tol))] of each call; operands are (A, W) or (A8, W8, sa, sw)."""
    out = []
    for i, c in enumerate(calls):
        M, N, K, kind = c["M"], c["N"], c["K"], c["kind"]
        if fp8:
            opt = dict(bias=True, act=c["act"], rows_per_item=c["rpi"], out_item_stride=c["stride"],
                       out_row_offset=c["offset"], qk_region=D, regions=c["regions"])
            op, e = _linear_case(M, N, K, kind, opt, dtype, seed=M + N + i, qk_seed=i)
            out.append((op.cuda(), e, _reference(op, e, dtype)))
            continue
        e = _epi(c, torch.Generator().manual_seed(M + N + K + i))
        a, w = make_operands(M, N, K, dtype, big_scale(dtype, True), seed=M * 7 + N + K + i)
        A, W = poisoned_2d(a), poisoned_2d(w)
        z = A.double() @ W.double().T
        P = A.double().abs() @ W.double().abs().T
        out.append(((A, W), e, epilogue_reference(z, P, K, e, dtype)))
    return out


def _launch(inputs, rows, cols, dtype, peers=False, gemm_2cta=1, gemm_bn=0):
    """Runs the calls into one fresh sentinel buffer (and two peers: the register store path);
    returns the buffer."""
    from opendwm_b200 import ops
    bufs = [sentinel_buffer(rows, cols, dtype) for _ in range(3 if peers else 1)]
    view = lambda b: b[GUARD:GUARD + rows, :cols]  # noqa: E731
    with _Options(gemm_2cta=gemm_2cta, gemm_bn=gemm_bn):
        for ops_, e, _ in inputs:
            A, W = ops_[0], ops_[1]
            kw = dict(a_scale=ops_[2], w_scale=ops_[3], out_dtype=dtype) if len(ops_) == 4 else {}
            ops.linear(A, W, e.bias, epilogue=e.kind, act=e.act, out=view(bufs[0]),
                       rows_per_item=e.rows_per_item, out_item_stride=e.out_item_stride,
                       out_row_offset=e.out_row_offset, q_norm_weight=e.qw, k_norm_weight=e.kw,
                       qk_region=e.qk_region, eps=e.eps, qk_norm_regions=e.regions if e.kind == QKNORM else 0,
                       peer_out=[view(b).data_ptr() for b in bufs[1:]] or None, **kw)
        torch.cuda.synchronize()
    for p in bufs[1:]:
        assert torch.equal(_bits(p), _bits(bufs[0])), "a peer output differs from out"
    return bufs[0]


def _check(name, calls, dtype, fp8=False):
    inputs = _inputs(calls, dtype, fp8)
    es = [e for _, e, _ in inputs]
    Ms = [c["M"] for c in calls]
    rows = max([c["out_rows"] for c in calls] + [int(e.out_rows(M).max()) + 1 for e, M in zip(es, Ms)])
    cols = es[0].out_cols(calls[0]["N"])
    out = _launch(inputs, rows, cols, dtype)
    check_output(out, torch.cat([e.out_rows(M) for e, M in zip(es, Ms)]), cols,
                 torch.cat([r for _, _, (r, _) in inputs]), torch.cat([t for _, _, (_, t) in inputs]), name)
    assert torch.equal(_bits(_launch(inputs, rows, cols, dtype, peers=True)), _bits(out)), \
        "%s: the register store path gave other bits" % name
    sms = _sms()
    key = lambda two, bn: tuple(linear_kernel(c["M"], c["N"], c["kind"], sms, two, bn) for c in calls)  # noqa: E731
    seen = {key(1, 0)}
    for two in (1, 0):
        for bn in (128, 256):
            if key(two, bn) not in seen:
                seen.add(key(two, bn))
                assert torch.equal(_bits(_launch(inputs, rows, cols, dtype, False, two, bn)), _bits(out)), \
                    "%s: gemm_2cta %d gemm_bn %d gave other bits" % (name, two, bn)


DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,calls", CASES, ids=[c[0] for c in CASES])
def test_tma_store_conforms(name, calls, dtype):
    _check(name, [c for _, c in calls], dtype)


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name,calls", FP8_CASES, ids=[c[0] for c in FP8_CASES])
def test_tma_store_conforms_e4m3(name, calls, dtype):
    """E4M3 operands; `dtype` is out_dtype."""
    _check(name, [c for _, c in calls], dtype, fp8=True)
