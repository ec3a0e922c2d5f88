"""Frame-shard GroupNorm(+SiLU) kernels of the temporal ResBlock, on one GPU.

The "neighbour" operands are tensors on the same device.  For the same window-wide statistics,
every shard's operand [nb, T_loc + 2, H, W, C] (its frames plus the halo frames its neighbours
store into it, zero at the window's ends) equals frames [t_offset, t_offset + T_loc + 2) of the
unsharded operand [nb, T + 2, H, W, C] bit for bit: 16-bit (fp16, bf16) and E4M3 (split amax /
quantize passes against dwm_b200_groupnorm_silu_e4m3, bytes and scales).  The (3,1,1)
convolution over a shard's operand gives the unsharded convolution's rows of those frames."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _counts(T, shards):
    q, r = divmod(T, shards)
    return [q + (1 if i < r else 0) for i in range(shards)]


def _case(T, C, nb=3, H=4, W=6, seed=0):
    from opendwm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(nb, T, H, W, C, device="cuda", generator=g) * 1.5 + 0.3
    gamma = 1 + 0.1 * torch.randn(C, device="cuda", generator=g)
    beta = 0.1 * torch.randn(C, device="cuda", generator=g)
    return x, ops.groupnorm_stats(x, 32), gamma, beta


def _shard_operands(T, shards, x, dtype):
    """Per shard: (local x, operand filled with a non-zero byte pattern, t_offset)."""
    nb, _, H, W, C = x.shape
    out, off = [], 0
    for n in _counts(T, shards):
        buf = torch.full((nb, n + 2, H, W, C * dtype.itemsize), 0x5A, device="cuda",
                         dtype=torch.uint8)
        out.append((x[:, off:off + n].contiguous(), buf.view(dtype), off))
        off += n
    return out


CASES = [(8, 2), (5, 4), (7, 3), (11, 4), (4, 1)]
IDS = ["8_over_2", "5_over_4_uneven", "7_over_3_uneven", "11_over_4_uneven", "one_shard"]


@pytest.mark.parametrize("C", [64, 320])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("T,shards", CASES, ids=IDS)
def test_halo_norm_equals_unsharded(T, shards, dtype, C):
    from opendwm_b200 import ops
    x, sums, gamma, beta = _case(T, C)
    nb, _, H, W, _ = x.shape
    ref = torch.zeros(nb, T + 2, H, W, C, device="cuda", dtype=dtype)
    ops.spatialnorm_silu(x, sums, gamma, beta, ref, groups=32, eps=1e-5, out_t0=1, silu=True)
    parts = _shard_operands(T, shards, x, dtype)
    for r, (xl, buf, _) in enumerate(parts):
        ops.groupnorm_silu_halo(
            xl, sums, gamma, beta, buf, groups=32, stat_frames=T, eps=1e-5,
            prev_out=parts[r - 1][1] if r > 0 else None,
            next_out=parts[r + 1][1] if r + 1 < shards else None)
    for r, (xl, buf, off) in enumerate(parts):
        want = ref[:, off:off + xl.shape[1] + 2]
        assert torch.equal(buf.view(torch.int16), want.contiguous().view(torch.int16)), r


@pytest.mark.parametrize("T,shards", CASES, ids=IDS)
def test_halo_norm_e4m3_equals_unsharded(T, shards):
    from opendwm_b200 import ops
    x, sums, gamma, beta = _case(T, 320, seed=1)
    nb, _, H, W, C = x.shape
    fp8 = torch.float8_e4m3fn
    ref = torch.zeros(nb, T + 2, H, W, C, device="cuda", dtype=fp8)
    ref_s = torch.empty(nb, device="cuda")
    ops.groupnorm_silu_e4m3(x, sums, gamma, beta, ref, ref_s, groups=32, eps=1e-5, out_t0=1)
    parts = _shard_operands(T, shards, x, fp8)
    amax = torch.stack([ops.groupnorm_silu_e4m3_amax(
        xl, sums, gamma, beta, torch.empty(nb, device="cuda"), groups=32, stat_frames=T,
        eps=1e-5) for xl, _, _ in parts]).amax(0)        # the frame group's all-reduce MAX
    for r, (xl, buf, _) in enumerate(parts):
        scale = torch.full((nb,), -1.0, device="cuda")
        ops.groupnorm_silu_e4m3_halo(
            xl, sums, gamma, beta, amax, buf, scale, groups=32, stat_frames=T, eps=1e-5,
            prev_out=parts[r - 1][1] if r > 0 else None,
            next_out=parts[r + 1][1] if r + 1 < shards else None)
        assert torch.equal(scale, ref_s), r
    for r, (xl, buf, off) in enumerate(parts):
        want = ref[:, off:off + xl.shape[1] + 2]
        assert torch.equal(buf.view(torch.uint8), want.contiguous().view(torch.uint8)), r


@pytest.mark.parametrize("T,shards", CASES, ids=IDS)
def test_temporal_conv_over_halo_operand(T, shards):
    """The conv reads the same operand bytes in the same tap and channel order for a frame
    whether the operand holds the window or a shard; the rows must agree bit for bit."""
    from opendwm_b200 import ops
    dtype, C, Co = torch.float16, 320, 320
    x, sums, gamma, beta = _case(T, C, seed=2)
    nb, _, H, W, _ = x.shape
    g = torch.Generator(device="cuda").manual_seed(3)
    w = (torch.randn(3, Co, C, device="cuda", generator=g) / C ** 0.5).to(dtype).contiguous()
    ref = torch.zeros(nb, T + 2, H, W, C, device="cuda", dtype=dtype)
    ops.spatialnorm_silu(x, sums, gamma, beta, ref, groups=32, eps=1e-5, out_t0=1, silu=True)
    want = ops.conv(ref, w, kernel=(3, 1, 1)).view(nb, T, H * W, Co)
    parts = _shard_operands(T, shards, x, dtype)
    for r, (xl, buf, _) in enumerate(parts):
        ops.groupnorm_silu_halo(
            xl, sums, gamma, beta, buf, groups=32, stat_frames=T, eps=1e-5,
            prev_out=parts[r - 1][1] if r > 0 else None,
            next_out=parts[r + 1][1] if r + 1 < shards else None)
    for r, (xl, buf, off) in enumerate(parts):
        n = xl.shape[1]
        got = ops.conv(buf, w, kernel=(3, 1, 1)).view(nb, n, H * W, Co)
        assert torch.equal(got, want[:, off:off + n]), \
            (r, (got - want[:, off:off + n]).abs().max().item())


def test_halo_norm_rejects_bad_operands():
    from opendwm_b200 import ops
    x, sums, gamma, beta = _case(4, 64)
    nb, T, H, W, C = x.shape
    with pytest.raises(ValueError, match="T \\+ 2"):
        ops.groupnorm_silu_halo(x, sums, gamma, beta,
                                torch.empty(nb, T, H, W, C, device="cuda", dtype=torch.float16),
                                groups=32, stat_frames=T)
    with pytest.raises(RuntimeError, match="stat_frames"):
        ops.groupnorm_silu_halo(x, sums, gamma, beta,
                                torch.empty(nb, T + 2, H, W, C, device="cuda",
                                            dtype=torch.float16),
                                groups=32, stat_frames=T - 1)
