"""Kernel time of the cross-view row-wise attention of a view shard at the DiT shape: local query
views against the gathered K,V of all views, on the wgmma kernel (separate K,V tensor map) and
on the mma.sync kernel, next to the unsharded launch.

  python tools/view_attention_bench.py [--bt 16] [--views 6] [--view-counts 3,3] [--out F]

Default shape: one CFG branch of the 16-frame north-star window (bt = 16), 6 views of a 16 x 28
patch grid, 24 heads of 64 (D = 1536), bf16, ring view mask.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def _device_info():
    """(card name, power limit) of GPU 0, read-only query."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def _time(fn, iters=50, warm=5, rounds=5):
    """Median over `rounds` of the mean ms per call over `iters` calls (CUDA events)."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / iters)
    return sorted(res)[len(res) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bt", type=int, default=16)
    ap.add_argument("--views", type=int, default=6)
    ap.add_argument("--hp", type=int, default=16)
    ap.add_argument("--wp", type=int, default=28)
    ap.add_argument("--heads", type=int, default=24)
    ap.add_argument("--view-counts", default="3,3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from opendwm_b200 import lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("view_attention_bench needs a CUDA device")
    BT, V, Hp, Wp, heads = args.bt, args.views, args.hp, args.wp, args.heads
    S, D, dt = Hp * Wp, heads * 64, torch.bfloat16
    counts = [int(c) for c in args.view_counts.split(",")]
    assert sum(counts) == V, "view counts must add up to --views"
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(BT * V * S, 3 * D, generator=g).to(dt).cuda()
    kv_all = qkv[:, D:].contiguous()
    i = torch.arange(V)
    d = (i.view(-1, 1) - i.view(1, -1)) % V
    mask = ((d == 0) | (d == 1) | (d == V - 1)).to(torch.uint8).expand(BT, V, V).contiguous().cuda()
    out = torch.empty(BT * V * S, D, dtype=dt, device="cuda")

    def unsharded():
        ops.attention(qkv, out, D=D, heads=heads, group_dims=[BT, Hp], group_strides=[V * S, Wp],
                      seq=V * Wp, inner=Wp, stride_outer=S, stride_inner=1, mask=mask, mask_div=1)

    V_loc, v_off = counts[0], 0
    q_loc = qkv.view(BT, V, S, 3 * D)[:, :V_loc, :, :D].reshape(-1, D).contiguous()
    o_loc = torch.empty(BT * V_loc * S, D, dtype=dt, device="cuda")

    def shard():
        ops.attention(q_loc, o_loc, D=D, heads=heads, group_dims=[BT, Hp],
                      group_strides=[V_loc * S, Wp], seq=V_loc * Wp, inner=Wp, stride_outer=S,
                      stride_inner=1, mask=mask, mask_div=1, mask_q_offset=v_off,
                      kv=kv_all, k_col=0, v_col=D, kv_group_strides=[V * S, Wp], seq_kv=V * Wp,
                      inner_kv=Wp, kv_stride_outer=S, kv_stride_inner=1)

    res = {"device": _device_info(), "dtype": "bf16",
           "shape": {"bt": BT, "views": V, "hp": Hp, "wp": Wp, "heads": heads,
                     "shard_views": V_loc}}
    try:
        for name, tc in (("wgmma", 1), ("mma_sync", 0)):
            lib.set_option("attn_tc", tc)
            res["unsharded_ms_" + name] = _time(unsharded)
            res["shard_ms_" + name] = _time(shard)
    finally:
        lib.set_option("attn_tc", -1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
