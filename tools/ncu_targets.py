"""Launches ONE instance of every hot kernel at its north-star (or VAE / UNet) shape so that a
single `ncu --set full` capture covers them:

  ncu --set full --clock-control none --import-source on -o kernels \\
      -k regex:"gemm|attn|layernorm|conv_wgmma|gn_stats|spatialnorm" python tools/ncu_targets.py

Each op runs once un-profiled first (lazy attribute setup), then once inside the
cudaProfilerStart/Stop range (use `--profile-from-start off`)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "src"))
import torch
from opendwm_b200 import ops, lib


def main():
    dt = torch.float16 if os.environ.get("DWM_NCU_DTYPE", "bf16") == "fp16" else torch.bfloat16
    D, heads, N, S, L = 1536, 24, 192, 448, 154
    M = N * S
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    todo = []

    # --- attention -------------------------------------------------------------------
    qkv = rnd(N * (S + L), 3 * D).to(dt)
    o, o2 = torch.empty(M, D, device=dev, dtype=dt), torch.empty(N * L, D, device=dev, dtype=dt)
    todo.append(("joint attention 602 (attn_wgmma)", lambda: ops.attention(
        qkv, o, D=D, heads=heads, group_dims=[N], group_strides=[S + L], seq=S + L,
        out_group_strides=[S], out_stride_outer=0, out_stride_inner=1, split=S, out2=o2)))
    qs = rnd(M, 3 * D).to(dt)
    B, T, V, H, W = 2, 16, 6, 16, 28
    todo.append(("temporal point-wise attention (attn_kernel)", lambda: ops.attention(
        qs, o, D=D, heads=heads, group_dims=[B, V * S], group_strides=[T * V * S, 1], seq=T,
        inner=1, stride_outer=V * S, stride_inner=0)))
    ring = torch.zeros(V, V, dtype=torch.bool)
    for i in range(V):
        for d in (-1, 0, 1):
            ring[i, (i + d) % V] = True
    mask = ring.unsqueeze(0).repeat(B, 1, 1).to(dev).to(torch.uint8).contiguous()
    todo.append(("cross-view row-wise attention + mask (attn_wgmma gathered)", lambda: ops.attention(
        qs, o, D=D, heads=heads, group_dims=[B * T, H], group_strides=[V * S, W], seq=V * W,
        inner=W, stride_outer=S, stride_inner=1, mask=mask, mask_div=T)))

    # --- LayerNorm ---------------------------------------------------------------------
    x = rnd(M, D)
    a16 = torch.empty(M, D, device=dev, dtype=dt)
    mod = rnd(N, 6 * D)
    todo.append(("layernorm + AdaLN modulate", lambda: ops.layernorm(
        x, a16, eps=1e-6, rows_per_item=S, shift=mod[:, :D], scale=mod[:, D:2 * D])))

    # --- GEMMs ---------------------------------------------------------------------------
    w_sq = (rnd(D, D) * 0.02).to(dt)
    gate = rnd(N, D)
    xr = rnd(M, D)
    todo.append(("GEMM out-proj 86016x1536x1536 RESID+gate", lambda: ops.linear(
        a16, w_sq, None, epilogue=lib.EPI_RESID, resid=xr, out=xr, gate=gate, rows_per_item=S)))
    g16 = rnd(M, 4 * D).to(dt)
    w_ff2 = (rnd(D, 4 * D) * 0.02).to(dt)
    todo.append(("GEMM FF2 86016x1536x6144 RESID+gate", lambda: ops.linear(
        g16, w_ff2, None, epilogue=lib.EPI_RESID, resid=xr, out=xr, gate=gate, rows_per_item=S)))
    w_ff1 = (rnd(4 * D, D) * 0.02).to(dt)
    todo.append(("GEMM FF1 86016x6144x1536 STORE+GELU", lambda: ops.linear(
        a16, w_ff1, None, act=lib.ACT_GELU_TANH, out=g16)))
    # the step's dominant kernel: VT-block FF1 with the GEGLU epilogue (packed 8D x D weight)
    w_gg, b_gg = ops.pack_geglu(rnd(8 * D, D) * 0.02, torch.zeros(8 * D, device=dev))
    w_gg = w_gg.to(dt)
    todo.append(("GEMM GEGLU 86016x12288x1536 (dominant)", lambda: ops.linear(
        a16, w_gg, b_gg, epilogue=lib.EPI_GEGLU, out=g16)))

    # --- convolution / GroupNorm (VAE shapes) ----------------------------------------------
    xc = rnd(2, 2 + 2, 128, 224, 256).to(dt)                  # CogVideoX up-block, 256 ch
    wc = ops.pack_conv_weight(rnd(256, 256, 3, 3, 3) * 0.02, dt)
    bc = torch.zeros(256, device=dev)
    todo.append(("conv 3x3x3 256->256 @ 2x2x128x224 (CogVideoX)", lambda: ops.conv(
        xc, wc, bc, kernel=(3, 3, 3), epilogue=lib.EPI_F32)))
    xc2 = rnd(6, 1, 256, 448, 128).to(dt)                      # last VAE block, 128 ch
    wc2 = ops.pack_conv_weight(rnd(128, 128, 3, 3) * 0.02, dt)
    bc2 = torch.zeros(128, device=dev)
    todo.append(("conv 3x3 128->128 @ 6x256x448 (AutoencoderKL)", lambda: ops.conv(
        xc2, wc2, bc2, kernel=(1, 3, 3), epilogue=lib.EPI_F32)))
    hf = rnd(6, 1, 256, 448, 128)
    gam, bet = torch.ones(128, device=dev), torch.zeros(128, device=dev)
    out16 = torch.empty(6, 1, 256, 448, 128, device=dev, dtype=dt)

    def gn():
        sums = ops.groupnorm_stats(hf, 32)
        ops.spatialnorm_silu(hf, sums, gam, bet, out16, groups=32, eps=1e-6, silu=True)
    todo.append(("GroupNorm stats + apply+SiLU 6x256x448x128", gn))

    only = [t for t in os.environ.get("DWM_NCU_ONLY", "").split(",") if t]
    if only:      # e.g. DWM_NCU_ONLY="cross-view,out-proj": capture a subset
        todo = [(n, f) for n, f in todo if any(t in n for t in only)]
    for _, f in todo:
        f()
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    for name, f in todo:
        f()
        torch.cuda.synchronize()
        print("launched:", name)
    torch.cuda.cudart().cudaProfilerStop()


if __name__ == "__main__":
    main()
