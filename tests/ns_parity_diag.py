"""Measurement only (not collected by pytest): WHERE the 16-bit paths drift from the fp32
oracle at the full north-star size.  Captures the sample stream after every joint / temporal
/ cross-view block of the fp32 oracle on the GPU and compares (a) the native bf16 path,
(b) the native fp16 path, (c) the oracle itself in eager bf16 autocast, stage by stage; also
(d) the fp32 oracle's own sensitivity to a bf16 rounding of its input latents.  A kernel
bug shows as a jump at one stage; rounding noise amplified by random weights grows smoothly
and equally in (a) and (c).   Usage: python tests/ns_parity_diag.py [mix] [std]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src")):
    sys.path.insert(0, p)
import torch  # noqa: E402


def rel(a, b):
    d = (a.float() - b.float())
    return [float(d.pow(2).mean().sqrt() / b.float().pow(2).mean().sqrt()),
            float(d.abs().max() / b.float().abs().max())]


def main():
    import bench
    from oracle import ctsd as octsd
    from opendwm_b200 import lib
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    mix = float(sys.argv[1]) if len(sys.argv) > 1 else 0.4
    cfg = bench.load_config()
    B, T, V, C, H, W = cfg["latent_shape"]
    steps = cfg["inference_steps"]
    spi = steps // T
    dev = torch.device("cuda", 0)

    def native(dtype):
        torch.set_default_dtype(dtype)
        try:
            with torch.device(dev):
                m = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
        finally:
            torch.set_default_dtype(torch.float32)
        bench.init_weights_(m)
        with torch.no_grad():
            for n, p in m.named_parameters():
                if n.endswith("mix_factor"):
                    p.fill_(mix)
        return m

    model = native(torch.bfloat16)
    with torch.device(dev):
        oracle = octsd.DiTCrossviewTemporalConditionModel(**cfg["model"])
    oracle.load_state_dict(model.state_dict())
    oracle.to(dev).eval()
    cond = bench.synthetic_conditions(cfg, 2 * B, T, V, dev, torch.bfloat16)
    cond32 = {k: (v.float() if v.is_floating_point() else v) for k, v in cond.items()}
    lat = torch.randn(B, T, V, C, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    x2 = torch.cat([lat, lat])
    sched = octsd.FlowMatchEulerDiscreteScheduler(shift=3.0)
    sched.set_timesteps(steps)
    idx = torch.tensor(octsd.df_timestep_indices(steps - 2, T, spi), device=dev)
    ts = sched.timesteps.to(dev)[idx].view(1, T, 1).expand(2 * B, T, V).contiguous()

    # ---- fp32 oracle with captures -------------------------------------------------
    caps, order = {}, []
    sink = {"store": True, "cmp": None, "out": None}

    def record(key, h):
        h = h.reshape(-1, h.shape[-1])
        if sink["store"]:
            caps[key] = h.detach().float().clone()
            order.append(key)
        else:
            sink["out"][str(key)] = rel(h, caps[key])

    for i, blk in enumerate(oracle.transformer_blocks):
        blk.register_forward_hook(lambda m, a, out, i=i: record(("joint", i), out[1]))
    f_t, f_c = oracle.forward_temporal_block_and_mix_result, \
        oracle.forward_crossview_block_and_mix_result
    tl, cl = list(oracle.temporal_block_layers), list(oracle.crossview_block_layers)

    def wrap_t(block, *a, **k):
        out = f_t(block, *a, **k)
        record(("temporal", tl[list(oracle.temporal_transformer_blocks).index(block)]), out)
        return out

    def wrap_c(block, *a, **k):
        out = f_c(block, *a, **k)
        record(("crossview", cl[list(oracle.crossview_transformer_blocks).index(block)]), out)
        return out
    oracle.forward_temporal_block_and_mix_result = wrap_t
    oracle.forward_crossview_block_and_mix_result = wrap_c

    with torch.no_grad():
        ref = oracle(x2, ts, **cond32)[0][0]
    res = {"mix_factor": mix, "stages": [str(k) for k in order], "ref_absmax": float(ref.abs().max())}

    # (d) fp32 oracle, latents rounded to bf16
    sink.update(store=False, out={})
    with torch.no_grad():
        y = oracle(x2.bfloat16().float(), ts, **cond32)[0][0]
    res["oracle_fp32_bf16_rounded_input"] = {"stages": sink["out"], "out": rel(y, ref)}
    # (c) oracle in eager bf16 autocast
    sink["out"] = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        y = oracle(x2, ts, **cond)[0][0]
    res["oracle_eager_bf16_autocast"] = {"stages": sink["out"], "out": rel(y, ref)}
    sink["out"] = {}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        y = oracle(x2, ts, **{k: (v.half() if v.is_floating_point() else v) for k, v in cond.items()})[0][0]
    res["oracle_eager_fp16_autocast"] = {"stages": sink["out"], "out": rel(y, ref)}

    # (a)/(b) native
    def run_native(m, c, tag, **opts):
        for k, v in opts.items():
            lib.set_option(k, v)
        out = {}
        m._trace = lambda key, x: out.__setitem__(str(key), rel(x, caps[key]))
        y = m(x2, ts, **c)[0][0]
        torch.cuda.synchronize()
        res[tag] = {"stages": out, "out": rel(y, ref)}
        for k in opts:
            lib.set_option(k, -1)
    run_native(model, cond, "native_bf16")
    run_native(model, cond, "native_bf16_legacy_kernels", gemm_2cta=0, attn_tc=0)
    del model
    torch.cuda.empty_cache()
    sd = {k: v.clone() for k, v in oracle.state_dict().items()}     # same (bf16-exact) weights
    m16 = native(torch.float16)
    m16.load_state_dict(sd)
    run_native(m16, {k: (v.half() if v.is_floating_point() else v) for k, v in cond.items()},
               "native_fp16")

    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "ns_parity_diag.json"), "w") as f:
        json.dump(res, f, indent=1)
    for tag in ("oracle_fp32_bf16_rounded_input", "oracle_eager_bf16_autocast",
                "oracle_eager_fp16_autocast", "native_bf16", "native_bf16_legacy_kernels",
                "native_fp16"):
        st = res[tag]["stages"]
        keys = [str(k) for k in order]
        pick = [keys[j] for j in (0, 1, 2, len(keys) // 4, len(keys) // 2, -2, -1)]
        print(tag, "out rms/max", ["%.2e" % v for v in res[tag]["out"]],
              " ".join("%s:%.1e" % (k.replace("'", ""), st[k][0]) for k in pick if k in st))


if __name__ == "__main__":
    main()
