"""Per-rank compute of the N-GPU sharded step on ONE GPU (no communication): the model runs on
this rank's share of the view-frame grid — one CFG branch, T/t_ways frames, all views — i.e. the
GEMM / attention / LayerNorm shapes a rank of `bench.py --gpus N` launches (temporal attention
sees only the local frames; < 1 % of the step).  Prints the step time and the per-shape GEMM
rates so that shard-size effects (tile quantisation, fixed per-launch costs) can be profiled
without an N-GPU box.

    python tools/shard_emulate.py 8 [steps] [dtype]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "src")):
    sys.path.insert(0, p)
import torch  # noqa: E402

import bench  # noqa: E402
from opendwm_b200 import ops  # noqa: E402


def main():
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[sys.argv[3] if len(sys.argv) > 3 else "fp16"]
    cfg = bench.load_config()
    B, T, V, C, H, W = cfg["latent_shape"]
    cfg_ways = 2 if n >= 2 else 1
    t_ways = n // cfg_ways
    Tl, Bl = T // t_ways, (2 * B) // cfg_ways
    dev = torch.device("cuda", 0)
    torch.set_default_dtype(dtype)
    with torch.device(dev):
        model = DiTCrossviewTemporalConditionModel(**cfg["model"], compute_dtype=dtype)
    torch.set_default_dtype(torch.float32)
    bench.init_weights_(model)
    cond = bench.synthetic_conditions(cfg, Bl, Tl, V, dev, dtype)
    x = torch.randn(Bl, Tl, V, C, H, W, device=dev)
    ts = torch.full((Bl, Tl, V), 500.0, device=dev)

    def step():
        model.forward_tokens(x, ts, cond["encoder_hidden_states"], cond["pooled_projections"],
                             cond["condition_image_tensor"], cond["disable_crossview"],
                             cond["disable_temporal"], cond["crossview_attention_mask"],
                             cond["added_time_ids"], t_offset=0, T_total=T)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    ops.profile_begin()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    prof = ops.profile_end()
    ms = e0.elapsed_time(e1) / steps
    agg = {}
    for p_ in prof["linear"]:
        k = (tuple(p_["shape"]), p_["epilogue"])
        a = agg.setdefault(k, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += p_["ms"]
        a[2] += p_["flops"]
    rows = [{"M": k[0][0], "N": k[0][1], "K": k[0][2], "epilogue": k[1],
             "launches_per_step": v[0] / steps, "ms_per_step": v[1] / steps,
             "us_per_launch": 1e3 * v[1] / v[0], "tflops": v[2] / v[1] / 1e9}
            for k, v in agg.items()]
    rows.sort(key=lambda r: -r["ms_per_step"])
    gemm_ms = sum(r["ms_per_step"] for r in rows)
    res = {"emulated_world": n, "items_per_rank": Bl * Tl * V, "dtype": str(dtype), "ms_per_step": ms,
           "ideal_ms_from_flops": bench.F_STEP_TFLOP / n / 1.4, "gemm_ms_per_step": gemm_ms,
           "non_gemm_ms_per_step": ms - gemm_ms, "launches_per_step": prof["launches"] / steps,
           "rows": rows[:14]}
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "shard_emulate_%d.json" % n), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
