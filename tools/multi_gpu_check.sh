#!/usr/bin/env bash
# N-GPU validation + measurement on one node with N GPUs (results under bench_out/):
#   bash tools/multi_gpu_check.sh N
# 1. tools/shard_check.py (sharded == unsharded, bit for bit, T in {5,8,11,19}, peer scatter and
#    NCCL all-gather);  2. bench.py --gpus N without and with CUDA-graph replay of the sharded step.
N=${1:-8}
mkdir -p bench_out
run() { timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $1 "${@:2}"; }
for ps in 1 0; do
  DWM_PEER_SCATTER=$ps run $((29540 + ps)) tools/shard_check.py 2>&1 | grep -E "shard_check|rror" | head -12
done
for g in 0 1; do
  DWM_BENCH_WATCHDOG=240 DWM_CUDA_GRAPH_SHARDED=$g run $((29550 + g)) bench.py --gpus $N --no-extras --no-cpu-baseline \
      > bench_out/bench_${N}gpu_graph$g.json 2> bench_out/bench_${N}gpu_graph$g.err
  tail -c 400 bench_out/bench_${N}gpu_graph$g.err
  python - <<PY
import json
try:
    d = json.load(open("bench_out/bench_${N}gpu_graph$g.json"))
    print("N=%d graph=%d ms_per_step=%.2f value=%.2f e2e=%.2f (cuda_graph=%s) gemm=%.0f TF/s" % (
        d["n_gpus"], $g, d["ms_per_step"], d["value"], d["e2e"]["value"], d["e2e"]["cuda_graph"],
        d["roofline"]["all_gemm_achieved"]))
except Exception as e:
    print("no result:", e)
PY
done
