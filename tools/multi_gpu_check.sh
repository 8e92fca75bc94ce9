#!/bin/bash
# usage (on an N-GPU node, from the repository root): bash tools/multi_gpu_check.sh N [OUT_DIR]
# the pose-board check under torchrun (bitwise against ncclAllGather) + the default bench line at N ranks → OUT_DIR
N=$1; out=${2:-$(mktemp -d)}; mkdir -p $out; echo "output: $out"
if [ "$N" = "2" ]; then timeout 600 python -m pytest tests/test_gpu_pose_board.py -x -q 2>&1 | tail -3; fi
timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29521 tools/check_pose_board.py 2>&1 | grep -v "^W\|^\*\*\*\|OMP_NUM" | tail -4
run() { # tag, env
  env $2 timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $3 bench.py --gpus $N --steps 20 --warmup 5 --no-cpu-baseline > $out/bench_n${N}_$1.json 2> $out/bench_n${N}_$1.err
  python - <<PY
import json
try:
    l = json.loads(open("$out/bench_n${N}_$1.json").read().strip().splitlines()[-1])
    print("$1 N=$N value %.0f e2e %.0f pageable %.0f exchange %s checked %s launches %s" % (l["value"], l["e2e"]["value"], l["e2e"]["pageable"]["value"], l["details"]["pose_exchange"], l["details"]["pose_exchange_equals_nccl_all_gather"], l["gpu_launches"]))
    for p in l["per_rank"]: print("   ", {k: (round(v, 4) if not isinstance(v, dict) else {a: round(b, 4) for a, b in v.items()}) for k, v in p.items()})
    c = l.get("c4")
    if c: print("   c4 value %.0f ms_total %.2f per_rank %s" % (c["value"], c["ms_total"], [round(x, 2) for x in c["per_rank_ms"]]))
except Exception as e:
    print("$1 failed", e); print(open("$out/bench_n${N}_$1.err").read()[-3000:])
PY
}
run board BENCH_X=1 29514
if [ "$N" = "2" ]; then run board2 BENCH_X=1 29515; fi
