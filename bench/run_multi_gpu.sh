#!/bin/bash
# Multi-GPU evidence run (N GPUs):  bash bench/run_multi_gpu.sh N [quick]
# Writes bench_out/scale_N/*.json|log : fused-engine tests, flagship bench (ours fused / unfused, reference),
# Mixtral-shape block (config #3), all-to-all sweep vs NCCL (config #5).
N=${1:-8}
MODE=${2:-full}
OUT=bench_out/scale_$N
mkdir -p $OUT
T="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
P=29600
run() { name=$1; shift; P=$((P+1)); timeout 240 $T --master-port $P "$@" > $OUT/$name.json 2> $OUT/$name.err; tail -c 2000 $OUT/$name.json | python -c "
import sys, json
try:
    d = json.loads(sys.stdin.read().strip().splitlines()[-1])
    print('$name', 'ms/step', round(d['ms_per_step'], 3), 'tok/s', round(d['value']), 'e2e', round(d['e2e']['value']) if d.get('e2e') else None, d.get('clocks'))
except Exception as ex:
    print('$name FAILED', ex)
"; grep -E "timeout|Error" $OUT/$name.err | head -3; }

timeout 300 $T --master-port 29599 tests/workers/p2p_worker.py all > $OUT/p2p_worker.log 2>&1; grep -cE "OK" $OUT/p2p_worker.log; grep -E "FAIL|timeout|WORKER_OK" $OUT/p2p_worker.log | head -5
run bench_ours bench.py --gpus $N --steps 20 --warmup 5
run bench_reference bench.py --impl reference --gpus $N --steps 20 --warmup 5
if [ "$MODE" != "lean" ]; then TUTEL_B200_FUSED=0 run bench_ours_unfused bench.py --gpus $N --steps 20 --warmup 5; fi
if [ "$MODE" = "full" ] || [ "$MODE" = "lean" ]; then
  run mixtral_ours_bf16_fused bench.py --gpus $N --steps 10 --warmup 3 --expert_type llama_ffn
  TUTEL_B200_FUSED=0 run mixtral_ours_bf16_unfused_d2 bench.py --gpus $N --steps 10 --warmup 3 --expert_type llama_ffn --overlap 2
  run mixtral_reference_bf16_d2 bench.py --impl reference --gpus $N --steps 10 --warmup 3 --expert_type llama_ffn --overlap 2
  P=$((P+1)); timeout 300 $T --master-port $P -m tutel_b200.examples.bandwidth_test --sweep --compare_nccl --loop 10 --json $OUT/a2a_sweep.json > $OUT/a2a_sweep.log 2>&1
  grep -E "all_to_all" $OUT/a2a_sweep.log | tail -8
fi
