#!/bin/bash
# Every example program for a few steps on N GPUs (small shapes): proves they run on the GPU paths.  Usage: bash bench/examples_smoke.sh 2
N=${1:-2}
OUT=bench_out/examples_$N
mkdir -p $OUT
export TUTEL_B200_SPIN_TIMEOUT_SEC=20
T="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
P=29300
COMMON="--num_steps 6 --batch_size 8 --num_tokens 256 --model_dim 512 --hidden_size 1024"
run() { name=$1; shift; P=$((P+1)); timeout 150 $T --master-port $P -m tutel_b200.examples.$name "$@" > $OUT/$name.log 2>&1; rc=$?; echo "$name rc=$rc $(grep -E 'STEP-5|Summary|OK' $OUT/$name.log | tail -1 | cut -c1-120)"; }
run helloworld $COMMON --dtype bfloat16
run helloworld $COMMON --dtype float16 --num_local_experts -$N --parallel_type model
run helloworld_switch $COMMON --dtype bfloat16 --num_local_experts -$N
run helloworld_amp $COMMON
run helloworld_ddp $COMMON --dtype bfloat16
run helloworld_ddp_tutel $COMMON --dtype float32
run helloworld_from_scratch --num_steps 6 --model_dim 512 --hidden_size 1024 --num_samples 2048
run helloworld_custom_gate_expert $COMMON --dtype bfloat16
run helloworld_custom_expert_sharded $COMMON --dtype bfloat16
run nccl_all_to_all_v
run nccl_all_gather_v
run bandwidth_test --size_mb 16 --loop 5
