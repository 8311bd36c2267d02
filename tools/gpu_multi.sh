#!/bin/bash
# Multi-GPU session (gpurun --gpus N -- tools/gpu_multi.sh N): the record exchange over peer memory vs ncclAllGather,
# N-GPU == 1-GPU equivalence on hardware, the bench at N, evaluate over a split at N, and the dense_align sweep at N
# (BASELINE configs[4]).
N=${1:-2}
out=gpurun_out
mkdir -p $out
export PYTHONUNBUFFERED=1
T="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511"
if [ "$N" -le 2 ]; then
echo "== sanity: composed forward"
timeout 300 python -m pytest tests/test_gpu_model.py -m gpu -q --timeout 150 -k "forward_small_fp16 or conv_tc_fp16" > $out/pytest_sanity_$N.log 2>&1; echo "rc=$?"; tail -3 $out/pytest_sanity_$N.log
fi
echo "== gather + shard equivalence tests ($N GPUs visible)"
timeout 600 python -m pytest tests/test_gpu_round2.py -m gpu -q --timeout 500 -s -k "record_gather" > $out/pytest_multi_$N.log 2>&1; echo "rc=$?"; tail -6 $out/pytest_multi_$N.log
if [ -n "$WITH_LAG0" ]; then
echo "== bench N=$N, peer gather, same-step (lag 0)"
timeout 400 $T bench.py --gpus $N --steps 20 --warmup 5 --gather peer --gather-lag 0 > $out/bench_n${N}_peer0.json 2> $out/bench_n${N}_peer0.err; echo "rc=$?"; tail -c 200 $out/bench_n${N}_peer0.err
fi
echo "== bench N=$N, peer gather, pipelined (default)"
timeout 400 $T bench.py --gpus $N --steps 20 --warmup 5 --gather peer > $out/bench_n${N}_peer.json 2> $out/bench_n${N}_peer.err; echo "rc=$?"; tail -c 300 $out/bench_n${N}_peer.err
echo "== bench N=$N, nccl gather"
timeout 400 $T bench.py --gpus $N --steps 20 --warmup 5 --gather nccl > $out/bench_n${N}_nccl.json 2> $out/bench_n${N}_nccl.err; echo "rc=$?"; tail -c 300 $out/bench_n${N}_nccl.err
echo "== evaluate over a split, sharded over $N GPUs (run with N = 2 and 8)"
timeout 600 $T tools/evaluate_bench.py > $out/evaluate_n$N.json 2> $out/evaluate_n$N.err; echo "rc=$?"; tail -c 300 $out/evaluate_n$N.err; cut -c1-1200 $out/evaluate_n$N.json
if [ -z "$SKIP_SWEEP" ]; then
echo "== dense_align sweep, $N GPUs"
timeout 300 $T tests/tools/dense_align_sweep.py > $out/dense_sweep_n$N.log 2>&1; echo "rc=$?"; tail -4 $out/dense_sweep_n$N.log
fi
cat $out/bench_n${N}_peer.json | cut -c1-600
