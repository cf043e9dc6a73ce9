#!/bin/bash
mkdir -p build
timeout 100 python -m pytest tests/test_gpu_dist.py -m gpu -x -q --timeout 90 --timeout-method=thread 2>&1 | tail -2
timeout 100 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 bench.py --gpus 2 --steps 5 --warmup 3 --no-cpu > build/bench_n2.json 2> build/bench_n2.err; echo "bench rc=$?"; cut -c1-700 build/bench_n2.json; tail -2 build/bench_n2.err
