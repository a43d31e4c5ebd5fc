set -x
timeout 600 python -m pytest tests/test_gpu_sharded.py -x -q 2>&1 | tail -3
timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29655 bench.py --gpus 2 --no-cpu-baseline
