mkdir -p gpurun_out
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1"
timeout 300 $TR --master-port 29533 tools/ddp_train_check.py 2>&1 | tail -3
timeout 300 $TR --master-port 29534 bench.py --mode train --gpus 2 --steps 10 --warmup 3 2>/dev/null | tail -1 | python -c "import sys,json; d=json.loads(sys.stdin.read()); print(d['ms_per_step'], d['value'])"
