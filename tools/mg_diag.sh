#!/bin/bash
# Diagnostic A/B of the shared-volume mode on N GPUs (NG, default 2): where does the time of the one-stream / one-volume frame go?
NG=${NG:-2}
run() { echo "== $*"; env "$@" KT_BENCH_FRAMES=24 python -m torch.distributed.run --nnodes=1 --nproc-per-node $NG --master-addr 127.0.0.1 --master-port 29533 bench.py --gpus $NG --steps 60 --warmup 5 --shared-only 2>&1 | tail -1 | python tools/mg_diag.py; }
run KT_DUMMY=1
run KT_MG_SPLIT_ICP=1
