#!/bin/bash
# Multi-GPU run on one host: the multi-GPU tests, then BASELINE configs[4] -- the 16K Hap Q stream delivered to rank 0 -- at
# every power of two up to the GPUs present, ring delivery and NCCL gatherv in the same line.
#   bash tools/gpu_stream_scale.sh r03s [DIR]      -> everything lands in DIR/r03s_* (DIR defaults to validate_out)
TAG=${1:-scale}
OUT=${2:-validate_out}
mkdir -p "$OUT"
G=$(nvidia-smi -L | wc -l)
(time timeout 600 python -m pytest tests/test_gpu_multi.py -m gpu -x -q --timeout 300) > $OUT/${TAG}_tests.log 2>&1
tail -3 $OUT/${TAG}_tests.log
for N in 8 4 2; do
  [ $N -le $G ] || continue
  timeout 240 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((29550 + N)) bench.py --gpus $N --workload 16k_stream --steps 8 --warmup 4 > $OUT/${TAG}_stream_n$N.json 2> $OUT/${TAG}_stream_n$N.err
done
timeout 200 python bench.py --workload 16k_stream --steps 8 --warmup 4 > $OUT/${TAG}_stream_n1.json 2> $OUT/${TAG}_stream_n1.err
python - <<PY
import json
for n in (1, 2, 4, 8):
    try:
        d = json.load(open("$OUT/${TAG}_stream_n%d.json" % n)); b = d.get("nccl_gatherv_baseline") or {}; r = d.get("ring_delivery") or d
        print(n, d.get("delivery"), "fps %.0f | ring fps %.0f nccl fps %.0f | encode alone %.3f ms" % (d["fps"], r["fps"], b.get("fps", 0), d["encode_only_ms_per_step"]))
    except Exception as e:
        print(n, "no line:", e)
PY
