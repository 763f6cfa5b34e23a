#!/bin/bash
# BASELINE.json configs[4]: batch sweep 1 -> 512 synthetic 4-s clips, N = 30, on G GPUs of one box (default 1).
#   bash tools/sweep_batch.sh [G]        -> one bench.py JSON line per batch size in ${OUT:-sweep_out}/sweep_g${G}.jsonl
# Per-GPU batch b is sampled in micro-batches of min(b, 16) (one captured graph per micro-batch shape); under
# torch.distributed.run the same line shards G*b clips over G ranks with no data-path collective.
G=${1:-1}
mkdir -p "${OUT:-sweep_out}"
out=${OUT:-sweep_out}/sweep_g${G}.jsonl
: > $out
for b in 1 2 4 8 16 32 64 128 256 512; do
  mb=$(( b < 16 ? b : 16 ))
  pb=$(( (b + G - 1) / G ))            # clips per GPU
  pmb=$(( pb < 16 ? pb : 16 ))
  if [ "$G" = "1" ]; then
    python bench.py --batch $b --micro-batch $mb --steps 2 --warmup 3 --no-cpu-baseline --no-roofline >> $out
  else
    python -m torch.distributed.run --nnodes=1 --nproc-per-node $G --master-addr 127.0.0.1 --master-port 29517 \
      bench.py --gpus $G --batch $pb --micro-batch $pmb --steps 2 --warmup 3 --no-cpu-baseline --no-roofline >> $out
  fi
done
python - <<PY
import json
for l in open("$out"):
    l = l.strip()
    if l.startswith("{"):
        d = json.loads(l)
        print(f'global batch {d["config"]["global_batch"]:4d}  {d["value"]:8.2f} utt/s  {d["ms_per_step"]:9.1f} ms/step')
PY
