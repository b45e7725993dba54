#!/usr/bin/env bash
# Same-build A/B of the dirty-row marks: bench.py with GLAVA_B200_FULL_STORE=1 (every zero row stored, the marks ignored)
# and without, alternated, REPS times per configuration, plus --dump-outputs of both arms of the first pair.
#
#   tools/full_store_ab.sh OUT_DIR [REPS] [CONFIG ...]        (default: 3 headline graph720 wave720)
#
# Writes OUT_DIR/<config>_<arm>_<i>.json (one bench line each), OUT_DIR/dump_<config>_<arm>/ and OUT_DIR/card.txt.
set -u
OUT=${1:?out dir}; REPS=${2:-3}; shift 2 2>/dev/null || shift $#
CONFIGS=${*:-headline graph720 wave720}
cd "$(dirname "$0")/.."
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$OUT/card.txt"
for cfg in $CONFIGS; do
    for i in $(seq 1 "$REPS"); do
        for arm in full marks; do
            dump=()
            [ "$i" = 1 ] && dump=(--dump-outputs "$OUT/dump_${cfg}_${arm}")
            if [ "$arm" = full ]; then export GLAVA_B200_FULL_STORE=1; else unset GLAVA_B200_FULL_STORE; fi
            python bench.py --gpus 1 --steps 200 --warmup 3 --config "$cfg" --no-cpu-baseline --no-extras "${dump[@]}" \
                > "$OUT/${cfg}_${arm}_${i}.json" 2> "$OUT/${cfg}_${arm}_${i}.err"
            unset GLAVA_B200_FULL_STORE
        done
    done
    if cmp -s "$OUT/dump_${cfg}_full/frames_sample.npy" "$OUT/dump_${cfg}_marks/frames_sample.npy"; then
        echo "$cfg frames_sample.npy identical" >> "$OUT/dumps.txt"
    else
        echo "$cfg frames_sample.npy DIFFER" >> "$OUT/dumps.txt"
    fi
done
python - "$OUT" $CONFIGS <<'EOF'
import json, glob, os, statistics, sys
out = sys.argv[1]
for cfg in sys.argv[2:]:
    for arm in ("full", "marks"):
        rows = []
        for f in sorted(glob.glob(os.path.join(out, f"{cfg}_{arm}_*.json"))):
            try:
                d = json.loads(open(f).read().strip().splitlines()[-1])
            except Exception:
                continue
            r = d["roofline"]
            rows.append((d["value"], d["ms_per_step"], r["kernel_ms"], r["kernel_ms_isolated"]))
        if rows:
            v = [x[0] for x in rows]
            print(f"{cfg:9s} {arm:5s} value median {statistics.median(v):10.0f}  min {min(v):10.0f}  max {max(v):10.0f}  "
                  f"ms/step {statistics.median([x[1] for x in rows]):.4f}  raster ms {statistics.median([x[2] for x in rows]):.4f}  "
                  f"isolated {statistics.median([x[3] for x in rows]):.4f}")
EOF
