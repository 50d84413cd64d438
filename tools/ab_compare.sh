#!/bin/bash
# Same-machine A/B of two builds of libqcnn_b200.so (machine-to-machine spread of a step time is ~3-5 %, more than most
# kernel changes are worth): build the alternative, keep it next to the product library, and let one run swap them.
#   git stash; make -C quantized-cnn_b200 -j8; cp quantized-cnn_b200/libqcnn_b200.so quantized-cnn_b200/alt.so
#   git stash pop; make -C quantized-cnn_b200 -j8
#   bash tools/ab_compare.sh quantized-cnn_b200/alt.so [rounds, default 3] [extra bench.py arguments]
# Each round runs `python bench.py --gpus 1 --steps 20 --warmup 3` once with the current library, then once with the
# alternative; the JSON lines go to $AB_OUT (default bench_out)/ab_{cur,alt}_<round>.json.  Printed per run: `value`
# (batch 256, images/s), `config4.value` (batch 1024), `value_strict.value`, `extra.latency_b1_ms` and the per-layer ms;
# then the median and min-max of `value` per side.  The current library is put back on exit, also after a failure.
set -u
ALT=${1:?path of the alternative libqcnn_b200.so}
ROUNDS=${2:-3}
shift 2 2>/dev/null || shift $#
OUT=${AB_OUT:-bench_out}
LIB=quantized-cnn_b200/libqcnn_b200.so
mkdir -p "$OUT"
cp "$LIB" "$OUT/.ab_cur.so"
trap 'cp "$OUT/.ab_cur.so" "$LIB"; rm -f "$OUT/.ab_cur.so"' EXIT
for r in $(seq 1 "$ROUNDS"); do
  cp "$OUT/.ab_cur.so" "$LIB"
  python bench.py --gpus 1 --steps 20 --warmup 3 "$@" 2> "$OUT/ab_cur_$r.err" | tail -n 1 > "$OUT/ab_cur_$r.json"
  cp "$ALT" "$LIB"
  python bench.py --gpus 1 --steps 20 --warmup 3 "$@" 2> "$OUT/ab_alt_$r.err" | tail -n 1 > "$OUT/ab_alt_$r.json"
done
python - "$OUT" "$ROUNDS" <<'PY'
import json, sys
import numpy as np
out, rounds = sys.argv[1], int(sys.argv[2])
vals = {"cur": [], "alt": []}
for r in range(1, rounds + 1):
    for side in ("cur", "alt"):
        try:
            j = json.load(open("%s/ab_%s_%d.json" % (out, side, r)))
        except (OSError, ValueError) as e:
            print("%s round %d: no result (%s)" % (side, r, e))
            continue
        vals[side].append(j["value"])
        c4 = (j.get("config4") or {}).get("value")
        st = (j.get("value_strict") or {}).get("value")
        lat = (j.get("extra") or {}).get("latency_b1_ms")
        layers = " ".join("%s=%.4f" % (k, v["ms"]) for k, v in (j.get("per_layer") or {}).items())
        print("%s round %d: value %.1f  config4.value %s  value_strict %s  latency_b1_ms %s | %s"
              % (side, r, j["value"], "%.1f" % c4 if c4 else "-", "%.1f" % st if st else "-", lat, layers))
for side, v in vals.items():
    if v:
        print("%s: value median %.1f  (min %.1f, max %.1f, %d runs)" % (side, float(np.median(v)), min(v), max(v), len(v)))
PY
