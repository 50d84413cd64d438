#!/bin/bash
# Same-machine A/B of two builds of libqcnn_b200.so (machine-to-machine spread of a layer time is ~3-5 %, more than most
# kernel changes are worth): build the alternative, keep it next to the product library, and let one run swap them.
#   git stash; make -C quantized-cnn_b200 -j8; cp quantized-cnn_b200/libqcnn_b200.so quantized-cnn_b200/alt.so
#   git stash pop; make -C quantized-cnn_b200 -j8
#   bash tools/ab_compare.sh quantized-cnn_b200/alt.so 256 [layer_times.py arguments, e.g. --tc 0: the strict path]
# Output: $AB_OUT (default bench_out)/ab_{cur,alt}_{1,2}.log (tools/layer_times.py, two alternating rounds), a one-line
# summary per run.
set -u
ALT=${1:?path of the alternative libqcnn_b200.so}
B=${2:-256}
shift 2 2>/dev/null || shift $#
OUT=${AB_OUT:-bench_out}
LIB=quantized-cnn_b200/libqcnn_b200.so
mkdir -p "$OUT"
cp "$LIB" "$OUT/.ab_cur.so"
for r in 1 2; do
  python tools/layer_times.py --batch "$B" --reps 40 "$@" > "$OUT/ab_cur_$r.log" 2>&1
  cp "$ALT" "$LIB"
  python tools/layer_times.py --batch "$B" --reps 40 "$@" > "$OUT/ab_alt_$r.log" 2>&1
  cp "$OUT/.ab_cur.so" "$LIB"
done
rm -f "$OUT/.ab_cur.so"
for f in "$OUT/ab_cur_1.log" "$OUT/ab_alt_1.log" "$OUT/ab_cur_2.log" "$OUT/ab_alt_2.log"; do
  echo "$f: $(grep -v autotune "$f" | awk '/^batch/{printf "%s ms/forward |", $3} /^  layer/{printf " %s", $3}')"
done
