#!/bin/bash
# Nsight Compute capture of one workload on ONE GPU:   profiles/run_ncu.sh <tag> <workload> [copies] [output directory, default ncu_out]
#   workload = CornellBox | ShaderBalls | CornellBox_Dragon | Synthetic10M   (bench.py's WORKLOADS)
# Captures, of the SECOND frame that tools/render_frames.py renders (the first one warms up):
#   prof_<workload>_<tag>.csv          --set full of every launch of the per-phase schedule with the shadow pass as its own kernel
#                                      (k_trace_closest, k_shadow_accumulate, k_shade_queues: the kernel classes bench.py times with CUDA events)
#   prof_<workload>_src_<tag>.ncu-rep  bounce 1 of k_trace_closest and of k_shade_queues with --import-source on (hot lines)
#   prof_<workload>_frame[8]_<tag>.csv   the whole-frame kernel (k_frame) on the full image and on a 1/8 scanline partition
# then:  python profiles/make_summaries.py <tag> <output directory>
set -x
TAG=${1:-r02}
W=${2:-CornellBox}
COPIES=${3:-183}
OUT=${4:-ncu_out}
mkdir -p "$OUT"
NB=9; [ "$W" = CornellBox_Dragon ] && NB=17          # bounces 0..max_bounces
PER_FRAME=$((3 * NB))
ncu --set full --clock-control none -k regex:'k_trace_closest|k_shadow_accumulate|k_shade_queues' -s $PER_FRAME -c $PER_FRAME -f \
    -o $OUT/prof_${W}_${TAG} python tools/render_frames.py $W 2 0 1 $COPIES 0 > $OUT/ncu_${W}_${TAG}.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:'k_trace_closest|k_shade_queues' -s $((2 * NB + 2)) -c 2 -f \
    -o $OUT/prof_${W}_src_${TAG} python tools/render_frames.py $W 2 0 1 $COPIES 0 >> $OUT/ncu_${W}_${TAG}.log 2>&1
ncu --set full --clock-control none -k regex:k_frame -s 1 -c 1 -f \
    -o $OUT/prof_${W}_frame_${TAG} python tools/render_frames.py $W 2 1 1 $COPIES >> $OUT/ncu_${W}_${TAG}.log 2>&1
ncu --set full --clock-control none -k regex:k_frame -s 1 -c 1 -f \
    -o $OUT/prof_${W}_frame8_${TAG} python tools/render_frames.py $W 2 1 8 $COPIES >> $OUT/ncu_${W}_${TAG}.log 2>&1
# the raw pages are kept as CSV (the all-launch report is ~45 MB); the reports themselves are dropped except the small
# source-level one
for R in "" _frame _frame8; do
    ncu -i $OUT/prof_${W}${R}_${TAG}.ncu-rep --page raw --csv > $OUT/prof_${W}${R}_${TAG}.csv 2>> $OUT/ncu_${W}_${TAG}.log
    rm -f $OUT/prof_${W}${R}_${TAG}.ncu-rep
done
tail -3 $OUT/ncu_${W}_${TAG}.log
ls -la $OUT/prof_${W}_*
