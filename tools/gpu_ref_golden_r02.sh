#!/usr/bin/env bash
# Runs on a GPU machine: round-2 reference outputs -> ref_out/ref2/
#   OpenCV SiftMode, float images (+ float texture probe), grid filter, descriptor modes, the brute-force
#   matcher (FeaturesDev::match) and device-resident results, the synthetic affine set (BASELINE configs[4]
#   stand-in), and the parity of the benchmark workload itself (tools/bench_parity.py).
# tests/golden/make_golden_r02.py turns the small files into committed fixtures.
set -uo pipefail
cd "$(dirname "$0")/.."
O=ref_out/ref2; mkdir -p $O
R=$PWD/oracle/_ref
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm --format=csv > $O/gpu.txt 2>&1
python -m popsift_b200.synth 256 192 3 $O/f256.pgm
python -m popsift_b200.synth 640 480 1 $O/f640.pgm
python -m popsift_b200.synth 640 480 2 $O/f640b.pgm
python -m popsift_b200.synth affine $O/aff
# --- OpenCV SiftMode (s_extrema.cu:236-284)
$R/ref_dump -i $O/f256.pgm -o $O/f256_opencv_classic.bin --mode opencv --norm classic 2>&1 | tail -1
$R/ref_dump -i $O/f640.pgm -o $O/f640_opencv_rs.bin --mode opencv 2>&1 | tail -1
# --- float images (s_image.cu:262-291; pixels = u8/256 as popsift-demo --float-mode)
$R/texprobe fpairs $O/tex_fpairs.bin
( mkdir -p $O/logf256 && cd $O/logf256 && $R/ref_dump -i ../f256.pgm -o feat.bin --mode vlfeat --norm classic --float-mode --log ) 2>&1 | tail -1
( cd $O/logf256 && rm -rf dir-octave dir-dog dir-dog-txt dir-desc dir-fpt dir-dog-dump && cd dir-octave-dump && ls | grep -v -e "-o-0-l-0" -e "-o-0-l-1" -e "-o-1-l-0" | xargs rm -f )
$R/ref_dump -i $O/f640.pgm -o $O/f640_float_vlfeat_classic.bin --mode vlfeat --norm classic --float-mode 2>&1 | tail -1
$R/ref_dump -i $O/f640.pgm -o $O/f640_float_ds0.bin --float-mode --downsampling 0 2>&1 | tail -1
# --- grid filter (s_filtergrid.cu:112-325)
for fm in 300 1000; do for g in 2 3; do for s in up down; do
  $R/ref_dump -i $O/f640.pgm -o $O/f640_filter_${fm}_${g}_${s}.bin --mode vlfeat --norm classic --filter-max-extrema $fm --filter-grid $g --filter-sort $s 2>&1 | tail -1
done; done; done
$R/ref_dump -i $O/f640.pgm -o $O/f640_filter_300_2_random.bin --mode vlfeat --norm classic --filter-max-extrema 300 --filter-grid 2 --filter-sort random 2>&1 | tail -1
# --- descriptor modes (s_desc_iloop.cu, s_desc_grid.cu, s_desc_igrid.cu, s_desc_notile.cu)
for dm in iloop grid igrid notile; do
  $R/ref_dump -i $O/f256.pgm -o $O/f256_desc_${dm}.bin --mode vlfeat --norm classic --desc-mode $dm 2>&1 | tail -1
done
# --- direct scaling (s_pyramid_build.cu:478-546)
$R/ref_dump -i $O/f256.pgm -o $O/f256_direct.bin --mode vlfeat --norm classic --direct-scaling 2>&1 | tail -1
# --- matcher + device-resident results (features.cu:187-304, sift_pyramid.cu:324-362)
$R/ref_dump -i $O/f640.pgm -i $O/f640b.pgm -o $O/match_640 --match > $O/match_640.txt 2>$O/match_640.err; tail -1 $O/match_640.err
$R/ref_dump -i $O/aff1.pgm -i $O/aff2.pgm -o $O/match_aff12 --mode vlfeat --norm classic --match > $O/match_aff12.txt 2>$O/match_aff12.err; tail -1 $O/match_aff12.err
# --- affine set, VLFeat mode (BASELINE configs[4] stand-in)
for k in 1 2 3 4 5 6; do
  $R/ref_dump -i $O/aff$k.pgm -o $O/aff${k}_vlfeat_classic.bin --mode vlfeat --norm classic 2>&1 | tail -1
done
# --- the benchmark workload itself: reference twice + this library, per-keypoint orientation diffs
python tools/bench_parity.py $O/bench_parity.json 32 > $O/bench_parity.log 2>&1; tail -3 $O/bench_parity.log
rm -f $O/*.pgm
du -sh $O
