#!/usr/bin/env bash
# Runs on a GPU machine: reference outputs + texture probe -> ref_out/ref1/
set -uo pipefail
cd "$(dirname "$0")/.."
O=ref_out/ref1; mkdir -p $O
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv > $O/gpu.txt 2>&1
nproc > $O/nproc.txt
R=$PWD/oracle/_ref
python -m popsift_b200.synth 256 192 3 $O/f256.pgm
python -m popsift_b200.synth 640 480 1 $O/f640.pgm
python -m popsift_b200.synth 1920 1080 100 $O/f1080.pgm
python -m popsift_b200.synth 3840 2160 7 $O/f4k.pgm
$R/texprobe pairs $O/tex_pairs.bin
$R/texprobe coords 640 480 1 $O/tex_c640.bin
$R/texprobe coords 3840 2160 1 $O/tex_c4k.bin
$R/texprobe coords 641 479 1 $O/tex_c641.bin
$R/texprobe coords 640 480 0 $O/tex_c640u0.bin
# planes (LogMode::All dumps into cwd)
( mkdir -p $O/log256 && cd $O/log256 && $R/ref_dump -i ../f256.pgm -o feat_vl_classic.bin --mode vlfeat --norm classic --log ) 2>&1 | tail -3
( cd $O/log256 && rm -rf dir-octave dir-dog dir-dog-txt dir-desc dir-fpt )
for run in a b; do
  $R/ref_dump -i $O/f640.pgm -o $O/f640_popsift_rs_$run.bin 2>&1 | tail -1
  $R/ref_dump -i $O/f640.pgm -o $O/f640_vlfeat_classic_$run.bin --mode vlfeat --norm classic 2>&1 | tail -1
done
$R/ref_dump -i $O/f256.pgm -o $O/f256_popsift_rs.bin 2>&1 | tail -1
$R/ref_dump -i $O/f1080.pgm -o $O/f1080_popsift_rs.bin 2>&1 | tail -1
$R/ref_dump -i $O/f1080.pgm -o $O/f1080_vlfeat_classic.bin --mode vlfeat --norm classic 2>&1 | tail -1
$R/ref_dump -i $O/f640.pgm -o $O/f640_ds0.bin --downsampling 0 2>&1 | tail -1
$R/ref_dump -i $O/f4k.pgm --octaves 5 2>&1 | tail -1
# timings of the reference (wall, host buffers in/out)
$R/ref_dump -i $O/f1080.pgm --bench 20 3 > $O/bench_ref_1080.json 2>$O/bench_ref_1080.err
$R/ref_dump -i $O/f4k.pgm --octaves 5 --bench 10 3 > $O/bench_ref_4k.json 2>$O/bench_ref_4k.err
$R/ref_dump -i $O/f4k.pgm --octaves 5 --downsampling 0 --bench 10 3 > $O/bench_ref_4k_ds0.json 2>$O/bench_ref_4k_ds0.err
cat $O/bench_ref_*.json
rm -f $O/f4k.pgm $O/f1080.pgm
du -sh $O
