#!/bin/bash
# One-GPU validation of the tree on an H100: GPU tests, smoke(), both bench arms, block codecs alone,
# ncu launch list of the bench command, ncu --set full captures of the main kernels, memcheck on a subset of the tests.
#   bash tools/gpu_validate.sh r03a [DIR]      -> everything lands in DIR/r03a_* (DIR defaults to validate_out)
TAG=${1:-val}
OUT=${2:-validate_out}
mkdir -p "$OUT"
(time timeout 900 python -m pytest tests -m gpu -x -q --timeout 300) > $OUT/${TAG}_tests.log 2>&1
tail -4 $OUT/${TAG}_tests.log
timeout 120 python -c "import __graft_entry__ as g; g.smoke()" > $OUT/${TAG}_smoke.log 2>&1; tail -1 $OUT/${TAG}_smoke.log
python bench.py --impl reference --steps 5 --warmup 2 > $OUT/${TAG}_ref.json 2> $OUT/${TAG}_ref.err
python bench.py --steps 10 --warmup 3 > $OUT/${TAG}_bench.json 2> $OUT/${TAG}_bench.err
python tools/measure_block_codecs.py 32 > $OUT/${TAG}_block_codecs.json 2> $OUT/${TAG}_block_codecs.err
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"bc_|hap_|snappy_" -c 200 --csv --log-file $OUT/${TAG}_launches.csv \
    python bench.py --profile --steps 2 --warmup 3 > $OUT/${TAG}_ncu_launches.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:"snappy_encode_fragments|snappy_execute|bc_encode|hap_place" -c 8 \
    -o $OUT/${TAG}_prof python bench.py --profile --frames 64 --steps 1 --warmup 1 > $OUT/${TAG}_ncu_full.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"snappy_execute|snappy_index" -c 2 \
    -o $OUT/${TAG}_prof_noindex python bench.py --profile --no-index --frames 64 --steps 1 --warmup 1 > $OUT/${TAG}_ncu_full_noindex.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"bc_encode" -c 6 \
    -o $OUT/${TAG}_prof_codecs python tools/measure_block_codecs.py 8 > $OUT/${TAG}_ncu_codecs.log 2>&1
timeout 600 compute-sanitizer --tool memcheck python -m pytest tests/test_gpu_parity.py -q -x -k "fragment_index and Hap5 or offset_table or delivery_ring or header_walks" > $OUT/${TAG}_memcheck.log 2>&1
tail -3 $OUT/${TAG}_memcheck.log
head -c 400 $OUT/${TAG}_bench.json; echo
head -c 300 $OUT/${TAG}_ref.json; echo
# afterwards, without a GPU: tools/ncu_summary.py, tools/src_hotspots.py, tools/launch_summary.py and tools/ncu_traffic.py turn the
# reports in $OUT into summaries under profiles/ (local, git-ignored; bench.py reads profiles/traffic.json when present)
