# end-of-round evidence: full GPU suite, driver-shaped bench lines for every BASELINE config, launch list, ncu captures at the
# bench configuration.  gpurun copies back at most 64 MiB of gpurun_out/: every .ncu-rep is summarised ON THE BOX (key metrics as
# JSON + the top source lines) and deleted, except the dominant kernel's (KEEP_REP).  SKIP_TESTS=1 leaves pytest to another call.
set -x
R=${1:-r02}; O=gpurun_out
[ "${SKIP_TESTS:-0}" = 1 ] || python -m pytest tests -m gpu -q -x 2>&1 | tail -4
python bench.py --steps 10 --warmup 3 > $O/${R}_bench_config3_speed.json 2> $O/${R}_bench.err; tail -c 600 $O/${R}_bench_config3_speed.json
python bench.py --zstd-mode dense --steps 6 --warmup 3 --no-cpu-baseline > $O/${R}_bench_config3_dense.json 2>> $O/${R}_bench.err
python bench.py --corpus R --steps 6 --warmup 3 --no-cpu-baseline > $O/${R}_bench_config3_R.json 2>> $O/${R}_bench.err
python bench.py --config 0 --steps 3 --warmup 1 > $O/${R}_bench_config0.json 2>> $O/${R}_bench.err
python bench.py --config 1 --steps 6 --warmup 3 --no-cpu-baseline > $O/${R}_bench_config1.json 2>> $O/${R}_bench.err
python bench.py --config 2 --steps 6 --warmup 3 --no-cpu-baseline > $O/${R}_bench_config2.json 2>> $O/${R}_bench.err
python bench.py --config 4 --steps 16 --warmup 3 > $O/${R}_bench_config4_own.json 2>> $O/${R}_bench.err
python bench.py --config 4 --frames libzstd --steps 16 --warmup 3 > $O/${R}_bench_config4_libzstd.json 2>> $O/${R}_bench.err
python bench.py --config 4 --zstd-mode dense --steps 16 --warmup 3 --no-cpu-baseline > $O/${R}_bench_config4_own_dense.json 2>> $O/${R}_bench.err
python bench.py --config 4 --window-mib 1024 --steps 4 --warmup 3 --no-cpu-baseline > $O/${R}_bench_bulk_fetch_own.json 2>> $O/${R}_bench.err
python bench.py --config 4 --window-mib 1024 --zstd-mode dense --steps 4 --warmup 3 --no-cpu-baseline > $O/${R}_bench_bulk_fetch_own_dense.json 2>> $O/${R}_bench.err
python bench.py --impl reference --steps 3 --warmup 1 > $O/${R}_bench_reference.json 2>> $O/${R}_bench.err; tail -c 500 $O/${R}_bench_reference.json
python tests/perf/bench_detransform.py 256 > $O/${R}_detransform.json 2>> $O/${R}_bench.err
python scripts/pcie_ceiling.py > $O/${R}_pcie_ceiling_1rank.json 2>> $O/${R}_bench.err; cat $O/${R}_pcie_ceiling_1rank.json
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 80 --csv --log-file $O/${R}_launches.csv python bench.py --steps 2 --warmup 1 --no-e2e --no-cpu-baseline --no-verify > /dev/null 2>&1
# cap NAME KERNEL_REGEX COUNT -- command: one `ncu --set full` report, summarised here, deleted unless NAME is in KEEP_REP
KEEP_REP=${KEEP_REP:-zstd_enc_blocks}
cap() {
  name=$1; rx=$2; cnt=$3; shift 4
  timeout 900 ncu --set full --clock-control none --import-source on -k "regex:$rx" -s ${SKIPK:-1} -c $cnt -o $O/prof_${R}_$name -f "$@" > /dev/null 2>&1
  rep=$O/prof_${R}_$name.ncu-rep
  [ -f $rep ] || { echo "no report for $name"; return; }
  python scripts/ncu_summary.py $rep $O/${R}_$name.ncu.json > /dev/null
  ncu -i $rep --page source --csv --print-source cuda,sass > /tmp/src_$name.csv 2>/dev/null
  python scripts/ncu_by_line.py /tmp/src_$name.csv 60 > $O/${R}_$name.by_line.txt 2>&1
  case " $KEEP_REP " in *" $name "*) ;; *) rm -f $rep;; esac
}
cap zstd_enc_blocks zstd_enc_blocks 1 -- python bench.py --steps 1 --warmup 1 --no-e2e --no-cpu-baseline --no-verify
cap zstd_enc_regions zstd_enc_regions 1 -- python bench.py --zstd-mode dense --steps 1 --warmup 1 --no-e2e --no-cpu-baseline --no-verify
cap gcm_main gcm_main 1 -- python bench.py --steps 1 --warmup 1 --no-e2e --no-cpu-baseline --no-verify
SKIPK=3 cap zstd_dec_blk 'zstd_dec_blk_literals|zstd_dec_blk_sequences|zstd_dec_indep_execute' 3 -- python tests/perf/bench_detransform.py 256
cap zstd_dec_regions zstd_dec_regions 1 -- python bench.py --direction fetch --frames own --zstd-mode dense --segment-mib 256 --window-mib 256 --steps 1 --warmup 1 --no-e2e --no-cpu-baseline
SKIPK=0 cap zstd_dec_libzstd 'zstd_dec_par_entropy|zstd_dec_par_execute' 2 -- python bench.py --direction fetch --frames libzstd --steps 1 --warmup 0 --no-e2e --no-cpu-baseline --segment-mib 64
# compute-sanitizer over the smoke invocation (both compressors, every decode path, AES both ways): logs go to the output directory
timeout 420 compute-sanitizer --tool memcheck --log-file $O/${R}_sanitizer_memcheck.log python -c "import __graft_entry__ as g; g.smoke()" > $O/${R}_sanitizer_memcheck.out 2>&1; echo "memcheck exit $?" >> $O/${R}_sanitizer_memcheck.out
timeout 420 compute-sanitizer --tool racecheck --log-file $O/${R}_sanitizer_racecheck.log python -c "import __graft_entry__ as g; g.smoke()" > $O/${R}_sanitizer_racecheck.out 2>&1; echo "racecheck exit $?" >> $O/${R}_sanitizer_racecheck.out
for f in $O/${R}_sanitizer_memcheck.log $O/${R}_sanitizer_racecheck.log; do tail -n 3 $f; done
du -sh $O; ls -la $O | grep ${R} | tail -40; tail -5 $O/${R}_bench.err
