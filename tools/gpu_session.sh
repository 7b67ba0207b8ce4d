#!/bin/bash
# One parameterised GPU session script (replaces the per-session scripts of round 1).  Run through gpurun from the
# repo root:   gpurun --timeout 1500 -- 'bash tools/gpu_session.sh <step> [<step> ...]'
# Every step writes its artefacts to gpurun_out/ (merged back into the build container); summaries that matter are
# copied to profiles/ by hand afterwards.  Steps:
#   tests        python -m pytest tests -m gpu            -> r02_pytest_gpu.log
#   bench        the default bench line + the reference arm   -> r02_bench.json, r02_bench_reference.json
#   chain        tests/programs/resident_chain.py, 3 parties, n = 10^6: off / install / resident   -> r02_chain.jsonl
#   demos        np_aes / np_cnnmnist timings with and without the engine                          -> r02_demos.txt
#   ncu_<cfg>    launch list + one --set full capture of the split/recombine kernels of a bench config
#   scale_N      (gpurun --gpus N) the driver's N-GPU launch line: multi_selftest, gather timing, e2e over all ranks; N=2 also tests/test_gpu_multi.py
#   overlap      tools/time_e2e_overlap.py at three pipeline chunk sizes
#   variants_<cfg>  bench a config with every libmpyc_b200_*.so tuning build present
#   local        K6 protocol-local kernels: tests/test_gpu_local.py, tools/time_local.py, ncu capture of k_bits_compose
#   demos2       np_cnnmnist -M3 (batch 1 and 4) with / without the engine, -M7 -T3 256-bit with the engine
#   localncu     ncu --set full of the K6 elementwise / matrix kernels (tools/time_local.py --ncu-all)
#   compare      tests/programs/resident_compare.py (np_sgn / np_trunc through the runtime), 3 parties: off vs resident
#   sass         per-kernel SASS / ptxas summary (no GPU needed, also runs in the build container)
set -u
OUT=gpurun_out
mkdir -p $OUT
export PYTHONDONTWRITEBYTECODE=1
REFDIR=$PWD/oracle/_ref        # build() with MPYC_REFERENCE set (oracle/reference.py)
launcher() { MPYC_REFERENCE=$REFDIR python tests/run_installed.py "$@"; }

for step in "$@"; do
  echo "=== step $step"
  case $step in
    tests)
      python -m pytest tests -m gpu -q -x 2>&1 | tail -60 > $OUT/r02_pytest_gpu.log; tail -3 $OUT/r02_pytest_gpu.log ;;
    bench)
      python bench.py > $OUT/r02_bench.json 2> $OUT/r02_bench.err; tail -c 1500 $OUT/r02_bench.json
      python bench.py --impl reference --steps 3 --warmup 1 > $OUT/r02_bench_reference.json 2>> $OUT/r02_bench.err; tail -c 600 $OUT/r02_bench_reference.json ;;
    chain)
      : > $OUT/r02_chain.jsonl
      for n in 100000 1000000; do
        for h in off install install,limb_wire install,resident; do
          echo "# harness=$h n=$n" >> $OUT/r02_chain.jsonl
          MPYC_B200_HARNESS=$h launcher tests/programs/resident_chain.py $n -M3 -B $((15000 + RANDOM % 2000)) --no-log 2>&1 | tail -n 1 >> $OUT/r02_chain.jsonl
        done
      done
      cat $OUT/r02_chain.jsonl ;;
    demos)
      # BASELINE configs[3] / configs[4] as the reference ships them (unmodified demos), with and without the engine;
      # configs[4]'s 256-bit m=7 t=3 variant through MPYC_B200_FORCE_PRIME (SecInt/SecFxp accept p=, sectypes.py:685-718)
      : > $OUT/r02_demos.txt
      P256=0xffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff43
      cd $REFDIR/_checkout/demos
      run_demo() {   # label, harness, extra env, args...
        label=$1; h=$2; extra=$3; shift 3
        s=$(date +%s.%N)
        res=$(env $extra MPYC_B200_OPS_MIN_SIZE=256 MPYC_B200_HARNESS=$h MPYC_REFERENCE=$REFDIR timeout 1500 python $OLDPWD/tests/run_installed.py "$@" -B $((15000 + RANDOM % 2000)) --no-log 2>&1 | tail -n 2 | tr '\n' ' ')
        e=$(date +%s.%N)
        echo "$label | harness=$h | wall=$(python -c "print(round($e - $s, 2))") s | $res" >> $OLDPWD/$OUT/r02_demos.txt
      }
      for h in off install install,resident; do
        run_demo "np_aes 1 party" $h "X=1" np_aes.py -1
        run_demo "np_aes -M3" $h "X=1" np_aes.py -1 -M3
        run_demo "np_cnnmnist -M3 (69-bit default field)" $h "X=1" np_cnnmnist.py 1 0 -M3
      done
      for h in off install,resident,spread; do
        run_demo "np_cnnmnist -M7 -T3 256-bit prime (configs[4])" $h "MPYC_B200_FORCE_PRIME=$P256" np_cnnmnist.py 1 0 -M7 -T3
      done
      cd $OLDPWD; cat $OUT/r02_demos.txt ;;
    ncu_*)
      cfg=${step#ncu_}
      QUICK="--no-cpu --no-e2e --no-extras --sustain 0"
      ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $OUT/r02_launches_$cfg.csv \
          python bench.py --config $cfg --steps 2 --warmup 3 $QUICK > $OUT/r02_ncu_$cfg.log 2>&1
      case $cfg in prss) kernels="k_prss";; modmul*) kernels="k_binop";; *) kernels="k_split k_recombine";; esac
      for k in $kernels; do
        ncu --set full --clock-control none -k regex:$k -s 3 -c 1 -o $OUT/r02_ncu_${cfg}_$k -f \
            python bench.py --config $cfg --steps 1 --warmup 3 $QUICK >> $OUT/r02_ncu_$cfg.log 2>&1 || true
        python tools/ncu_summary.py $OUT/r02_ncu_${cfg}_$k.ncu-rep $OUT/r02_ncu_${k#k_}_$cfg.txt > /dev/null 2>&1 || true
        ncu -i $OUT/r02_ncu_${cfg}_$k.ncu-rep --page details --csv > $OUT/r02_ncu_${cfg}_${k}_details.csv 2>/dev/null || true
        ncu -i $OUT/r02_ncu_${cfg}_$k.ncu-rep --page raw --csv > $OUT/r02_ncu_${cfg}_${k}_raw.csv 2>/dev/null || true
        rm -f $OUT/r02_ncu_${cfg}_$k.ncu-rep      # 35-55 MB each: only the extracted pages travel back (gpurun_out is capped at 64 MiB)
      done ;;
    scale_*)
      # gpurun --gpus N -- 'bash tools/gpu_session.sh scale_N': the driver's launch line for N > 1, plus the 2-GPU tests
      N=${step#scale_}
      python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29517 bench.py \
          --gpus $N --steps 20 --warmup 5 > $OUT/r02_scale_n$N.json 2> $OUT/r02_scale_n$N.err
      tail -c 2500 $OUT/r02_scale_n$N.json; tail -5 $OUT/r02_scale_n$N.err
      python bench.py --impl reference --gpus $N --steps 3 --warmup 1 > $OUT/r02_scale_n${N}_reference.json 2>> $OUT/r02_scale_n$N.err
      if [ "$N" = "2" ]; then python -m pytest tests/test_gpu_multi.py -q -m gpu 2>&1 | tail -3 | tee $OUT/r02_pytest_multi.log; fi ;;
    overlap)
      : > $OUT/r02_e2e_overlap.jsonl
      for mb in 32 8 128; do MPYC_B200_CHUNK_MB=$mb python tools/time_e2e_overlap.py $mb >> $OUT/r02_e2e_overlap.jsonl 2>&1; done
      cat $OUT/r02_e2e_overlap.jsonl ;;
    variants_*)
      cfg=${step#variants_}
      for lib in libmpyc_b200.so $(cd mpyc_b200 && ls libmpyc_b200_*.so 2>/dev/null); do
        [ -f mpyc_b200/$lib ] || continue
        echo "# $lib" >> $OUT/r02_variants_$cfg.txt
        MPYC_B200_LIB=$lib python bench.py --config $cfg --steps 10 --no-cpu --no-e2e --no-extras --sustain 0 2>&1 | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); r=d['roofline']; print(r['kernel'], round(r['frac'],4), round(r['ms'],4), 'rec', round(r.get('recombine',{}).get('frac',0),4), 'value', d['value'])" >> $OUT/r02_variants_$cfg.txt 2>&1
      done; cat $OUT/r02_variants_$cfg.txt ;;
    local)
      # the protocol-local kernels (K6): parity tests, timings, one ncu --set full capture of k_bits_compose
      bash tools/gpu_local_session.sh ;;
    demos2)
      # np_cnnmnist with the engine (resident + local algebra) after the K6 work, and the plain reference on the same box
      : > $OUT/r02_demos2.txt
      P256=0xffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff43
      cd $REFDIR/_checkout/demos
      run_demo2() {   # label, harness, extra env, args...
        label=$1; h=$2; extra=$3; shift 3
        s=$(date +%s.%N)
        res=$(env $extra MPYC_B200_STATS=1 MPYC_B200_OPS_MIN_SIZE=256 MPYC_B200_HARNESS=$h MPYC_REFERENCE=$REFDIR timeout 900 python $OLDPWD/tests/run_installed.py "$@" -B $((15000 + RANDOM % 2000)) --no-log 2>&1 | grep -E "predicted|pid\": 0|^ *\[|^ *-?[0-9]" | tail -n 4 | tr '\n' ' ')
        e=$(date +%s.%N)
        echo "$label | harness=$h | wall=$(python -c "print(round($e - $s, 2))") s | $res" >> $OLDPWD/$OUT/r02_demos2.txt
      }
      run_demo2 "np_cnnmnist -M3 (69-bit default field)" off "X=1" np_cnnmnist.py 1 0 -M3
      run_demo2 "np_cnnmnist -M3 (69-bit default field)" install,resident "X=1" np_cnnmnist.py 1 0 -M3
      run_demo2 "np_cnnmnist -M3 batch 4" off "X=1" np_cnnmnist.py 4 0 -M3
      run_demo2 "np_cnnmnist -M3 batch 4" install,resident "X=1" np_cnnmnist.py 4 0 -M3
      run_demo2 "np_cnnmnist -M7 -T3 256-bit prime (configs[4])" install,resident,spread "MPYC_B200_FORCE_PRIME=$P256" np_cnnmnist.py 1 0 -M7 -T3
      cd $OLDPWD; cat $OUT/r02_demos2.txt ;;
    localncu)
      # one ncu --set full capture per K6 elementwise / matrix kernel (second launch of each), 128-bit field
      ncu --set full --clock-control none -k regex:"k_fma|k_axpb|k_low_bits|k_nonzero|k_bits_decompose|k_transpose|k_scan_cols|k_scan_rows|k_binop_rows" \
          -o $OUT/r02_ncu_local -f python tools/time_local.py --ncu-all > $OUT/r02_ncu_local.log 2>&1
      python tools/ncu_summary.py $OUT/r02_ncu_local.ncu-rep $OUT/r02_ncu_local.txt > /dev/null 2>&1 || true
      rm -f $OUT/r02_ncu_local.ncu-rep
      grep -E "^kernel|gpu__time_duration|dram__bytes_read.sum |dram__bytes_write.sum |gpu__dram_throughput" $OUT/r02_ncu_local.txt | head -80 ;;
    compare)
      # secure comparison (np_sgn) and fixed-point product (np_trunc) through the unmodified runtime, 3 parties on one GPU
      : > $OUT/r02_compare.jsonl
      for n in 20000 100000; do
        for h in off install,resident; do
          if [ "$h" = "off" ] && [ "$n" != "20000" ]; then continue; fi
          echo "# harness=$h n=$n" >> $OUT/r02_compare.jsonl
          MPYC_B200_OPS_MIN_SIZE=256 MPYC_B200_HARNESS=$h launcher tests/programs/resident_compare.py $n -M3 -B $((15000 + RANDOM % 2000)) --no-log 2>&1 | tail -n 1 >> $OUT/r02_compare.jsonl
        done
      done
      cat $OUT/r02_compare.jsonl ;;
    sass)
      python tools/sass_summary.py > $OUT/r02_sass_summary.txt 2>&1; tail -5 $OUT/r02_sass_summary.txt ;;
    *) echo "unknown step $step" ;;
  esac
done
