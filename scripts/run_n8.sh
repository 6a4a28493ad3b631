#!/bin/bash
# One-node multi-GPU validation + numbers: NP=8 scripts/run_n8.sh   (writes ${OUT:-run_n8_out}/n${NP}_*.log)
cd "$(dirname "$0")/.."
NP=${NP:-8}
OUTDIR=${OUT:-run_n8_out}
mkdir -p $OUTDIR
TRP="python -m torch.distributed.run --nnodes=1 --nproc-per-node $NP --master-addr 127.0.0.1"
F='^\*\|OMP_NUM\|^$\|W09'
O=$OUTDIR/n${NP}
echo "== parity (python, oracle-checked)"; timeout 400 $TRP --master-port 29701 tests/test_multi_gpu.py 2>&1 | grep -v "$F" | tee ${O}_multigpu_parity.log | tail -16
echo "== timeline"; timeout 200 $TRP --master-port 29709 scripts/trace_timeline.py 2>&1 | grep "trace rank [07]" | tee ${O}_trace.log | grep "rank 0"
echo "== bench"; timeout 500 $TRP --master-port 29702 bench.py --gpus $NP --steps 5 --warmup 3 2>&1 | grep -v "$F" | tail -2 | tee ${O}_bench.json | cut -c1-3500
echo "== bench, fused partition+exchange (A/B)"; DJ_EXCHANGE=fused timeout 300 $TRP --master-port 29712 bench.py --gpus $NP --steps 5 --warmup 3 --no-e2e --no-parity 2>&1 | grep -v "$F" | tail -2 | tee ${O}_bench_fused.json | cut -c1-1500
cd distributed-join_b200
TR="$TRP --no-python"
echo "== C++ compare_against_single_gpu"; timeout 300 $TR --master-port 29706 bin/compare_against_single_gpu 2>&1 | grep -v "$F" | tee ../${O}_compare_single_gpu.log | tail -6
echo "== C++ compare_against_analytical + test_shuffle_on"; (timeout 200 $TR --master-port 29707 bin/compare_against_analytical; timeout 200 $TR --master-port 29708 bin/test_shuffle_on) 2>&1 | grep -v "$F" | tee ../${O}_cpp_tests.log | tail -4
echo "== shuffle_on (config 4)"; timeout 300 $TR --master-port 29704 bin/shuffle_on --nrows ${SHUFFLE_ROWS:-400000000} --iterations 3 2>&1 | grep -v "$F" | tee ../${O}_shuffle_on.log | tail -4
echo "== distributed_join (config 5: duplicates, sel 0.9, odf 4)"; timeout 400 $TR --master-port 29705 bin/distributed_join --build-table-nrows 100000000 --probe-table-nrows 400000000 --selectivity 0.9 --duplicate-build-keys --over-decomposition-factor 4 --nvlink-domain-size $NP --iterations 3 2>&1 | grep -v "$F" | grep "Elasped\|benchmark\|ERROR" | tee ../${O}_join_cfg5.log | tail -6
if [ -n "$A2A" ]; then echo "== all_to_all (config 3)"; timeout 300 $TR --master-port 29703 bin/all_to_all --max-size 8192000000 2>&1 | grep -v "$F" | tee ../${O}_all_to_all.log | tail -16; fi
