#!/bin/bash
# scripts/sanitize.sh -- compute-sanitizer evidence (needs a GPU and compute-sanitizer): memcheck over ALL GPU tests, racecheck over a subset
# that reaches every kernel: small and config-B windows (k_tri, k_jac with the blocked gate Cholesky, Gram kernels,
# the fused cluster tail with the ticket counters of k_jac / k_syrk), the large-window tail (L = 98), the device batch,
# the streaming path (propagate_n / augment / gather).  Logs go to the directory given as the first argument.
set -u
OUT=${1:?usage: scripts/sanitize.sh OUT_DIR}
timeout 1500 compute-sanitizer --tool memcheck --leak-check no --error-exitcode 9 --log-file $OUT/r02_memcheck.log \
  python -m pytest tests/test_engine_gpu.py tests/test_asl_gpu.py -m gpu -q -x > $OUT/r02_memcheck_pytest.log 2>&1
echo "memcheck exit $?" >> $OUT/r02_memcheck_pytest.log
# the side updates (k_aid on both storage paths, k_nees to 37 panels, k_lmk_* and k_lmk_set at their row, observation and
# group caps, device batches of 33 members)
timeout 1500 compute-sanitizer --tool memcheck --leak-check no --error-exitcode 9 --log-file $OUT/r02_memcheck_side.log \
  python -m pytest tests/test_side_shapes_gpu.py -m gpu -q -x > $OUT/r02_memcheck_side_pytest.log 2>&1
echo "memcheck exit $?" >> $OUT/r02_memcheck_side_pytest.log
SELR='window_fp64_vs_clean_oracle and not 300 or persistent_batch'
timeout 1500 compute-sanitizer --tool racecheck --racecheck-report all --error-exitcode 9 --log-file $OUT/r02_racecheck.log \
  python -m pytest tests/test_engine_gpu.py -m gpu -q -x -k "$SELR" > $OUT/r02_racecheck_pytest.log 2>&1
echo "racecheck exit $?" >> $OUT/r02_racecheck_pytest.log
tail -n 3 $OUT/r02_memcheck_pytest.log $OUT/r02_memcheck_side_pytest.log $OUT/r02_racecheck_pytest.log
tail -n 5 $OUT/r02_memcheck.log $OUT/r02_memcheck_side.log $OUT/r02_racecheck.log
# the consensus on mapped-landmark matches (k_lmk_hyp, k_lmk_cons, k_lmk_clone<..., CONS>) at every shape of its GPU tests
timeout 1500 compute-sanitizer --tool memcheck --leak-check no --error-exitcode 9 --log-file $OUT/r02_memcheck_consensus.log \
  python -m pytest tests/test_landmark_consensus_gpu.py -m gpu -q -x > $OUT/r02_memcheck_consensus_pytest.log 2>&1
echo "memcheck exit $?" >> $OUT/r02_memcheck_consensus_pytest.log
timeout 1500 compute-sanitizer --tool racecheck --racecheck-report all --error-exitcode 9 --log-file $OUT/r02_racecheck_consensus.log \
  python -m pytest tests/test_landmark_consensus_gpu.py -m gpu -q -x > $OUT/r02_racecheck_consensus_pytest.log 2>&1
echo "racecheck exit $?" >> $OUT/r02_racecheck_consensus_pytest.log
tail -n 3 $OUT/r02_memcheck_consensus_pytest.log $OUT/r02_racecheck_consensus_pytest.log
