#!/bin/bash
# compute-sanitizer over a small slice of the GPU suite (memcheck + racecheck); results in $OUT/sanitize_*.log
# usage: tools/sanitize.sh [OUT]   (default: a directory under ${TMPDIR:-/tmp})
set -u
OUT=${1:-${TMPDIR:-/tmp}/kvz_sanitize}
mkdir -p "$OUT"
SEL='tests/test_framepass.py::test_cuda_frame_pass_matches_reference tests/test_deblock.py tests/test_interpass.py'
K='dims6 or dims7 or dims0 or case0 or case3 or 10bit or inter'
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 --log-file "$OUT"/sanitize_memcheck.log python -m pytest $SEL -m gpu -x -q -k "$K" > "$OUT"/sanitize_memcheck_pytest.txt 2>&1; echo "memcheck rc=$?"
tail -3 "$OUT"/sanitize_memcheck_pytest.txt; tail -5 "$OUT"/sanitize_memcheck.log
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 9 --log-file "$OUT"/sanitize_racecheck.log python -m pytest tests/test_framepass.py::test_cuda_frame_pass_matches_reference tests/test_rdoq.py -m gpu -x -q -k "dims6 or (vs_reference and 16-27-0-1) or (coeff_cost and 16-0-1-1)" > "$OUT"/sanitize_racecheck_pytest.txt 2>&1; echo "racecheck rc=$?"
tail -3 "$OUT"/sanitize_racecheck_pytest.txt; tail -8 "$OUT"/sanitize_racecheck.log
