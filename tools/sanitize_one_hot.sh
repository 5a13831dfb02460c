#!/bin/bash
# compute-sanitizer memcheck over the one-hot row commitments (tests/test_gpu_one_hot.py): the warp-aggregated counting
# sort, the row passes through the shared scan / accumulation / wide fold, the invalid-address flag and the error paths.
# The shapes at 2^22..2^26 cycles are left out (the same kernels, only longer).
# usage: tools/sanitize_one_hot.sh [LOG_DIR]   (default: the current directory; writes sanitizer_one_hot_memcheck.log)
LOG_DIR=${1:-.}
mkdir -p "$LOG_DIR"
LOG="$LOG_DIR/sanitizer_one_hot_memcheck.log"
SEL='(test_matches_oracle and (16-16 or 1024-2 or 16-256 or 2-1)) or skewed or agrees or errors'
timeout 600 compute-sanitizer --tool memcheck --leak-check no --error-exitcode 7 \
    python -m pytest tests/test_gpu_one_hot.py -q -x -k "$SEL" > "$LOG" 2>&1
echo "memcheck rc=$?" >> "$LOG"
tail -n 4 "$LOG"
