#!/bin/bash
# Sanitizer runs (SURVEY 5.2).  CPU side: BB_SANITIZE=asan|tsan python build.py && pytest (or the tsan'd bb-bench
# control).  GPU side (needs an H100): compute-sanitizer over bench/sanitize_target.py, one tool per run.
#   scripts/sanitize.sh [memcheck|synccheck|racecheck|initcheck] [out_dir]
set -u
TOOL=${1:-memcheck}
OUT=${2:-build/sanitize}
mkdir -p "$OUT"
exec compute-sanitizer --tool "$TOOL" --print-limit 20 --error-exitcode 9 python bench/sanitize_target.py > "$OUT/sanitize_$TOOL.log" 2>&1
