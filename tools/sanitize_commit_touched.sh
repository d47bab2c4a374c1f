#!/bin/bash
# tools/sanitize_commit_touched.sh: compute-sanitizer (memcheck, racecheck, synccheck) over bf_resident_commit_touched — the list
# build, the list-mode check, scan, rewrites and apply, and the due marks of touched ticks and schedules — through the twin-batch
# tests of tests/test_gpu_commit_touched.py (all four forms, full and listed calls, refusals, the list-length edges).  Prints the
# tools' summaries.
cd "$(dirname "$0")/.."
for tool in memcheck racecheck synccheck; do
  echo "== $tool"
  compute-sanitizer --tool $tool --print-limit 5 python -m pytest -q -p no:cacheprovider tests/test_gpu_commit_touched.py \
    -k "edges or 64-243" 2>&1 | tail -6
done
