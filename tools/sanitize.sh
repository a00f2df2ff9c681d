#!/usr/bin/env bash
# compute-sanitizer over the TINY decode / prefill / batch paths (SURVEY.md section 5), on a machine with a GPU:
#   bash tools/sanitize.sh
# Output: profiles/sanitizer_{memcheck,racecheck,synccheck}_engine{1,0}.txt (profiles/ output is not committed).
set -u
mkdir -p profiles
for eng in 1 0; do
for tool in memcheck racecheck synccheck; do
  f=profiles/sanitizer_${tool}_engine${eng}.txt
  echo "== LNB_ENGINE=$eng compute-sanitizer --tool $tool" > $f
  LNB_ENGINE=$eng LNB_P2P_TIMEOUT_MS=0 timeout 300 compute-sanitizer --tool $tool --print-limit 30 python tools/sanitize_run.py >> $f 2>&1
  echo "exit code $?" >> $f
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY|sanitize_run\]|exit code" $f | tail -6
done
done
