#!/bin/bash
# compute-sanitizer memcheck + racecheck over profiles/sanitize_cases.py (on a GPU machine, from the repo root):
#   bash profiles/sanitize.sh tag      -> profiles/out/tag_{memcheck,racecheck}.log (+ one-line summaries on stdout)
tag=${1:-rXX}
mkdir -p profiles/out
for tool in memcheck racecheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 python profiles/sanitize_cases.py > profiles/out/${tag}_$tool.log 2>&1
  echo "$tool rc=$? : $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|SANITIZE_CASES_OK' profiles/out/${tag}_$tool.log | tr '\n' ' ')"
done
