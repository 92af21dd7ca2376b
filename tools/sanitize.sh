#!/bin/bash
# Run on a GPU machine: compute-sanitizer over the parity tests that exercise the newest device code
# (pages cut at restart points, the overlap-merge pass, boolean pages, gorilla decode, tombstones, device CRC, error
# paths). memcheck slows kernels 10-50x, the selected tests use small arenas.
# Usage: bash tools/sanitize.sh [memcheck|racecheck|initcheck] [-k expression]
TOOL=${1:-memcheck}
SEL=${2:-"gorilla or tombstone or small or errors or crc or empty or maximum or predicates or pruning or concurrent or host_resident or decode or parts or malformed or merge or overlapping or bool"}
mkdir -p profile_out
compute-sanitizer --tool "$TOOL" --error-exitcode 1 --print-limit 20 \
  python -m pytest tests -m gpu -x -q -k "$SEL" > profile_out/sanitize_${TOOL}.log 2>&1
echo "exit $?"
grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|Invalid|Race" profile_out/sanitize_${TOOL}.log | tail -20
