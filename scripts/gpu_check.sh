#!/bin/bash
# Checks the whole tree on one GPU: the -m gpu suite (unbuffered, with the slowest tests listed: the CPU oracle of the
# full-size tests dominates), smoke(), the beam bench and a short bench, one log file per check.
#   bash scripts/gpu_check.sh
set -u
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
run() { name=$1; shift; echo "=== $name"; timeout ${TMO:-300} "$@" > gpurun_out/check_$name.log 2>&1; echo "exit $? ($name)"; tail -n ${TAILN:-4} gpurun_out/check_$name.log | cut -c1-1500; }
TMO=1100 TAILN=40 run suite python -u -m pytest tests -q --tb=short -m gpu --durations=15 -p no:cacheprovider
TAILN=3 run smoke python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')"
TAILN=1 run beam python scripts/beam_bench.py --max-new-tokens 512 --repeats 2
TAILN=1 run bench python bench.py --steps 2 --warmup 3 --max-new-tokens 512 --no-cpu-baseline --no-extras
