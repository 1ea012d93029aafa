#!/bin/bash
# A/B of compile-time variants of k_verify on a GPU machine with nvcc: for every variant rebuild libs4g.so with
# S4G_NVCC_DEFINES, run the Verify parity tests (bit-exact counts against the oracle) and the headline bench without the CPU
# leg; the default build is restored at the end.  One JSON line per variant under ab_out/verify_ab.jsonl.
#   bash scripts/verify_ab.sh
#   VARIANTS='-DS4G_PROBE4|-DS4G_VERIFY_MIN_BLOCKS=10' bash scripts/verify_ab.sh        ('|' separates variants)
# Knobs (super4pcs_b200/csrc/verify.cu): S4G_PROBE4 (four P points in flight per probe iteration instead of two),
# S4G_VERIFY_MIN_BLOCKS (launch bound: resident CTAs per SM the register allocation aims at, default 16),
# S4G_QUEUE_CAP (shared-memory queue entries per round, default 3072).
cd "$(dirname "$0")/.."
mkdir -p ab_out
OUT=${OUT:-ab_out/verify_ab.jsonl}
: > "$OUT"
IFS='|' read -r -a LIST <<< "${VARIANTS:-|-DS4G_PROBE4|-DS4G_VERIFY_MIN_BLOCKS=8|-DS4G_VERIFY_MIN_BLOCKS=10|-DS4G_VERIFY_MIN_BLOCKS=12|-DS4G_QUEUE_CAP=2048|-DS4G_QUEUE_CAP=4096|-DS4G_PROBE4 -DS4G_VERIFY_MIN_BLOCKS=10}"
for v in "${LIST[@]}"; do
  echo "== variant: '${v:-default}'"
  if ! S4G_NVCC_DEFINES="$v" timeout 300 python -c "from super4pcs_b200 import build; build.build_lib()" > ab_out/ab_build.log 2>&1; then
    echo "{\"variant\": \"$v\", \"error\": \"build failed\"}" >> "$OUT"; tail -3 ab_out/ab_build.log; continue
  fi
  # the test fixture rebuilds a stale library: keep the same defines in its environment
  if ! S4G_NVCC_DEFINES="$v" timeout 600 python -m pytest ${TESTS:-tests/test_verify_gpu.py} -x -q -m gpu > ab_out/ab_tests.log 2>&1; then
    echo "{\"variant\": \"$v\", \"error\": \"parity tests failed\"}" >> "$OUT"; tail -5 ab_out/ab_tests.log; continue
  fi
  S4G_NVCC_DEFINES="$v" timeout 300 python bench.py --steps 10 --warmup 3 --no-cpu-baseline 2> ab_out/ab_bench.err | tail -1 |
    V="$v" python -c "import json,os,sys; d=json.loads(sys.stdin.read()); print(json.dumps({'variant': os.environ['V'] or 'default', 'value': d['value'], 'ms_per_step': d['ms_per_step'], 'kernel_ms': d['roofline']['kernel_ms'], 'e2e': d['e2e']['value'], 'sm_mhz': (d.get('clocks') or {}).get('sm_mhz')}))" >> "$OUT" ||
    echo "{\"variant\": \"$v\", \"error\": \"bench failed\"}" >> "$OUT"
  tail -1 "$OUT"
done
timeout 300 python -c "from super4pcs_b200 import build; build.build_lib()" > /dev/null 2>&1    # back to the default build
echo "== summary"; cat "$OUT"
