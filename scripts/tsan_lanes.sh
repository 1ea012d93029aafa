#!/bin/bash
# ThreadSanitizer run of the speculative multi-base path (row f1, S4PCS_LANES) WITHOUT a GPU: the reference's demo main,
# the product's C++ layer, the test-only oracle stand-in for libs4g and the oracle port compiled into one binary with
# -fsanitize=thread; hippo pair, 4 lanes (LANES=), optionally sharded over DEVICES= device contexts (S4PCS_DEVICES; NCCL=1: the library-side reduction of S4PCS_NCCL with its shard gate).  Prints the number of TSAN reports (expected 0) and the score (expected 0.64).
set -e
R="$(cd "$(dirname "$0")/.." && pwd)"
REF="${S4_REFERENCE_ROOT:-/root/reference}"
W="$(mktemp -d)"
python - "$R" "$W" <<'PY'
import sys
import numpy as np
h = np.load(sys.argv[1] + "/tests/golden/hippo.npz")
for nme, arr in (("a.obj", h["P"]), ("b.obj", h["Q"])):
    with open(sys.argv[2] + "/" + nme, "w") as f:
        for p in arr:
            f.write("v %.9g %.9g %.9g\n" % tuple(p))
PY
# C++17: the stand-in holds the restatements of the point-cloud utilities (oracle/*_port.cc), FPFH's with hex-float literals
g++ -std=c++17 -O1 -g -fsanitize=thread -fopenmp -w -I "$R/include" -I "$REF/3rdparty/Eigen" -I "$REF/demos" \
    "$REF/demos/Super4PCS/super4pcs_test.cc" "$R"/cpp/match4pcsBase.cc "$R"/cpp/super4pcs.cc "$R"/cpp/pair_order.cc "$R"/cpp/io.cc \
    "$R"/tests/stubs/s4g_oracle_shim.cc "$R"/oracle/port.cc "$R"/oracle/*_port.cc -o "$W/demo_tsan" -pthread
cd "$W"
S4PCS_NCCL=${NCCL:-0} S4PCS_DEVICES=${DEVICES:-1} S4PCS_LANES=${LANES:-4} OMP_NUM_THREADS=1 ./demo_tsan -i a.obj b.obj -o 0.7 -d 0.01 -t 1000 -n 200 -m mat.txt > log.txt 2>&1 || true
echo "tsan reports: $(grep -c 'WARNING: ThreadSanitizer' log.txt || true)"
tr "\r" "\n" < log.txt | grep -E "^Score"
