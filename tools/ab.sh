#!/bin/bash
# A/B of library variants on ONE box (run under gpurun): tools/ab.sh lib1.so lib2.so ...  (names under faster_b200/lib;
# a name may carry bench flags after a colon, e.g. libfaster_b200.so:--single-stream).  Each variant: bench.py --quick (cfg4
# chain, resident + e2e); AB_ROUNDS rounds (default 2) to see the noise.
for round in $(seq 1 ${AB_ROUNDS:-2}); do
  for spec in "$@"; do
    lib=${spec%%:*}; flags=""; [[ "$spec" == *:* ]] && flags=${spec#*:}
    FQ_LIB=$PWD/faster_b200/lib/$lib python bench.py --steps ${AB_STEPS:-10} --quick $flags > gpurun_out/ab_tmp.json 2>gpurun_out/ab_tmp.err
    python - "$spec" <<'PY'
import json, sys
try:
    d = json.loads(open("gpurun_out/ab_tmp.json").read().strip().splitlines()[-1])
    print("%-44s resident %.2f M  e2e %.2f M  pass %.4f ms  (sm %s MHz)" %
          (sys.argv[1], d["value"] / 1e6, d["e2e"]["value"] / 1e6, d["ms_per_pass"], d["clocks"]["sm_mhz"]))
except Exception as e:
    print(sys.argv[1], "FAILED", e, open("gpurun_out/ab_tmp.err").read()[-400:])
PY
  done
done
