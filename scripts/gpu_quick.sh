#!/bin/bash
# quick GPU check: all parity tests, then the short headline bench (per-kernel times) of the default library
mkdir -p gpurun_out
if [ -z "${SKIP_TESTS:-}" ]; then python -m pytest tests -m gpu -q -x 2>&1 | tail -8 > gpurun_out/pytest_quick.log; tail -3 gpurun_out/pytest_quick.log; fi
one() {
    python bench.py --no-cpu-baseline --no-e2e --no-other-configs --cfo-hz 0 --steps 10 > gpurun_out/bench_var_$1.json 2> gpurun_out/bench_var_$1.err
    python - "$1" <<'PY'
import json, sys
lib = sys.argv[1]
try:
    d = json.loads(open(f"gpurun_out/bench_var_{lib}.json").read().strip().splitlines()[-1]); k = d["kernels"]
    print(lib, "|", round(d["value"]), "frames/s", round(d["ms_per_step"], 3), "ms/step | ofdm frac", round(d["roofline"]["frac"], 4), "|",
          " ".join(f"{n.replace('_kernel', '')} {v['ms_per_step']:.3f}" for n, v in k.items() if v["ms_per_step"] >= 0.02), flush=True)
except Exception as e:
    print(lib, "| bench failed:", e, flush=True)
PY
}
unset DABB_LIB
one default
