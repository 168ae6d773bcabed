#!/bin/bash
# On the GPU box: a short bench (headline config, no CPU / e2e / side measurements) for the default library and for every variant_*.so
# built by scripts/build_variants.sh, with the stage + pipeline parity tests for each variant.  One line per variant: frames/s, ms/step,
# ofdm_demod_kernel ms and roofline fraction, Viterbi ms.
mkdir -p gpurun_out
one() {   # label
    python bench.py --no-cpu-baseline --no-e2e --no-other-configs --cfo-hz 0 --steps 10 > gpurun_out/bench_var_$1.json 2> gpurun_out/bench_var_$1.err
    python - "$1" "$2" <<'PY'
import json, sys
lib, t = sys.argv[1], sys.argv[2]
try:
    d = json.loads(open(f"gpurun_out/bench_var_{lib}.json").read().strip().splitlines()[-1])
    k = d["kernels"]
    print(lib, "|", t, "|", round(d["value"]), "frames/s", round(d["ms_per_step"], 3), "ms/step | ofdm", round(d["roofline"]["ms_per_launch"], 4), "ms frac", round(d["roofline"]["frac"], 4),
          "survey-frac", round(d["roofline"]["frac_with_survey_bytes"], 4), "| viterbi FIC", round(k["viterbi_kernel(FIC)"]["ms_per_step"], 3), "MSC", round(k["viterbi_kernel(MSC)"]["ms_per_step"], 3), flush=True)
except Exception as e:
    print(lib, "|", t, "| bench failed:", e, flush=True)
PY
}
unset DABB_LIB
one default "-"
for lib in $(ls variant_*.so 2>/dev/null); do
    export DABB_LIB=$PWD/$lib
    t=$(python -m pytest tests/test_gpu_stages.py tests/test_gpu_pipeline.py -m gpu -q 2>&1 | tail -1)
    one "$lib" "$t"
done
