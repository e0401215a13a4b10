# tuning sweep (run under gpurun): prints us/step for the headline workload
run() { env "$@" python bench.py --steps 480 --warmup 20 --cpu-budget 0.1 --no-sweep > gpurun_out/b.json 2> gpurun_out/b.err; python - "$*" <<PY
import json,sys
try:
    j=json.load(open("gpurun_out/b.json")); print(sys.argv[1], "us/step", round(1e3*j["ms_per_step"],3), "frac", round(j["roofline"]["frac"],3), "parity", j["parity_vs_oracle"])
except Exception as ex: print(sys.argv[1], "FAILED", ex, open("gpurun_out/b.err").read()[-500:])
PY
}
for t in 0 24 48 96; do run EGPU_ROWS_PER_THREAD=$t; done  # 0 = the built-in rule
