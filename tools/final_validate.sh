#!/bin/bash
# Validation on one H100: GPU tests, smoke, the default bench line (both arms), two ncu captures of the search kernel.
# Outputs: ${TAG}_* in the output directory below.
TAG=${1:-r2}
mkdir -p gpurun_out
O=gpurun_out/$TAG
timeout 600 python -m pytest tests -q -m gpu 2>&1 | tail -5 > ${O}_pytest_gpu.log; cat ${O}_pytest_gpu.log
# the small test corpora are dense: by default most of their queries are handed back to the plain kernel — once more with
# every eligible query forced through the seeded kernel
BM25X_SEED_FORCE=1 timeout 600 python -m pytest tests/test_gpu_parity.py tests/test_gpu_paths.py tests/test_gpu_margins.py tests/test_gpu_margin_paths.py tests/test_gpu_prune_points.py tests/test_gpu_zx_stress.py tests/test_gpu_zz_growing.py tests/test_gpu_growing_segment.py tests/test_gpu_seal.py tests/test_gpu_segment_steps.py tests/test_gpu_segment_kinds.py tests/test_gpu_zy_segment_scale.py tests/test_gpu_batch.py -q -m gpu 2>&1 | tail -3 > ${O}_pytest_gpu_seed_forced.log; cat ${O}_pytest_gpu_seed_forced.log
timeout 60 python -c "import __graft_entry__ as g; g.smoke()" > ${O}_smoke.log 2>&1; tail -1 ${O}_smoke.log
timeout 300 python bench.py --impl reference --steps 5 --warmup 2 > ${O}_bench_ref.json 2> ${O}_bench_ref.err; echo "ref rc=$?"
timeout 300 python bench.py > ${O}_bench_c3.json 2> ${O}_bench_c3.err; echo "bench rc=$?"
timeout 200 ncu --set full --clock-control none --import-source on -k regex:k_search_ring -s 2 -c 1 -f -o gpurun_out/prof_$TAG \
    python bench.py --steps 1 --warmup 2 --no-cpu-baseline --no-strong --queries 20000 > ${O}_ncu_full.log 2>&1; echo "ncu full rc=$?"
timeout 300 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none -c 400 --csv \
    --log-file ${O}_launches.csv python bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-strong > ${O}_ncu_b.log 2>&1; echo "ncu list rc=$?"
python - <<PY
import json
for w in ("c3", "ref"):
    try:
        l = json.loads(open("${O}_bench_%s.json" % w).read().strip().splitlines()[-1])
        print(w, round(l["value"]), "q/s", round(l["ms_per_step"], 3), "ms", "e2e", round(l["e2e"]["value"]), l.get("roofline", {}).get("frac"),
              l["cpu_baseline"] and (round(l["cpu_baseline"]["value"]), l["cpu_baseline"]["cores"]), l.get("top100"), l.get("clocks"))
    except Exception as e:
        print(w, "failed", e)
PY
