# What a GPU session of this repo runs (one H100): the -m gpu tests, the smoke check and the default bench.
OUT=${OUT:-gpu_check_out}
mkdir -p "$OUT"
timeout 1500 python -m pytest tests -m gpu -q -x > "$OUT/pytest_gpu.log" 2>&1; echo "pytest rc=$?"; tail -4 "$OUT/pytest_gpu.log"
timeout 300 python __graft_entry__.py smoke 2>&1 | tail -6
timeout 900 python bench.py --steps 5 --warmup 3 > "$OUT/bench_n1.json" 2> "$OUT/bench_n1.err"; echo "bench rc=$?"; cut -c1-400 "$OUT/bench_n1.json"
