# experiment helper: run the bench with a few part counts of the class pipeline (one line each)
export KVIDX_BENCH_SKIP_CPU=1 KVIDX_BENCH_NOCHECK=1 KVIDX_BENCH_SKIP_MIXED=1
run() { python bench.py --steps 6 --warmup 3 2>/dev/null | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('$1', round(d['ms_per_step'],3))"; }
for pp in 6 8 10 12 16; do KVIDX_ROUNDS_PARTS=$pp run parts$pp; done
