# run from the repository root after __graft_entry__.build(), on one H100 80GB HBM3 (700 W power limit; gpu.txt was
# read in the same run)
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > profiles/h100_remap/gpu.txt
python tools/remap_bench.py --reps 50 > profiles/h100_remap/remap_bench.txt 2>&1
# bench.py, parent commit (its own checkout, built the same way) and this change, alternated twice
python bench.py --gpus 1 --steps 2000 --warmup 20 > profiles/h100_remap/bench_par_$i.json   # parent
python bench.py --gpus 1 --steps 2000 --warmup 20 > profiles/h100_remap/bench_new_$i.json   # this change
