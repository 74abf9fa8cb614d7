# run from the repository root after __graft_entry__.build(), on one H100 80GB HBM3 (700 W power limit)
python tools/chunks_bench.py --reps 50 > profiles/h100_chunks/chunks_bench.txt 2>&1
# bench.py, parent commit (its own checkout, built the same way) and this change, alternated three times
python bench.py --gpus 1 --steps 2000 --warmup 20 > profiles/h100_chunks/bench_par_$i.json   # parent
python bench.py --gpus 1 --steps 2000 --warmup 20 > profiles/h100_chunks/bench_new_$i.json   # this change
# chunks_bench_staged_reader.txt: the same tool on the first design of k_chunks_scatter, which staged each warp's 32
# chunks in shared memory, with a section timing that kernel against the plain per-lane reader kept here
# (DESIGN.md §8g).  The saved outputs omit torch.profiler's two-line warning and an nvcc remark.
