# run from the repository root after __graft_entry__.build(), on one H100 80GB HBM3 (700 W power limit)
python tools/samples_bench.py --reps 50 > profiles/h100_samples/samples_bench.txt 2>&1
# (the saved output omits a two-line torch.profiler warning)
