#!/bin/bash
# The ring-session suite and its neighbours on one H100, smoke(), and the card's name and power limit.
# Run from the repository root after __graft_entry__.build().
set -o pipefail
out=${OUT:-profiles/h100_ring_session}; mkdir -p $out
nvidia-smi --query-gpu=name,power.limit --format=csv > $out/gpu.txt
python -m pytest -q -m gpu -p no:cacheprovider tests/test_gpu_session_ring.py tests/test_gpu_session.py \
    tests/test_gpu_resident*.py tests/test_gpu_chunks.py tests/test_gpu_samples.py --durations=15 2>&1 | tail -40 > $out/pytest_gpu.txt
python -c 'import __graft_entry__ as g; g.smoke()' > $out/smoke.txt 2>&1
python bench.py --gpus 1 --steps 50 --warmup 10 > $out/bench.json 2> $out/bench.err
