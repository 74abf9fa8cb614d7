#!/bin/bash
# Run from the repository root after __graft_entry__.build(), on one H100.  $PARENT holds the parent commit's tree
# (git archive HEAD~ | tar -x -C $PARENT), built the same way.  $MUTANTS/libgpr_mN.so is this tree's library built
# with one single-line mutation each (m1-m3 in csrc/gpr_chunks.cuh, m4-m6 in csrc/gpr_chunks_encode.cuh):
#   m1  dod > (1ull << (sz - 1u))      ->  dod >= (1ull << (sz - 1u))
#   m2  trail = (64u - lead - sig) & 0xffu;  ->  trail = (64u - lead - sig);
#   m3  sig = m ? m : 64u;             ->  sig = m;
#   m4  if (lead > 31u) lead = 31u;    ->  if (lead > 32u) lead = 31u;
#   m5  dod <= (1ll << (n - 1u))       ->  dod < (1ll << (n - 1u))        (in_bucket)
#   m6  put(e.w, sig & 63u, 6u);       ->  put(e.w, sig, 6u);
# Each changes a bit or a decision only, never a size, an offset or an address.  gpu.txt is read in the same run.
# The outputs here come from two runs on H100s of the same kind, with the same library: gpu_run1.txt, smoke.txt,
# pytest_gpu_existing.txt, bench_*.json and dump_compare.txt from the first; gpu.txt, pytest_gpu.txt and mutant_*.txt
# from the second, after a fix to the ring test's setup (its gaps hold the fill, not another NaN).
set -u
OUT=${OUT:-out}; mkdir -p $OUT
PARENT=${PARENT:-_parent}; MUTANTS=${MUTANTS:-_mutants}
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/gpu.txt
python -m pytest -m gpu tests/test_gpu_chunk_codec.py -v -p no:cacheprovider --durations=0 > $OUT/pytest_gpu.txt 2>&1
python -m pytest -m gpu tests/test_gpu_chunks.py tests/test_gpu_resident_export.py tests/test_gpu_daemon_snapshot.py \
  tests/test_gpu_session_ring.py -q -p no:cacheprovider > $OUT/pytest_gpu_existing.txt 2>&1
python -c "import __graft_entry__ as g; g.smoke()" > $OUT/smoke.txt 2>&1
cp gpu-pruner_b200/libgpr.so /tmp/libgpr_this.so
for m in m1 m2 m3 m4 m5 m6; do
  cp $MUTANTS/libgpr_$m.so gpu-pruner_b200/libgpr.so
  python -m pytest -m gpu tests/test_gpu_chunk_codec.py -q -p no:cacheprovider -rf > $OUT/mutant_$m.txt 2>&1
done
cp /tmp/libgpr_this.so gpu-pruner_b200/libgpr.so
# bench.py, parent and this change, alternated; the outputs of the last timed step compared
for i in 1 2; do
  for b in par new; do
    d=.; [ $b = par ] && d=$PARENT
    (cd $d && python bench.py --gpus 1 --steps 2000 --warmup 20 --dump-outputs /tmp/dump_${b}_$i) \
      > $OUT/bench_${b}_$i.json 2> /dev/null
  done
done
python - <<'PY' | tee $OUT/dump_compare.txt
import numpy as np, os
for f in sorted(f for f in os.listdir("/tmp/dump_par_1") if f.endswith(".npy")):
    a = [np.load(f"/tmp/dump_{b}_{i}/{f}") for b in ("par", "new") for i in (1, 2)]
    print(f, "identical" if all(np.array_equal(a[0], x) for x in a) else "DIFFER")
PY
rm -rf /tmp/dump_par_* /tmp/dump_new_* /tmp/libgpr_this.so
