"""C2 decisions as bench.py makes them (its four windows, gpr_decide_batch_async), timed over short runs of K = 5, 20
and 200 decisions (best and median of 7) and one isolated blocking decision (median of 21).  Run from a built tree."""
import sys, os
sys.path.insert(0, os.getcwd())
import numpy as np, torch
import gpu_pruner_b200 as g
P, G, T, SEED, ROT = 10000, 4, 1800, 0x5EED0002, 4
eng = g.IdleEngine(device=0)
wins = []
for i in range(ROT):
    u = torch.full((P, G, T), float("nan"), dtype=torch.float32, device="cuda:0")
    e = torch.zeros(P, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    eng.synth_fill(SEED + 16 * i, 0, u, 0, P, G, T)
    eng.synth_eligible(SEED + 16 * i, e, 0, P)
    wins.append((u, e))
db = torch.zeros((P + 31) // 32, dtype=torch.int32, device="cuda:0")
torch.cuda.synchronize()
step = lambda i, b=False: eng.decide_ptr(wins[i % ROT][0], P, G, T, db, eligible=wins[i % ROT][1], blocking=b)
batch = eng.make_batch([dict(util=wins[i % ROT][0], eligible=wins[i % ROT][1], P=P, G=G, T=T, decision_bits=db)
                        for i in range(200)])
for i in range(20): step(i)
eng.sync()
out = []
for K in (5, 20, 200):
    best = []
    for rep in range(7):
        eng.timer_begin(); eng.decide_batch_async(batch, K); ms = eng.timer_end(); eng.sync()
        best.append(ms / K * 1e3)
    out.append(f"K={K}: min {min(best):.2f} med {sorted(best)[3]:.2f}")
iso = sorted(step(i, True).kernel_ms for i in range(21))
out.append(f"iso med {iso[10]*1e3:.2f} min {iso[0]*1e3:.2f}")
print(sys.argv[1] if len(sys.argv) > 1 else "", " | ".join(out), flush=True)
