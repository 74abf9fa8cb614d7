"""The launch geometry of gpu-pruner_b200/csrc/gpr_launch.h, queried through tests/cpp/launch_plan.cpp: which reduce
kernel the library runs for a window on a device with given knobs, its grid and TMA ring layout, and the fold grid.
may_stop: the call passes no series_max target and no group table, so its rows may stop early (AUTO then runs the
probe kernel, k_reduce_probe, when the rows can be bulk-copied and the util plane is f32)."""
import os
import subprocess
from dataclasses import dataclass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = {1: "ldg", 2: "tma", 3: "u8", 4: "probe"}
FALLBACKS = {0: None, 1: "alignment", 2: "smem"}
VARIANT = {"auto": 0, "ldg": 1, "tma": 2}


@dataclass(frozen=True)
class Knobs:
    sm_count: int = 132
    tma_warps: int = 16
    tma_chunk: int = 8192
    tma_depth: int = 3
    ldg_ctas: int = 2
    fold_threads: int = 256

    def env(self):
        """the environment gpr_create reads these knobs from"""
        return {"GPR_TMA_WARPS": str(self.tma_warps), "GPR_TMA_CHUNK": str(self.tma_chunk),
                "GPR_TMA_DEPTH": str(self.tma_depth), "GPR_LDG_CTAS": str(self.ldg_ctas),
                "GPR_FOLD_THREADS": str(self.fold_threads)}


@dataclass(frozen=True)
class Plan:
    kernel: str
    fallback: object
    grid: int
    block: int
    smem: int
    depth: int
    stage_bytes: int
    chunk_elems: int
    n_chunks: int
    fold_grid: int
    fold_rounds: int
    head_elems: int

    def last_chunk(self, T):
        return T - (self.n_chunks - 1) * self.chunk_elems


def build(out_dir):
    exe = os.path.join(str(out_dir), "launch_plan")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cpp", "launch_plan.cpp"),
                    "-o", exe], check=True, capture_output=True, text=True)
    return exe


def plans(exe, queries):
    """queries: (knobs, variant, T, total_rows, tma_ok, util_u8, P[, may_stop]) -> [Plan]; may_stop defaults to
    False, the plan of a call that reads every row whole"""
    lines = []
    for q in queries:
        k, v, T, rows, ok, u8, P = q[:7]
        may_stop = q[7] if len(q) > 7 else False
        lines.append(f"{k.sm_count} {VARIANT[v]} {k.tma_warps} {k.tma_chunk} {k.tma_depth} {k.ldg_ctas} "
                     f"{k.fold_threads} {T} {rows} {int(ok)} {int(u8)} {P} {int(may_stop)}")
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, timeout=60)
    out = []
    for l in r.stdout.splitlines():
        f = [int(x) for x in l.split()]
        out.append(Plan(KERNELS[f[0]], FALLBACKS[f[1]], *f[2:]))
    assert len(out) == len(lines)
    return out


def plan(exe, knobs, variant, T, total_rows, tma_ok=True, util_u8=False, P=1, may_stop=False):
    return plans(exe, [(knobs, variant, T, total_rows, tma_ok, util_u8, P, may_stop)])[0]
