"""Which reduce kernel gpr_launch.h's plan_reduce picks once it knows whether rows may stop, and the probe kernel's
ring layout (k_reduce_probe, gpu-pruner_b200/csrc/gpr_probe.cuh).

AUTO runs the probe kernel exactly when every row may stop (no series_max target, no group table), the rows can be
bulk-copied and the util plane is f32; every other call gets the plan it got before may_stop existed."""
import itertools

import pytest

import geometry
from test_probe_emul import BUDGET, CTAS_PER_SM, CHUNK, HEAD, WARPS, layout

SM_SMEM = 228 * 1024        # H100: shared memory per SM
CTA_RESERVED = 1024         # shared memory the hardware reserves per resident CTA
FOLD_THREADS, FOLD_SMEM = 256, 128   # k_fold at the default fold_threads, and its static shared memory


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    return geometry.build(tmp_path_factory.mktemp("launch_plan"))


def _knobs(sm_count=132, warps=16):
    return geometry.Knobs(sm_count=sm_count, tma_warps=warps, tma_chunk=8192, tma_depth=3)


def _plans(exe, queries):
    """queries: (knobs, variant, T, rows, tma_ok, util_u8, may_stop)"""
    return geometry.plans(exe, [(k, v, T, rows, ok, u8, 1, ms) for k, v, T, rows, ok, u8, ms in queries])


def test_selection_matrix(plan_exe):
    qs = []
    for variant, may_stop, tma_ok, u8, warps in itertools.product(("auto", "ldg", "tma"), (0, 1), (0, 1), (0, 1),
                                                                   (4, 16)):
        qs.append((_knobs(warps=warps), variant, 1800, 80000, tma_ok, u8, may_stop))
        qs.append((_knobs(warps=warps), variant, 1800, 80000, tma_ok, u8, 0))   # the same call as before may_stop
    got = _plans(plan_exe, qs)
    n_probe = 0
    for i in range(0, len(qs), 2):
        _, variant, T, rows, tma_ok, u8, may_stop = qs[i]
        p, before = got[i], got[i + 1]
        if variant == "auto" and may_stop and tma_ok and not u8:
            n_probe += 1
            assert p.kernel == "probe" and p.fallback is None, qs[i]
            assert p.block == 32 * WARPS and p.grid == min(132 * CTAS_PER_SM, -(-rows // WARPS)), p
            assert (p.head_elems, p.chunk_elems) == layout(T) and p.smem <= BUDGET, p
        else:
            assert p == before, qs[i]
            assert p.kernel != "probe"
    assert n_probe == 2


@pytest.mark.parametrize("knob_warps", [4, 8, 16, 32])
def test_layout_fits_for_every_window_length(plan_exe, knob_warps):
    """GPR_TMA_WARPS does not change the probe plan: the kernel always has kProbeWarps warps"""
    warps = WARPS
    Ts = list(range(4, 7201, 4))
    got = _plans(plan_exe, [(_knobs(warps=knob_warps), "auto", T, 40000, 1, 0, 1) for T in Ts])
    for T, p in zip(Ts, got):
        h, ce = layout(T)
        assert p.kernel == "probe" and (p.head_elems, p.chunk_elems) == (h, ce) and p.block == 32 * warps, (T, p)
        assert 1 <= p.depth <= 32 and p.stage_bytes % 128 == 0 and p.stage_bytes >= 4 * ce, (T, p)
        # stages, one barrier per stage, the row counter
        assert p.smem == warps * p.depth * (p.stage_bytes + 8) + 8 <= BUDGET, (T, p)
        assert p.n_chunks == 1 + max(0, -(-(T - h) // ce)), (T, p)
    # the full-size stage leaves the ring as deep as the budget allows
    full = [p for T, p in zip(Ts, got) if T >= CHUNK]
    assert all(p.depth == min(32, (BUDGET - 8) // (warps * (4 * CHUNK + 8))) for p in full)
    assert HEAD % 4 == 0 and CHUNK % 4 == 0


def test_probe_cta_and_the_fold_share_an_sm(plan_exe):
    """the probe CTA leaves shared memory and threads for a 256-thread fold CTA beside it"""
    assert CTAS_PER_SM == 1
    for T in (4, 100, 544, 1800, 3600, 7200):
        p = _plans(plan_exe, [(_knobs(), "auto", T, 40000, 1, 0, 1)])[0]
        assert CTAS_PER_SM * (p.smem + CTA_RESERVED) + FOLD_SMEM + CTA_RESERVED <= SM_SMEM, (T, p)
        assert CTAS_PER_SM * p.block + FOLD_THREADS <= 2048


def test_row_split_at_the_series_limit(plan_exe):
    """2^32 - 2 rows (a power plane at the series limit): the grid and the strided split cover every row once"""
    for sm in (132, 1, 7):
        rows = 2 ** 32 - 2
        p = _plans(plan_exe, [(_knobs(sm_count=sm), "auto", 4, rows, 1, 0, 1)])[0]
        assert p.kernel == "probe" and p.grid == sm * CTAS_PER_SM
        per_cta = [(rows - b + p.grid - 1) // p.grid if rows > b else 0 for b in range(p.grid)]   # cta_row_count
        assert sum(per_cta) == rows and max(per_cta) < 2 ** 32 and max(per_cta) - min(per_cta) <= 1
    tiny = _plans(plan_exe, [(_knobs(), "auto", 1800, 3, 1, 0, 1)])[0]
    assert tiny.grid == 1
