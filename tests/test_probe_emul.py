"""k_reduce_probe, the reduce kernel AUTO runs when every row may stop early, checked byte for byte on the CPU.

The kernel is compiled from the source text of gpu-pruner_b200/csrc/gpr_probe.cuh and gpr_kernels.cuh under the host
shim (tests/cpp/probe_emul.cpp), with every load and bulk copy renamed to a counting version that charges its bytes to
the row it reads.  The shim's bulk copies land in a seeded random order, so the warps really serve their stages out
of order.  For each window the test requires the decision, candidate and veto bits and the counts to equal the numpy
oracle, and the bytes of every row to equal a numpy model of the rule: the head [0, 32), then 512-sample chunks, each
requested after the previous one was examined, up to the copy that holds the row's first settling sample (util > 0,
power >= thr), or to the end."""
import os
import subprocess

import numpy as np
import pytest

import test_early_exit_emul as EE
from test_hotpath_emul import ROOT, _drop_function, _thr_bits

HEAD = 32               # gpr_launch.h kProbeHeadElems
CHUNK = 512             # gpr_launch.h kProbeChunkElems
BUDGET = 208 * 1024     # gpr_launch.h kProbeSmemBudget
CTAS_PER_SM = 1         # gpr_launch.h kProbeCtasPerSm
WARPS = 32              # gpr_launch.h kProbeWarps
THR = EE.THR
PROBE = os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_probe.cuh")
PROBE_REWRITES = [
    ("extern __shared__ __align__(128) unsigned char smem[];", "unsigned char* smem = tl_cta->smem;", 1),
    ('asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");', ";", 1),
    ("tma_load_1d(", "cnt_tma_load_1d(", 1),
]


def _source():
    src = open(PROBE).read()
    body = src[src.index("namespace gpr {") + len("namespace gpr {"):src.rindex("}  // namespace gpr")]
    body = _drop_function(body, "mbar_test_wait")   # the shim's version lands copies out of order
    for old, new, n in PROBE_REWRITES:
        assert body.count(old) == n, (old, body.count(old))
        body = body.replace(old, new)
    assert "asm" not in body and "__shared__" not in body
    return EE._source() + "\n" + body


def _build(d, sanitize=None):
    (d / "probe_extract.inc").write_text(_source())
    exe = d / ("probe_emul_tsan" if sanitize else "probe_emul")
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function"]
    if sanitize:
        cmd += ["-g", "-fsanitize=" + sanitize]
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "probe_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("probe"))


def layout(T):
    """(head, chunk) of gpr_launch.h probe_layout"""
    ce = min(CHUNK, max((T + 3) // 4 * 4, 4))
    return min(HEAD, ce), ce


def model(first, T):
    h, ce = layout(T)
    return EE.model_tma(first, T, h, ce, False)


def _write(d, util, power, knobs, seed=1, ld=None, shift=0):
    """knobs: (sm_count, GPR_TMA_WARPS), the latter only to show that it does not change the probe plan"""
    P, G, T = util.shape
    ld = ld or T
    os.makedirs(d, exist_ok=True)

    def strided(x, fill):
        out = np.full((P * G, ld), fill, np.float32)
        out[:, :T] = x.reshape(P * G, T)
        return out
    strided(util, 77.0).tofile(os.path.join(d, "util.f32"))      # the padding between rows must never be read
    if power is not None:
        strided(power, 1e9).tofile(os.path.join(d, "power.f32"))
    with open(os.path.join(d, "params.txt"), "w") as f:
        f.write(f"{P} {G} {T} {ld} {int(power is not None)} {_thr_bits(THR)} {shift} {knobs[0]} {knobs[1]} {seed}\n")


def _run(emul, dirs, env=None):
    r = subprocess.run([emul] + [str(d) for d in dirs], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-2000:]
    out = {}
    words = lambda h: np.array([int(h[i:i + 8], 16) for i in range(0, len(h), 8)], np.uint32) if h != "-" else np.zeros(0, np.uint32)
    for l in r.stdout.splitlines():
        f = l.split()
        kv = dict(x.split("=") for x in f[9:])
        out[f[0]] = {"kernel": f[1], "d": words(f[2]), "c": words(f[3]), "v": words(f[4]),
                     "counts": tuple(int(x) for x in f[5:8]), **{k: int(v) for k, v in kv.items()}}
        n = np.fromfile(os.path.join(f[0], "bytes.u64"), np.uint64).astype(np.int64)
        out[f[0]]["bytes"] = n.reshape(2, -1)
    assert len(out) == len(dirs), r.stdout[-2000:]
    return out


def _check(res, util, power, oracle_np, tag):
    P, G, T = util.shape
    want = oracle_np.decide(util, power, None, None, 0, THR if power is not None else 0.0)
    assert res["kernel"] == "probe", tag
    assert (res["head"], res["chunk"]) == layout(T), tag
    assert np.array_equal(res["d"], want["decision_bits"]), tag
    assert np.array_equal(res["c"], want["candidate_bits"]), tag
    assert np.array_equal(res["v"], want["veto_bits"]), tag
    assert res["counts"] == (want["n_series"], want["n_candidates"], want["n_decisions"]), tag
    planes = [(util, False)] + ([(power, True)] if power is not None else [])
    for k, (x, is_power) in enumerate(planes):
        first = EE._first(x.reshape(P * G, T), is_power)
        m = model(first, T)
        got = res["bytes"][k]
        bad = np.nonzero(got != m)[0]
        assert bad.size == 0, (tag, "power" if is_power else "util", bad[:5], got[bad[:5]], m[bad[:5]], first[bad[:5]])


def _positions(T):
    """a settling sample at every head and chunk boundary, one before and one after, and at T - 1"""
    h, ce = layout(T)
    pos = {0, 1, h - 1, h, h + 1, T - 2, T - 1}
    e = h
    while e < T:
        pos |= {e - 1, e, e + 1, min(e + ce, T) - 1}
        e += ce
    return sorted(p for p in pos if 0 <= p < T)


def _boundary_window(T, power):
    quiet = 100.0 if power else 0.0
    rows = []
    for p in _positions(T):
        r = np.full(T, quiet, np.float32)
        r[p] = THR if power else 1.0
        rows.append(r)
    rows.append(np.full(T, quiet, np.float32))          # nothing settles it: read to the end
    while len(rows) % 4:
        rows.append(np.full(T, quiet, np.float32))
    return np.stack(rows).reshape(-1, 4, T)


def _random_window(rng, P, G, T):
    util = np.where(rng.random((P, G, 1)) < 0.4, 0.0,
                    rng.integers(0, 3, (P, G, T)) * (rng.random((P, G, T)) < 0.02)).astype(np.float32)
    util[rng.random((P, G, T)) < 0.05] = np.nan
    power = np.where(rng.random((P, G, T)) < 0.999, 140.0, 150.0).astype(np.float32)
    return util, power


# (sm_count, GPR_TMA_WARPS): one, two and three CTAs; the probe kernel always has kProbeWarps warps
KNOBS = [(2, 16), (1, 4), (3, 32)]


@pytest.mark.parametrize("T", [1800, 3600])
def test_settling_sample_at_every_boundary(emul, tmp_path, oracle_np, T):
    cases = []
    for power_plane in (False, True):
        util = _boundary_window(T, False)
        power = _boundary_window(T, True) if power_plane else None
        for i, knobs in enumerate(KNOBS):
            d = tmp_path / f"b{int(power_plane)}_{i}"
            _write(str(d), util, power, knobs, seed=i + 1)
            cases.append((d, util, power))
    res = _run(emul, [c[0] for c in cases])
    held = 0
    for d, util, power in cases:
        _check(res[str(d)], util, power, oracle_np, d.name)
        held += res[str(d)]["held"]
    assert held > 0      # copies really were held back while others landed


def test_edge_values(emul, tmp_path, oracle_np):
    """the f32 edge rows of test_early_exit_emul.py, placed around this kernel's head"""
    cases = []
    for T in (100, 1800):
        util, power = EE._edge_window(T, HEAD), EE._edge_power(T, HEAD)
        for i, knobs in enumerate(KNOBS[:2]):
            d = tmp_path / f"edge{T}_{i}"
            _write(str(d), util, power, knobs, seed=7 + i)
            cases.append((d, util, power))
    res = _run(emul, [c[0] for c in cases])
    for d, util, power in cases:
        _check(res[str(d)], util, power, oracle_np, d.name)


def test_shapes_strides_and_row_counts(emul, tmp_path, oracle_np):
    """every window length, strided rows (ld % 4 == 0), P % 32 != 0 with G >= 33, and more rows than the grid has
    stages as well as fewer"""
    rng = np.random.default_rng(11)
    cases = []
    shapes = [(9, 4, T, T) for T in (4, 32, 36, 100, 544, 1800, 3600)]
    shapes += [(9, 4, 1800, 1804), (9, 4, 544, 552), (37, 33, 100, 100), (1, 3, 1800, 1800)]
    for P, G, T, ld in shapes:
        util, power = _random_window(rng, P, G, T)
        for i, knobs in enumerate(KNOBS):
            d = tmp_path / f"s{P}_{G}_{T}_{ld}_{i}"
            _write(str(d), util, power if i != 1 else None, knobs, seed=100 + T + i, ld=ld)
            cases.append((d, util, power if i != 1 else None, knobs))
    res = _run(emul, [c[0] for c in cases])
    regimes = set()
    for d, util, power, knobs in cases:
        r = res[str(d)]
        _check(r, util, power, oracle_np, d.name)
        rows = util.shape[0] * util.shape[1] * (2 if power is not None else 1)
        regimes.add(rows > r["grid"] * knobs[1] * r["depth"])
    assert regimes == {True, False}


def test_synthetic_window_byte_share(emul, tmp_path, oracle_np):
    """a C2-shaped window (T 1800, 4 GPUs per pod, bench.py's generator and seed): the util plane costs about 0.41 of
    its bytes (0.48 with k_reduce_tma's 128-sample head and single rest copy)"""
    P, G, T = 400, 4, 1800
    util = oracle_np.synth_fill(0x5EED0002, 0, 0, P, G, T)
    power = oracle_np.synth_fill(0x5EED0002, 1, 0, P, G, T)
    d = tmp_path / "synth"
    _write(str(d), util, power, (2, 16), seed=3)
    r = _run(emul, [d])[str(d)]
    _check(r, util, power, oracle_np, "synth")
    share = r["bytes"][0].sum() / (4.0 * util.size)
    old = EE.model_tma(EE._first(util.reshape(P * G, T), False), T, 128, 1800, False).sum() / (4.0 * util.size)
    assert 0.36 < share < 0.46 and share < old - 0.04, (share, old)


def test_probe_under_thread_sanitizer(tmp_path, oracle_np):
    """copies that land out of order, stages that change rows, the shared row counter, under ThreadSanitizer"""
    exe = _build(tmp_path, sanitize="thread")
    T = 1100
    util = _boundary_window(T, False)
    power = np.full(util.shape, 100.0, np.float32)
    power[1, :, 600] = THR
    d = tmp_path / "tsan"
    _write(str(d), util, power, (1, 4), seed=5)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r = _run(exe, [d], env=env)[str(d)]
    _check(r, util, power, oracle_np, "tsan")
