"""`sum by` groups decided on the device (gpr_window.groups), checked on the CPU.

First the plain restatement of the rule (tests/groups_ref.py) is held to the host's exact `sum by`,
gph::resolve_sum_by_groups and gph::group_value, on windows ingested from the wire format.  Then the source of
k_group_rows / k_group_sum (gpu-pruner_b200/csrc/gpr_groups.cuh) runs under the host shim around k_reduce_ldg,
k_reduce_tma, k_reduce_u8 and k_fold (tests/cpp/groups_emul.cpp), and every output — decision, candidate and veto
bits, counts, idle_slots, series_max — must equal the restatement, bit for bit, and every row must cost the bytes the
rule says: 4 * T for a row of a group of two or more, the early-exit model of test_early_exit_emul.py for every
other row."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import groups_ref as R
import hostlib as H
import test_early_exit_emul as EE
from test_hotpath_emul import ROOT, _extract, _thr_bits

THR = EE.THR
SENTINEL = 0x7FF8DEADBEEF0000   # groups_emul.cpp: a NaN that no sum produces, in every slot it did not sum
RENAMES = EE.RENAMES + [("ldg_stream_u4(", "cnt_ldg_stream_u4(")]
KNOBS = {"tma": EE.LAYOUTS["four chunks"], "ldg": EE.LAYOUTS["one rest chunk"], "u8": EE.LAYOUTS["one rest chunk"]}


def _kernels_source():
    body = _extract()
    for old, new in RENAMES:
        assert old in body, old
        body = body.replace(old, new)
    return body


def _groups_source():
    src = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_groups.cuh")).read()
    body = src[src.index("namespace gpr {") + len("namespace gpr {"):src.rindex("}  // namespace gpr")]
    assert "asm" not in body and "__shared__" not in body and "k_group_rows" in body and "k_group_sum" in body
    # the emulator also records every summed group's float64 value (the kernel only publishes `== 0`), so the sum
    # itself — order of the members, compensation, `/ 100` — is compared with the host's, bit for bit
    old = "idle = s.any && s.value() == 0.0;"
    assert body.count(old) == 1
    return body.replace(old, old + " record_group_value(p, g, s.any, s.value());")


def build(d, sanitize=None, kernels=None, groups=None):
    (d / "groups_kernels_extract.inc").write_text(kernels or _kernels_source())
    (d / "groups_extract.inc").write_text(groups or _groups_source())
    exe = d / ("groups_emul_tsan" if sanitize else "groups_emul")
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function"]
    if sanitize:
        cmd += ["-g", "-fsanitize=" + sanitize]
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "groups_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return build(tmp_path_factory.mktemp("groups"))


def write_case(d, util, power, table, variant, smax=False, shift=0, ld=None):
    P, G, T = util.shape
    ld = ld or T
    os.makedirs(d, exist_ok=True)
    if variant == "u8":
        import gpu_pruner_b200 as g
        rows = np.zeros((P * G, ld), np.uint8)
        rows[:, :T] = g.to_biased_u8(util).reshape(P * G, T)
        rows.tofile(os.path.join(d, "util.u8"))
    else:
        rows = np.full((P * G, ld), 77.0, np.float32)
        rows[:, :T] = util.reshape(P * G, T)
        rows.tofile(os.path.join(d, "util.f32"))
    if power is not None:
        prow = np.full((P * G, ld), 1e9, np.float32)
        prow[:, :T] = power.reshape(P * G, T)
        prow.tofile(os.path.join(d, "power.f32"))
    if table is not None:
        np.ascontiguousarray(table, np.uint32).tofile(os.path.join(d, "groups.u32"))
    with open(os.path.join(d, "params.txt"), "w") as f:
        f.write(f"{P} {G} {T} {ld} {int(power is not None)} {_thr_bits(THR)} {int(smax)} {shift} "
                f"{' '.join(str(k) for k in KNOBS[variant])} {variant} {int(table is not None)}\n")


def run(exe, dirs, env=None):
    r = subprocess.run([exe] + [str(d) for d in dirs], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-2000:]
    words = lambda h: np.array([int(h[i:i + 8], 16) for i in range(0, len(h), 8)], np.uint32) if h != "-" else None
    out = {}
    for line in r.stdout.splitlines():
        f = line.split()
        out[f[0]] = {"kernel": f[1], "d": words(f[2]), "c": words(f[3]), "v": words(f[4]),
                     "counts": tuple(int(x) for x in f[5:8]), "islots": words(f[8]), "bad": int(f[9]),
                     "smax": None if f[10] == "-" else words(f[10]).view(np.float32)}
        out[f[0]]["bytes"] = np.fromfile(os.path.join(f[0], "bytes.u64"), np.uint64).astype(np.int64).reshape(2, -1)
        out[f[0]]["values"] = np.fromfile(os.path.join(f[0], "values.f64"), np.float64)
    return out


def grouped_rows(table):
    """rows of groups of two or more"""
    P, G = table.shape
    lead = (table & 0xFF).astype(np.int64)
    out = np.zeros((P, G), bool)
    for p in range(P):
        sizes = np.bincount(lead[p], minlength=G)
        out[p] = sizes[lead[p]] > 1
    return out


def check(res, util, power, table, variant, smax=False, shift=0, ld=None, tag=None):
    P, G, T = util.shape
    ld = ld or T
    want = R.decide(util, power, THR if power is not None else 0.0, table)
    tag = tag or (variant, P, G, T, smax)
    assert res["bad"] == 0, tag
    assert np.array_equal(res["d"], want["decision_bits"]), tag
    assert np.array_equal(res["c"], want["candidate_bits"]), tag
    assert np.array_equal(res["v"], want["veto_bits"]), tag
    assert res["counts"] == (want["n_series"], want["n_candidates"], want["n_candidates"]), (tag, res["counts"])
    assert np.array_equal(res["islots"], want["idle_slots"].ravel()), tag
    # the value of every summed group, bit for bit (NaN: no member with a sample); nothing else is summed
    vals = res["values"].reshape(P, G)
    summed = {(int(p), int(g)) for p, g in np.argwhere(vals.view(np.uint64) != SENTINEL)}
    assert summed == set(want["values"]), (tag, sorted(summed ^ set(want["values"]))[:5])
    for (p, g), v in want["values"].items():
        got_v = vals[p, g]
        assert (np.isnan(v) and np.isnan(got_v)) or np.float64(v).view(np.uint64) == got_v.view(np.uint64), \
            (tag, p, g, v, got_v)
    m = R.row_max(util)
    if smax:
        got = res["smax"].reshape(P, G)
        assert np.array_equal(np.isnan(got), np.isnan(m)) and np.array_equal(np.nan_to_num(got), np.nan_to_num(m)), tag
    # bytes: a grouped row is read whole, every other row as the early-exit model says
    full = np.zeros((P, G), bool) if table is None else grouped_rows(table)
    got = res["bytes"][0].reshape(P, G)
    if variant == "u8":
        assert np.all(got == T), tag
    else:
        first = EE._first(util.reshape(P * G, T), False).reshape(P, G)
        if res["kernel"] == "tma":
            h, ce = EE._tma_layout(KNOBS["tma"], T)
            model = EE.model_tma(first.ravel(), T, h, ce, smax).reshape(P, G)
        else:
            offsets = (shift + np.arange(P * G, dtype=np.int64) * ld) % 4
            model = EE.model_ldg(first.ravel(), T, offsets, smax).reshape(P, G)
        model = np.where(full, 4 * T, model)
        bad = np.argwhere(got != model)
        assert bad.size == 0, (tag, bad[:5], got[tuple(bad[:5].T)], model[tuple(bad[:5].T)])
    if power is not None and variant != "u8":
        pfirst = EE._first(power.reshape(P * G, T), True)
        if res["kernel"] == "tma":
            h, ce = EE._tma_layout(KNOBS["tma"], T)
            pm = EE.model_tma(pfirst, T, h, ce, smax)
        else:
            offsets = (shift + np.arange(P * G, dtype=np.int64) * ld) % 4
            pm = EE.model_ldg(pfirst, T, offsets, smax)
        assert np.array_equal(res["bytes"][1], pm), tag


# ---- the restatement against the host's exact `sum by` -------------------------------------------------------------
def _lab(pod, gpu, **kw):
    d = {"Hostname": "node1", "modelName": "NVIDIA A100", "UUID": "GPU-x", "gpu": str(gpu), "exported_pod": pod,
         "exported_namespace": "ml", "exported_container": "main"}
    d.update(kw)
    return d


def _series(labels, v, t_end):
    return {"metric": labels, "values": [[t_end, v]]}


def _resp(ss):
    return {"status": "success", "data": {"resultType": "matrix", "result": ss}}


# each pod: a list of groups; a group: members (kind, value text) in order of appearance
HOST_PODS = {
    "mixed": [[("util", "5"), ("util", "-5")]],                               # +5 / -5: idle
    "halfbusy": [[("util", "0"), ("util", "7")]],                             # 0 / 7: not idle
    "profutil": [[("util", "0"), ("prof", "0")], [("util", "3")]],            # PROF + UTIL mix, idle
    "cancel": [[("prof", "1"), ("prof", "1e16"), ("prof", "-1e16"), ("prof", "-1")]],  # idle only when compensated
    "cancel2": [[("prof", "1e16"), ("prof", "1"), ("prof", "-1e16")]],       # 1, not 0
    "nanmember": [[("util", "NaN"), ("util", "0")]],                          # NaN member skipped: idle
    "allnan": [[("util", "NaN"), ("prof", "NaN")]],                           # no element
    "infs": [[("util", "+Inf"), ("util", "-Inf")]],                           # NaN: not idle
    "inf": [[("util", "+Inf"), ("util", "5")]],
    "negzero": [[("util", "-0"), ("prof", "-0")]],
    "denorm": [[("util", "1e-45"), ("util", "-1e-45")], [("util", "1e-45")]],  # /100 in float64: cancels, lone stays
    "denorm2": [[("prof", "1e-45"), ("util", "0")]],
    "lone": [[("util", "0")], [("util", "1")]],
    "triple": [[("util", "2"), ("prof", "-0.01"), ("util", "-1")], [("util", "0"), ("util", "0")]],
    # the compensation term takes the absorbed addends 1, 2^-53, 2^-53 in slot order: (1 + 2^-53) + 2^-53 rounds to
    # 1, the other way round it is 1 + 2^-52 — a sum in any other order than the slots' has a different value
    "order": [[("prof", "1329227995784915872903807060280344576"), ("prof", "1"),
               ("prof", "1.1102230246251565404236316680908203125e-16"),
               ("prof", "1.1102230246251565404236316680908203125e-16"),
               ("prof", "-1329227995784915872903807060280344576")]],
}


def _host_window():
    t_end = 4000
    util, prof = [], []
    for pod, groups in HOST_PODS.items():
        for gpu, members in enumerate(groups):
            for i, (kind, v) in enumerate(members):
                extra = {"UUID": f"GPU-{i}"} if kind == "util" else {"profiled": f"p{i}"}
                (util if kind == "util" else prof).append(_series(_lab(pod, gpu, **extra), v, t_end))
    u, _, meta = H.ingest(_resp(util), _resp(prof), duration_min=1, step=1, t_end=t_end)
    P, G, _ = u.shape
    table = np.zeros((P, G), np.uint32)
    assert H.lib().gph_group_table(C.c_uint(P), table.ctypes.data_as(C.c_void_p)) == 0
    return u, table, [p["name"] for p in meta["pods"]]


def test_restatement_equals_the_hosts_exact_sum_by(oracle_np):
    u, table, names = _host_window()
    assert R.valid(table) and grouped_rows(table).any()
    raw = oracle_np.decide(u)
    want = R.decide(u, table=table)
    counts = (raw["n_series"], raw["n_candidates"], raw["n_decisions"])
    cb, db, counts2, _ = H.resolve_groups(raw["series_max"], raw["candidate_bits"], raw["decision_bits"], counts)
    assert np.array_equal(cb[:len(want["candidate_bits"])], want["candidate_bits"])
    assert counts2 == (want["n_series"], want["n_candidates"], want["n_candidates"])
    vals = H.group_values(raw["series_max"])
    for (p, g), v in want["values"].items():
        assert (math.isnan(v) and math.isnan(vals[p, g])) or (v == vals[p, g] and math.copysign(1, v) ==
                                                                math.copysign(1, vals[p, g])), (names[p], g, v)
    order = names.index("order")
    assert want["values"][(order, 0)] == 1.0 and R.neumaier([2.0 ** 120, 1.0, 2.0 ** -53, 2.0 ** -53, -2.0 ** 120][::-1]) \
        == 1.0 + 2.0 ** -52
    cand = {names[i] for i in np.flatnonzero(want["candidate"])}
    assert cand == {"mixed", "profutil", "cancel", "nanmember", "negzero", "denorm", "lone", "triple"}, cand
    # head-room pods of a resident ring lead themselves
    extra = np.zeros((len(names) + 3, table.shape[1]), np.uint32)
    H.lib().gph_group_table(C.c_uint(len(names) + 3), extra.ctypes.data_as(C.c_void_p))
    assert np.array_equal(extra[:len(names)], table) and np.array_equal(extra[len(names):] & 0xFF,
                                                                         np.tile(np.arange(table.shape[1]), (3, 1)))


def test_kernels_on_the_ingested_window(emul, tmp_path):
    u, table, _ = _host_window()
    cases = []
    for variant in ("ldg", "tma"):
        for smax in (False, True):
            d = tmp_path / f"{variant}_{int(smax)}"
            write_case(str(d), u, None, table, variant, smax)
            cases.append((d, variant, smax))
    res = run(emul, [c[0] for c in cases])
    for d, variant, smax in cases:
        check(res[str(d)], u, None, table, variant, smax)


# ---- the kernels on generated windows ------------------------------------------------------------------------------
def _generated(seed, P, G, T, u8=False, share=0.5, max_size=None, power=True):
    rng = np.random.default_rng(seed)
    table = R.random_table(rng, P, G, share, max_size)
    pal = R.PALETTE_U8 if u8 else R.PALETTE
    m = np.array(pal, np.float32)[rng.integers(0, len(pal), (P, G))]
    util = R.window_for(rng, m, T, u8)
    pw = None
    if power:
        pw = np.full((P, G, T), 100.0, np.float32)
        pw[rng.random(P) < 0.2, 0, T // 3] = THR
    return util, pw, table


SHAPES = [  # (P, G, T, max group size): P % 32 != 0, groups across the 31/32 word boundary, G = 256
    (37, 4, 256, None), (9, 40, 200, None), (3, 256, 64, None), (70, 3, 1800, 3), (33, 2, 132, 2)]


@pytest.mark.parametrize("variant", ["ldg", "tma", "u8"])
def test_generated_windows(emul, tmp_path, variant):
    cases = []
    for i, (P, G, T, size) in enumerate(SHAPES):
        util, power, table = _generated(i, P, G, T, variant == "u8", max_size=size)
        for smax in (False, True):
            for shift in ((0, 1) if variant == "ldg" else (0,)):
                d = tmp_path / f"s{i}_{int(smax)}_{shift}"
                write_case(str(d), util, power, table, variant, smax, shift)
                cases.append((d, util, power, table, smax, shift))
    res = run(emul, [c[0] for c in cases])
    sizes = set()
    for d, util, power, table, smax, shift in cases:
        check(res[str(d)], util, power, table, variant, smax, shift)
        lead = (table & 0xFF).astype(np.int64)
        for p in range(table.shape[0]):
            sizes |= set(np.bincount(lead[p]).tolist())
    assert {2, 3} <= sizes


def test_every_group_size_and_the_word_boundary(emul, tmp_path):
    """one group per pod: sizes 2..G (G = 40: a group of every size, members on both sides of slot 31/32)"""
    G, T = 40, 64
    rows = []
    for size in range(2, G + 1):
        t = np.arange(G, dtype=np.uint32)
        t[G - size + 1:] = 0 if size % 2 else G - size    # leader 0, or the slot just before the members
        rows.append(t | np.where(np.arange(G) % 3 == 0, R.UTIL, 0).astype(np.uint32))
    table = np.stack(rows)
    assert R.valid(table)
    P = table.shape[0]
    m = np.zeros((P, G), np.float32)
    m[::3, -1] = 5.0                                       # a busy member in every third group
    rng = np.random.default_rng(3)
    util = R.window_for(rng, m, T)
    cases = []
    for variant in ("ldg", "tma"):
        d = tmp_path / variant
        write_case(str(d), util, None, table, variant)
        cases.append((d, variant))
    res = run(emul, [c[0] for c in cases])
    for d, variant in cases:
        check(res[str(d)], util, None, table, variant)


def test_without_a_table_idle_slots_are_the_row_flags(emul, tmp_path, oracle_np):
    util, power, _ = _generated(11, 37, 4, 256)
    d = tmp_path / "none"
    write_case(str(d), util, power, None, "tma")
    r = run(emul, [d])[str(d)]
    check(r, util, power, None, "tma")
    raw = oracle_np.decide(util, power, power_threshold=THR)
    assert r["counts"][0] == raw["n_series"] and np.array_equal(r["c"], raw["candidate_bits"])


MALFORMED = {
    "leader above its slot": lambda t: t.__setitem__((1, 0), 2),
    "leader does not lead itself": lambda t: t.__setitem__((2, 3), 1) or t.__setitem__((2, 1), 0),
    "stray bit": lambda t: t.__setitem__((3, 2), 2 | 0x200),
    "leader beyond 8 bits": lambda t: t.__setitem__((0, 1), 0x1000),
}


@pytest.mark.parametrize("kind", sorted(MALFORMED))
def test_malformed_tables_raise_the_error_flag(emul, tmp_path, kind):
    util, _, _ = _generated(5, 5, 4, 64, power=False)
    table = np.tile(np.arange(4, dtype=np.uint32), (5, 1))
    MALFORMED[kind](table)
    if kind == "leader does not lead itself":
        table[2, 1], table[2, 3] = 0, 1                   # slot 3 names slot 1, which leads slot 0's group
    assert not R.valid(table)
    d = tmp_path / "bad"
    write_case(str(d), util, None, table, "ldg")
    r = run(emul, [d])[str(d)]
    bad_pods = [p for p in range(5) if not R.valid(table[p:p + 1])]
    assert r["bad"] - 1 in bad_pods, (r["bad"], bad_pods)


def test_groups_under_thread_sanitizer(tmp_path):
    exe = build(tmp_path, sanitize="thread")
    util, power, table = _generated(21, 33, 40, 128)
    cases = []
    for variant in ("tma", "ldg"):
        d = tmp_path / f"tsan_{variant}"
        write_case(str(d), util, power, table, variant)
        cases.append((d, variant))
    res = run(exe, [c[0] for c in cases], env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    for d, variant in cases:
        check(res[str(d)], util, power, table, variant)
