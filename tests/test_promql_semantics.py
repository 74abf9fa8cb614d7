"""CPU: PromQL semantics -> (C++ ingest of the wire format) -> dense tensor -> oracle, end to end.

tests/promql_mini.py evaluates the reference's expression (gpu-pruner/src/
query.promql.j2:1-44) the way Prometheus does, on labelled instant vectors, in float64.  For random clusters —
multi-GPU pods, PROF + UTIL series, `sum by` duplicates, hosts with and without node_dmi_info,
scrape gaps, series that start late, unconvertible series, power draw around the threshold — the set
of pods it returns (after the Rust-side dedup, main.rs:416-437) must equal the candidates the dense
path produces: range-query wire format -> gpu-pruner_b200/host ingest -> oracle decision.

The values come from tests/edges.py where f32 and float64 part ways: power readings within an f32 ulp of the
threshold (thresholds exact in f32 and not), non-zero utilisation that vanishes in f32, 17-digit PROF ratios,
NaN / +-Inf, numbers spelt with more than 19 digits, millisecond timestamps and several samples per bucket.
The same clusters go through the device parser on an emulated device (test_emulated_device_*) and, on an H100,
through the kernels (tests/test_gpu_promql.py).
"""
import json
import math
import os
import random
import subprocess

import numpy as np
import pytest

import edges as E
import hostlib as H
import promql_mini as Q


def make_cluster(rng, honor_labels=False, t_eval=100_000, duration_min=2, thr=None):
    """`thr`: the power threshold the draws are placed around (None: the old 60 / 149 / 150 / 151 / 400 W draws)"""
    T = duration_min * 60
    pl, nl, cl = ("pod", "namespace", "container") if honor_labels else (
        "exported_pod", "exported_namespace", "exported_container")
    db = []
    # a little history before the window too; some timestamps carry millisecond fractions, t_eval - T (excluded)
    # and t_eval (included) are always there
    ts = [t + (rng.choice([0.001, 0.5, 0.999]) if rng.random() < 0.15 and t not in (t_eval - T, t_eval) else 0)
          for t in range(t_eval - T - 30, t_eval + 1)]
    n_ts = len(ts)

    def pattern(kind, zeroish=E.UTIL_ZEROISH):
        if kind == "idle":
            return [0.0] * n_ts
        if kind == "busy":
            return [float(rng.choice([0, 0, 0, 37, 100])) for _ in ts]
        if kind == "burst":                                   # one sample somewhere in the window
            v = [0.0] * n_ts
            v[rng.randrange(31, n_ts)] = 5.0
            return v
        if kind == "old_burst":                               # activity only BEFORE the window
            v = [0.0] * n_ts
            v[rng.randrange(0, 30)] = 80.0
            return v
        if kind == "tiny":                                    # non-zero, but 0 or a denormal in f32; or -0
            v = [0.0] * n_ts
            for _ in range(rng.randrange(1, 3)):
                v[rng.randrange(25, n_ts)] = rng.choice(zeroish)
            return v
        if kind == "special":                                 # +-Inf / NaN among zeros
            v = [0.0] * n_ts
            v[rng.randrange(25, n_ts)] = rng.choice(E.SPECIAL)
            return v
        if kind == "nan_first":                               # max_over_time starts at NaN, then 0 replaces it
            return [math.nan] * 40 + [0.0] * (n_ts - 40)
        if kind == "all_nan":
            return [math.nan] * n_ts
        raise AssertionError(kind)

    def emit(name, labels, vals, gap=0.0, start=0):
        smp = [(t, v) for i, (t, v) in enumerate(zip(ts, vals)) if i >= start and rng.random() >= gap]
        if smp:
            db.append(Q.series(name, labels, smp))

    if thr and not math.isnan(thr):
        below = [v for v in E.power_edges(thr) if v < thr] + [thr / 2, math.nan]
        above = [v for v in E.power_edges(thr) if v >= thr] + [thr * 3, math.inf]
        between = min(55.0, thr / 3)                          # the readings between the draws stay below thr
    else:
        below, above, between = [60.0, 60.0, 149.0, math.nan], [150.0, 151.0, 400.0], 55.0
    hosts = [f"node-{i}" for i in range(4)]
    for h in hosts[:3]:                                       # node-3 has no DMI series
        db.append(Q.series("node_dmi_info", {"instance": h, "product_name": "DGX-B200"}, [(t_eval - 5, 1.0)]))
    n_pods = rng.randrange(6, 14)
    for p in range(n_pods):
        pod, ns = f"pod-{p}", rng.choice(["ml-team", "ml-team", "infra"])
        host = rng.choice(hosts)
        for g in range(rng.randrange(1, 5)):
            base = {"Hostname": host, "gpu": str(g), "modelName": rng.choice(["NVIDIA B200", "NVIDIA A100"]),
                    "UUID": f"GPU-{p}-{g}", pl: pod, nl: ns, cl: "main", "instance": host + ":9400", "job": "dcgm"}
            if not honor_labels:                              # Prometheus' own target labels ride along
                base.update(pod="dcgm-exporter-xyz", namespace="monitoring", container="exporter")
            r, dup = rng.random(), rng.random() < 0.15
            grouped = dup or 0.3 <= r < 0.4                   # this element is a `sum by` of several series
            kinds = ["idle", "idle", "busy", "burst", "old_burst", "tiny", "tiny", "special", "nan_first"]
            # an all-NaN member would make Prometheus' `sum by` NaN while the dense path cannot tell it from an
            # absent series: only lone series are all NaN
            kind = rng.choice(kinds + ([] if grouped else ["all_nan"]))
            start = rng.choice([0, 0, 0, rng.randrange(30, n_ts)])      # young series
            vals = pattern(kind)
            emit("DCGM_FI_DEV_GPU_UTIL", base, vals, gap=rng.choice([0, 0.05]), start=start)

            def ratios(pkind):
                if pkind == "tiny":                           # ratios are not divided: every ZEROISH value
                    return pattern(pkind, E.ZEROISH)
                v = [x / 100 for x in pattern(pkind)]
                if pkind == "busy":                           # 17-digit ratios
                    v = [rng.choice(E.RATIOS) if x else 0.0 for x in v]
                return v
            if r < 0.3:        # PROF with the identical label set: wins the `or`
                emit("DCGM_FI_PROF_GR_ENGINE_ACTIVE", base, ratios(rng.choice(["idle", "busy", "tiny"])), start=start)
            elif r < 0.4:      # PROF with an extra label: both survive `or`, `sum by` adds them
                emit("DCGM_FI_PROF_GR_ENGINE_ACTIVE", dict(base, profiled="yes"), ratios(rng.choice(["idle", "busy"])))
            if dup:            # `sum by` duplicate: same group, another UUID
                emit("DCGM_FI_DEV_GPU_UTIL", dict(base, UUID=f"GPU-{p}-{g}-b"), pattern(rng.choice(["idle", "busy"])))
            watts = rng.choice(above) if rng.random() < 0.2 else rng.choice(below)
            pw = dict(base)
            pw.pop("modelName") if rng.random() < 0.2 else None
            emit("DCGM_FI_DEV_POWER_USAGE", pw, [watts if i % 17 == 0 else between for i in range(n_ts)])
    # series the selector must ignore: empty pod label; and one that cannot become PodMetricData
    db.append(Q.series("DCGM_FI_DEV_GPU_UTIL", {"Hostname": "node-0", "gpu": "7", "modelName": "x", pl: "",
                                                 nl: "ml-team", cl: "main"}, [(t_eval, 0.0)]))
    return db, t_eval, duration_min


def spell(v, long=False):
    """the wire text of a sample: Prometheus' own spelling, or (long) more than 19 digits, which the device
    parser declines and the CPU re-parses"""
    if long and math.isfinite(v) and 1e-3 <= abs(v) < 1e6:
        return E.long_spelling(v)
    return E.go_float(v)


def wire(db, name, matchers, t_eval, range_s, rng=None):
    """what a range query for `name{matchers}[range]` returns: the matrix wire format.  With `rng`, a fifth of
    the series spell their values with more than 19 digits."""
    res = []
    for s in Q.select(db, name, matchers):
        long = rng is not None and rng.random() < 0.2
        vals = [[t, spell(v, long)] for (t, v) in s.samples if t_eval - range_s < t <= t_eval]
        if vals:
            res.append({"metric": dict(s.labels), "values": vals})
    return {"status": "success", "data": {"resultType": "matrix", "result": res}}


def scenario(seed, t_eval=100_000, long_spellings=True):
    """one cluster, its filters and threshold, the float64 PromQL answer and the three responses"""
    rng = random.Random(seed)
    honor = bool(seed % 2)
    ns_filter = rng.choice([None, None, "ml-.*"])
    model_filter = rng.choice([None, None, "NVIDIA B200"])
    thr = rng.choice([None, 0.0, math.nan] + E.THRESHOLDS * 3)
    step = rng.choice([1, 1, 2, 7])                       # several samples per bucket: the merge decides
    db, t_eval, dur = make_cluster(rng, honor, t_eval=t_eval, thr=thr)
    # (A) Prometheus-style evaluation of the template + the Rust dedup
    vec = Q.evaluate_template(db, t_eval, dur, ns_filter, model_filter, thr, honor)
    n_series, pods_a = Q.unique_pods(vec, honor)
    # (B) selectors -> wire format
    pl, nl = ("pod", "namespace") if honor else ("exported_pod", "exported_namespace")
    m_compute = [(pl, "!=", "")] + ([(nl, "=~", ns_filter)] if ns_filter else [])
    m_power = list(m_compute)
    if model_filter:
        m_compute.append(("modelName", "=~", model_filter))
    rng_s = dur * 60
    spell_rng = rng if long_spellings else None
    util = wire(db, "DCGM_FI_DEV_GPU_UTIL", m_compute, t_eval, rng_s, spell_rng)
    prof = wire(db, "DCGM_FI_PROF_GR_ENGINE_ACTIVE", m_compute, t_eval, rng_s, spell_rng)
    power = wire(db, "DCGM_FI_DEV_POWER_USAGE", m_power, t_eval, rng_s, spell_rng) if thr else None
    return dict(seed=seed, thr=thr, step=step, t_eval=t_eval, dur=dur, db=db, vec=vec, n_series=n_series,
                pods=pods_a, util=util, prof=prof, power=power, m_power=m_power, honor=honor)


def power_veto_f64(sc):
    """(pod, namespace) -> float64 `max_over_time(power) >= thr` of any of its power series (Prometheus' veto)"""
    out = {}
    if not sc["thr"] or math.isnan(sc["thr"]):
        return out
    hot = Q.max_over_time(Q.select(sc["db"], "DCGM_FI_DEV_POWER_USAGE", sc["m_power"]), sc["t_eval"], sc["dur"] * 60)
    for lab, v in hot.items():
        d = dict(lab)
        key = (d.get("exported_pod", d.get("pod")), d.get("exported_namespace", d.get("namespace")))
        out[key] = out.get(key, False) or v >= sc["thr"]
    return out


@pytest.mark.parametrize("seed", range(40))
def test_dense_path_equals_promql_semantics(seed, oracle_np, oracle_c):
    sc = scenario(seed)
    thr, pods_a, n_series, vec = sc["thr"], sc["pods"], sc["n_series"], sc["vec"]
    if not sc["util"]["data"]["result"] and not sc["prof"]["data"]["result"]:
        assert pods_a == []
        return
    H.ingest_mode(-1 if seed % 3 == 0 else seed % 3)      # DOM reference path / threaded text path
    try:
        u, w, meta = H.ingest(sc["util"], sc["prof"], sc["power"], duration_min=sc["dur"], step=sc["step"],
                              t_end=sc["t_eval"], power_threshold=thr)
    finally:
        H.ingest_mode(-1)
    names = [(p["name"], p["namespace"]) for p in meta["pods"]]
    veto_bits = oracle_np.decide(u, w, power_threshold=thr)["veto_bits"]
    # the veto itself, pod by pod, against float64 `max_over_time(power) >= thr`
    veto = oracle_np.unpack_bits(veto_bits, len(names))
    want = power_veto_f64(sc)
    for i, key in enumerate(names):
        assert bool(veto[i]) == want.get(key, False), (seed, key, thr)
    for orc in (oracle_np, oracle_c):
        r = orc.decide(u, w, power_threshold=thr)      # every tensor ROW an element: what the kernels compute
        # duplicate series of a `sum by` group: element = sum of the members' maxima (host-side, ingest.cpp)
        cb, db, counts, _ = H.resolve_groups(r["series_max"], r["candidate_bits"], r["decision_bits"],
                                             (r["n_series"], r["n_candidates"], r["n_decisions"]), veto_bits=veto_bits)
        cand = oracle_np.unpack_bits(cb, len(names))
        pods_b = {names[i] for i in np.flatnonzero(cand)}
        assert pods_b == set(pods_a), (seed, sorted(pods_b ^ set(pods_a)))
        assert counts[0] == n_series
        # the value PodMetricData would carry (lib.rs:184): 0 for every element that survived `== 0`, and the
        # same elements as the PromQL-style evaluation (one per idle group of a surviving pod)
        vals = H.group_values(r["series_max"])
        idle_groups = sum(int((vals[i] == 0.0).sum()) for i in np.flatnonzero(cand))
        assert idle_groups == n_series and all(v == 0.0 for v in vec.values())


def test_the_edges_reach_where_f32_and_float64_differ():
    """the generator is only worth something if its clusters contain the cases: readings that plain rounding would
    flip into a veto, thresholds that are not f32, values that vanish in f32, and spans the device declines"""
    flips, non_f32_thr, vanish, long = 0, 0, 0, 0
    for seed in range(40):
        sc = scenario(seed)
        if sc["thr"] and not math.isnan(sc["thr"]):
            non_f32_thr += float(np.float32(sc["thr"])) != sc["thr"]
            for res in sc["power"]["data"]["result"]:
                flips += any(float(v) in E.f32_rounding_flips(sc["thr"]) for _, v in res["values"])
        for res in sc["util"]["data"]["result"]:
            vs = [float(v) for _, v in res["values"]]
            vanish += any(x != 0 and np.float32(x) == 0 for x in vs)
            long += any(len(v) > 21 for _, v in res["values"])
    assert flips >= 3 and non_f32_thr >= 3 and vanish >= 5 and long >= 5, (flips, non_f32_thr, vanish, long)
    assert "149.999999" in [E.go_float(v) for v in E.power_edges(150.0)]
    assert [E.go_float(x) for x in (5e-07, 1.2345e21, 1e21, 1e-06, -0.0, 150.0, 0.1, 1e20)] == \
        ["5e-07", "1.2345e+21", "1e+21", "0.000001", "-0", "150", "0.1", "100000000000000000000"]


# ---- the same clusters through the device parser, on the emulated device ------------------------------------------
@pytest.fixture(scope="module", params=["tiles", "kernel"])
def emul(request, tmp_path_factory):
    """both flavours of the emulated device (tests/emul_build.py): parser core tile by tile / k_text_parse's source"""
    import emul_build
    return emul_build.build(tmp_path_factory.mktemp("emul_" + request.param), request.param)


def test_emulated_device_ingests_the_edge_clusters_like_the_cpu(emul, tmp_path):
    """tests/cpp/text_emul.cpp ingests each cluster through the CPU text path (whose verdict the test above holds to
    float64 PromQL) and through the device parser, power samples snapped to the cluster's threshold: every tensor
    cell must agree bit for bit — so the device parser's verdict is float64 PromQL's too"""
    dump = lambda j: json.dumps(j, separators=(",", ":"))    # Prometheus' compact encoding: the device path applies
    by_step = {}
    for seed in range(40):
        sc = scenario(seed)
        if not sc["util"]["data"]["result"]:
            continue
        d = tmp_path / f"s{seed}"
        d.mkdir()
        (d / "util.json").write_text(dump(sc["util"]))
        (d / "prof.json").write_text(dump(sc["prof"]))
        if sc["power"] is not None:
            (d / "power.json").write_text(dump(sc["power"]))
            (d / "power_threshold").write_text(repr(sc["thr"]))
        by_step.setdefault((sc["step"], sc["dur"], sc["t_eval"]), []).append(d)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1")
    hard = 0
    for (step, dur, t_eval), dirs in by_step.items():
        r = subprocess.run([emul, str(t_eval), str(step), str(dur)] + [str(x) for x in dirs], capture_output=True,
                           text=True, timeout=600, env=env)
        lines = r.stdout.splitlines()
        assert r.returncode == 0 and len(lines) == len(dirs), (r.stderr[-3000:], [l for l in lines if not l.startswith("OK")][:5])
        assert all(l.startswith("OK") and " device=1 " in l for l in lines), lines[:3]
        hard += sum(int(l.split("hard=")[1].split()[0]) for l in lines)
    assert hard >= 5          # the long spellings went through the CPU re-parse of hard rows


def test_duplicate_dmi_series_is_a_query_error():
    """two node_dmi_info series for one Hostname make Prometheus fail the whole query (many-to-many
    matching) — the error path noted in SURVEY.md §8(a6), not a value path"""
    rng = random.Random(1)
    db, t_eval, dur = make_cluster(rng)
    db.append(Q.series("node_dmi_info", {"instance": "node-0", "product_name": "other"}, [(t_eval - 3, 1.0)]))
    with pytest.raises(ValueError, match="many-to-many"):
        Q.evaluate_template(db, t_eval, dur)
