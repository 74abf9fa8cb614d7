"""GPU: the verdict of the device ingest + decision kernels against a float64 evaluation of the PromQL expression
(tests/promql_mini.py) — not against the f32 oracles, which share the engine's rounding of each sample.

The clusters are those of tests/test_promql_semantics.py, drawn from tests/edges.py: power readings within an f32
ulp of the threshold on either side (thresholds exact in f32 and not), non-zero utilisation that vanishes in f32,
17-digit PROF ratios, NaN / +-Inf, numbers the device parser declines, millisecond timestamps, several samples per
bucket.  Three levels:
  library  the responses parsed by gpr_text_scan / gpr_text_parse into the device planes (power snapped to the
           threshold), decided by both kernel variants on those planes: candidate pods and veto bits;
  binary   `gpu-pruner` in dry-run with the default GPU ingest, GPR_KERNEL=ldg and =tma: the pods it would scale
           and its `Query returned N series across M unique pods` line;
  daemon   the resident window across ticks while power readings sit at and just below the threshold.
"""
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest

import edges as E
import hostlib as H
import promql_mini as Q
import ticks as TK
from test_promql_semantics import power_veto_f64, scenario

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
NOW = 1_700_000_000
SEEDS = range(12)


@pytest.fixture(scope="module", params=["ldg", "tma"])
def eng(request):
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    e = g.IdleEngine(device=0, kernel=request.param)
    yield e
    e.close()


def _dump(j):
    return json.dumps(j, separators=(",", ":")).encode()     # Prometheus' compact encoding


def _key(labels):
    return labels.get("exported_pod", labels.get("pod")), labels.get("exported_namespace", labels.get("namespace"))


def _rows(sc):
    """the host's row assignment (gpu-pruner_b200/host/ingest_internal.hpp Assigner), restated: pods in order of
    first appearance over PROF, UTIL, POWER; every series its own slot in its pod; a UTIL series with the label set
    of a PROF series of its pod is shadowed; series without pod / namespace (and, for UTIL / PROF, container or
    modelName) get no row.  Returns (pods, G, {text: [row or None per series]})."""
    pods, slots, pslots, out = [], {}, {}, {}
    prof_sigs = {}
    for which in ("prof", "util", "power"):
        resp = sc[which]
        rows = []
        for s in ([] if resp is None else resp["data"]["result"]):
            lab = s["metric"]
            pod, ns = _key(lab)
            ctr = lab.get("exported_container", lab.get("container"))
            if not pod or ns is None or (which != "power" and (ctr is None or "modelName" not in lab)):
                rows.append(None)
                continue
            if (pod, ns) not in slots:
                pods.append((pod, ns))
                slots[(pod, ns)], pslots[(pod, ns)] = 0, 0
            sig = tuple(sorted((k, v) for k, v in lab.items() if k != "__name__"))
            if which == "prof":
                prof_sigs.setdefault((pod, ns), set()).add(sig)
            elif which == "util" and sig in prof_sigs.get((pod, ns), ()):
                rows.append(None)
                continue
            if which == "power":
                rows.append(((pod, ns), pslots[(pod, ns)]))
                pslots[(pod, ns)] += 1
            else:
                rows.append(((pod, ns), slots[(pod, ns)]))
                slots[(pod, ns)] += 1
        out[which] = rows
    G = max([1] + list(slots.values()) + list(pslots.values()))
    index = {k: i for i, k in enumerate(pods)}
    for which, rows in out.items():
        out[which] = [None if r is None else index[r[0]] * G + r[1] for r in rows]
    return pods, G, out


def _spans(eng, text, rows, slot):
    opens, closes = eng.text_scan(text, slot=slot)
    assert len(opens) == len(rows)
    keep = [i for i, r in enumerate(rows) if r is not None]
    spans = np.zeros(len(keep), eng.SPAN_DTYPE)
    for j, i in enumerate(keep):
        vb = int(opens[i]) + 12
        spans[j]["begin"], spans[j]["end"] = vb, int(closes[np.searchsorted(closes, vb)]) + 2
        spans[j]["row"] = rows[i]
    return spans


@pytest.mark.parametrize("seed", SEEDS)
def test_device_planes_decide_like_float64_promql(seed, eng, oracle_np):
    sc = scenario(seed, long_spellings=False)     # Prometheus' own spellings: nothing for a CPU re-parse
    thr, step, dur, t_end = sc["thr"], sc["step"], sc["dur"], sc["t_eval"]
    if not sc["util"]["data"]["result"] and not sc["prof"]["data"]["result"]:
        pytest.skip("no series selected")
    # the host's own ingest of the same responses: its pod table and its window for the exact `sum by`
    H.ingest_mode(0)
    try:
        u_cpu, w_cpu, meta = H.ingest(sc["util"], sc["prof"], sc["power"], duration_min=dur, step=step, t_end=t_end,
                              power_threshold=thr)
    finally:
        H.ingest_mode(-1)
    pods, G, rows = _rows(sc)
    assert pods == [(p["name"], p["namespace"]) for p in meta["pods"]]
    P, T = len(pods), -(-dur * 60 // step)
    n_rows = P * G
    # util plane: PROF first, then UTIL into the same plane; power plane snapped to the threshold
    hard = {0: set(), 1: set()}
    for k, (which, slot) in enumerate((("prof", 0), ("util", 1))):
        text = _dump(sc[which])
        out = eng.text_parse(_spans(eng, text, rows[which], slot), t_end, step, T, n_rows, slot=slot, plane=0,
                             fill=k == 0, window_seconds=dur * 60)
        hard[0] |= set(int(r) for r in out["row"][(out["flags"] & 2) != 0])
    use_power = sc["power"] is not None
    if use_power:
        text = _dump(sc["power"])
        out = eng.text_parse(_spans(eng, text, rows["power"], 2), t_end, step, T, n_rows, slot=2, plane=1,
                             window_seconds=dur * 60, power_threshold=thr)
        hard[1] |= set(int(r) for r in out["row"][(out["flags"] & 2) != 0])
    u_ptr, w_ptr = eng.text_planes()
    # rows the device declined (values below the f64 normal range: 5e-324, 1e-320) take the CPU's row, as in
    # gpu-pruner_b200/host/ingest_device.cpp
    for plane, (ptr, cpu) in enumerate(((u_ptr, u_cpu), (w_ptr, w_cpu))):
        for row in sorted(hard[plane]):
            src = np.ascontiguousarray(cpu.reshape(n_rows, T)[row])
            eng.memcpy(ptr + row * T * 4, src, src.nbytes, 1, 0)
    W = (P + 31) // 32
    db, cb, vb = (eng.host_array((max(W, 1),), np.uint32) for _ in range(3))
    smax = eng.host_array((P, G), np.float32)
    for a in (db, cb, vb):
        a[:] = 0
    r = eng.decide_ptr(u_ptr, P, G, T, db, power=w_ptr if use_power else None, power_threshold=thr if use_power else 0.0,
                       candidate_bits=cb, series_max=smax, veto_bits=vb, in_kind=1, out_kind=0)
    # veto per pod against float64 `max_over_time(power) >= thr`
    want_veto = power_veto_f64(sc)
    veto = oracle_np.unpack_bits(np.asarray(vb), P)
    assert [bool(v) for v in veto] == [want_veto.get(p, False) for p in pods], (seed, thr)
    cand_bits, _, counts, _ = H.resolve_groups(np.asarray(smax), np.asarray(cb), np.asarray(db),
                                               (r.n_series, r.n_candidates, r.n_decisions), veto_bits=np.asarray(vb))
    cand = oracle_np.unpack_bits(cand_bits, P)
    assert {pods[i] for i in np.flatnonzero(cand)} == set(sc["pods"]), seed
    assert counts[0] == sc["n_series"]


def test_the_seeds_cover_the_tma_fallback_and_the_power_edges():
    """a window whose T is not a multiple of 4 sends the tma engine down its LDG path; some threshold must sit where
    plain rounding flips a veto"""
    scs = [scenario(s) for s in SEEDS]
    assert any((-(-sc["dur"] * 60 // sc["step"])) % 4 for sc in scs)
    flips = sum(1 for sc in scs if sc["power"] is not None and sc["thr"] and not math.isnan(sc["thr"])
                for res in sc["power"]["data"]["result"]
                if any(float(v) in E.f32_rounding_flips(sc["thr"]) for _, v in res["values"]))
    assert flips >= 2


# ---- the binary: file:// fixtures, dry-run, both kernels -------------------------------------------------------
def _kube(root, pods):
    """every pod its own Deployment (Pod -> ReplicaSet -> Deployment), old enough to be eligible"""
    def put(plural, ns, obj):
        d = root / plural / ns
        d.mkdir(parents=True, exist_ok=True)
        (d / (obj["metadata"]["name"] + ".json")).write_text(json.dumps(obj))
    for pod, ns in pods:
        put("pods", ns, {"metadata": {"name": pod, "namespace": ns, "uid": f"uid-{ns}-{pod}",
                                      "creationTimestamp": H.rfc3339((NOW - 7200) * 1_000_000_000),
                                      "ownerReferences": [{"kind": "ReplicaSet", "name": f"rs-{pod}", "apiVersion": "apps/v1",
                                                           "uid": "o"}]},
                         "status": {"phase": "Running"}})
        put("replicasets", ns, {"metadata": {"name": f"rs-{pod}", "namespace": ns, "uid": f"rs-{ns}-{pod}",
                                             "ownerReferences": [{"kind": "Deployment", "name": f"dep-{pod}"}]}})
        put("deployments", ns, {"metadata": {"name": f"dep-{pod}", "namespace": ns, "uid": f"dep-{ns}-{pod}",
                                             "resourceVersion": "7"}})


def _run_bin(prom, kube, thr, kernel):
    cmd = [H.BIN, "--prometheus-url", f"file://{prom}", "--kube-fixture", str(kube), "-t", "2", "-g", "300",
           "--now", str(NOW), "-l", "json"]
    if thr is not None:
        cmd += ["--power-threshold", repr(thr)]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=dict(os.environ, GPR_KERNEL=kernel))
    assert p.returncode == 0, p.stderr[-3000:]
    return [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]


@pytest.mark.parametrize("seed", SEEDS)
def test_binary_dry_run_scales_what_float64_promql_returns(seed, tmp_path):
    sc = scenario(seed, t_eval=NOW)
    prom, kube = tmp_path / "prom", tmp_path / "kube"
    prom.mkdir()
    (prom / "util.json").write_bytes(_dump(sc["util"]))
    (prom / "prof.json").write_bytes(_dump(sc["prof"]))
    if sc["power"] is not None:
        (prom / "power.json").write_bytes(_dump(sc["power"]))
    (prom / "query.json").write_text(json.dumps({"end": NOW, "step": sc["step"]}))
    every = {_key(s["metric"]) for w in ("util", "prof") for s in sc[w]["data"]["result"]}
    _kube(kube, sorted(p for p in every if p[0]))
    for kernel in ("ldg", "tma"):
        msgs = _run_bin(prom, kube, sc["thr"], kernel)
        note = [m for m in msgs if m.startswith("Device ingest")]
        assert note and "parsed on the GPU" in note[0], (kernel, msgs[:6])
        assert f"Query returned {sc['n_series']} series across {len(sc['pods'])} unique pods" in msgs, \
            (seed, kernel, [m for m in msgs if m.startswith("Query returned")])
        sent = {(m.group(1), m.group(2)) for m in (re.match(r"Dry-run: Would have sent \[Deployment\] ([^:]+):dep-(\S+) for scaledown", x)
                                                   for x in msgs) if m}
        assert {(pod, ns) for ns, pod in sent} == set(sc["pods"]), (seed, kernel)


# ---- daemon mode: power at and just below the threshold, tick after tick ------------------------------------------
def test_daemon_ticks_veto_like_float64_promql(tmp_path):
    thr, N, step, interval, dur = 150.0, 120, 2, 30, 2
    t0 = NOW
    times = [t0 + N + k * interval for k in range(7)]
    horizon = times[-1] + 5
    below = [v for v in E.power_edges(thr) if v < thr]        # 149.999999, 150 - 2**-18, the f32 and float64 neighbours
    at = [v for v in E.power_edges(thr) if v >= thr]
    store = []
    for p in range(16):
        lab = TK.labels(f"pod-{p}", 0)
        ts = list(range(t0 + 1, horizon + 1, step))
        store.append(("DCGM_FI_DEV_GPU_UTIL", lab, [(t, 0) for t in ts]))
        # pods 0..7: readings just below the threshold all the time, one of them a reading AT it for one tick's slice;
        # pods 8..15: always just below
        hot_tick = p % len(times) if p < 8 else None
        vals = []
        for i, t in enumerate(ts):
            v = below[(p + i) % len(below)]
            if hot_tick is not None and times[hot_tick] - interval < t <= times[hot_tick] and i % 5 == 0:
                v = at[(p + i) % len(at)]
            vals.append((t, v))
        store.append(("DCGM_FI_DEV_POWER_USAGE", lab, vals))
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step, with_power=True)
    cmd = [H.BIN, "--prometheus-url", f"file://{tmp_path}", "-d", "-c", "0", "--max-ticks", str(len(times)), "-t", str(dur),
           "-l", "json", "--power-threshold", repr(thr)]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
    verdicts = [m for m in msgs if m.startswith("Query returned")]
    assert len(verdicts) == len(times)
    db = [Q.series(name, lab, samples) for name, lab, samples in store]
    seen = set()
    for k, (t, v) in enumerate(zip(times, verdicts)):
        vec = Q.evaluate_template(db, t, dur, power_threshold=thr)
        n_series, pods = Q.unique_pods(vec)
        assert v == f"Query returned {n_series} series across {len(pods)} unique pods", (k, v)
        seen.add(len(pods))
    assert len(seen) > 1            # the veto changed from tick to tick
    ingests = [m for m in msgs if m.startswith("Device ingest")]
    assert sum("appended to the resident" in m for m in ingests) >= len(times) - 2, ingests
