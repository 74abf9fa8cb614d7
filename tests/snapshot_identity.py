"""Two snapshot files compared by series identity (TEST INFRASTRUCTURE), through the independent reader of
tests/snapshot_ref.py.  Two runs that ingest the same window in a different order (one query, or --query-slice) number
pods and slots differently; what must agree is what each row holds and what the session knows about it:

  grid      span, step, T, t_end, power plane and threshold, selectors, pods_cap and G
  ring      per pod (name, namespace): its util rows as a multiset of (series key, the row's exported chunks) and its
            power rows as a multiset of chunks; no exported row outside a pod's slots
  session   per pod its `sum by` groups (series key -> key of the group's first series), power_slots, has_groups and
            power keys; the known series by their two hashes, with the result and, when placed, the pod and a slot whose
            row holds the same chunks; the PROF signatures and PROF rows by pod and series key

The exported chunks of a row depend on its cells only (not on the ring's head or shape), so equal chunks are equal rows.
mismatch(a, b) -> "" or what differs."""
from collections import Counter

import snapshot_ref as SR

PLACED = 2   # Assigner::Placed


def _key(slot):
    return (slot["hostname"], slot["container"], slot["gpu"], slot["model"], slot["from_prof"])


def _rows(plane):
    """ring row -> its exported chunks (lengths and bytes)"""
    sc, cb, data = plane["series_chunks"], plane["chunk_bytes"], plane["data"]
    out = {}
    for i, r in enumerate(plane["rows"]):
        c0, c1 = int(sc[i]), int(sc[i + 1])
        out[int(r)] = (tuple(int(x) for x in (cb[c0 + 1:c1 + 1] - cb[c0:c1])), bytes(data[int(cb[c0]):int(cb[c1])]))
    return out


def _view(doc):
    G = doc["G"]
    planes = [_rows(p) for p in doc["planes"]] + [{}] * (2 - len(doc["planes"]))
    pods, where = {}, {}
    used = set()
    for i, p in enumerate(doc["pods"]):
        pk = (p["name"], p["ns"])
        util = Counter((_key(s), planes[0].get(i * G + g)) for g, s in enumerate(p["slots"]))
        power = Counter(planes[1].get(i * G + g) for g in range(p["power_slots"]))
        groups = Counter((_key(s), _key(p["slots"][s["group"]])) for s in p["slots"])
        pods[pk] = (util, power, groups, p["power_slots"], p["has_groups"], sorted(doc["power_keys"][i]))
        where[i] = pk
        used.update(range(i * G, i * G + max(len(p["slots"]), p["power_slots"])))
    stray = [r for pl in planes for r in pl if r not in used]
    known = {}
    for h1, h2, res, pod, slot in doc["known"]:
        if res != PLACED:
            known[(h1, h2)] = (res,)
            continue
        p = doc["pods"][pod]
        util = (_key(p["slots"][slot]), planes[0].get(pod * G + slot)) if slot < len(p["slots"]) else None
        power = planes[1].get(pod * G + slot) if slot < p["power_slots"] else None
        known[(h1, h2)] = (res, where[pod], util, power)
    sigs = Counter((where[pod], _key(doc["pods"][pod]["slots"][grp]), tuple(sorted(s))) for (pod, grp), s in doc["prof_sigs"])
    prof_rows = Counter((where[pod], _key(doc["pods"][pod]["slots"][slot])) for pod, slot in doc["prof_rows"])
    grid = {k: doc[k] for k in ("span", "step", "T", "t_end", "power", "power_threshold", "selectors", "pods_cap", "G")}
    return grid, pods, stray, known, sigs, prof_rows


def _known_match(a, b):
    """a placed series matches when its pod is the same and its util row (key and chunks) or its power row is"""
    if a[0] != b[0] or len(a) == 1:
        return len(a) == len(b)
    return a[1] == b[1] and ((a[2] is not None and a[2] == b[2]) or (a[3] is not None and a[3] == b[3]))


def mismatch(blob_a, blob_b):
    ga, pa, sa, ka, xa, ra = _view(SR.read(blob_a, check_crc=False))
    gb, pb, sb, kb, xb, rb = _view(SR.read(blob_b, check_crc=False))
    if ga != gb:
        return "grid %s != %s" % (ga, gb)
    if sa or sb:
        return "exported rows outside every pod's slots: %s / %s" % (sa[:5], sb[:5])
    if pa.keys() != pb.keys():
        return "pods differ: %s" % sorted(set(pa) ^ set(pb))[:5]
    for pk in pa:
        for what, x, y in zip(("util rows", "power rows", "groups", "power_slots", "has_groups", "power keys"), pa[pk], pb[pk]):
            if x != y:
                return "%s of %s differ" % (what, pk)
    if ka.keys() != kb.keys():
        return "known series differ: %d / %d" % (len(ka), len(kb))
    for h in ka:
        if not _known_match(ka[h], kb[h]):
            return "known series %x:%x differs" % h
    if xa != xb:
        return "PROF signatures differ"
    if ra != rb:
        return "PROF rows differ"
    return ""
