"""Scale headroom (lwse_resident_scale_headroom) by its definition (lwse.h, "scale headroom"), without a GPU:

- ``mode="literal"``: for every R from r0 up to min(C_i + 1, R_pig), ``rollout_place_ref`` of the proposal P_i(R)
  (the rollout what-if's forecast, every namespace solved), all R of the query in one batched call; the clean set is
  asserted to be an interval [r0, H];
- ``mode="bisect"``: the device's search: the resident forecast's settled check, E_i(R) built directly, only ns_i
  solved, bisection over (r0, hi) and the final probe at R_pig.

``variant`` names a wrong statement the tests show to be caught: ``"bound_once"`` (one solve at the bound C_i, H one
below the first stranded group), ``"no_settled"`` (answer unsettled rows too, with E built from replicas) and
``"bumped_no_own"`` (LWSE_RPW_BUMPED counting only other objects' rows).  Worlds are those of
``rollout_place_ref``."""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast
from rollout_place_ref import count_row, edge_world, extra_groups, extra_rows, rollout_place_ref, solve

NOT_SETTLED_FC = R.LWSF_ROLLING | R.LWSF_UNFINISHED | R.LWSF_HELD
COUNTERS = ("surge", "placed", "stranded", "own_lost", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed",
            "n_unschedulable", "n_conflict")


def settled_flags(w, row, f, variant=None):
    lr = w.lws[row]
    lf, ff, r0 = int(lr["flags"]), int(f["flags"]), int(lr["replicas"])
    flags = 0
    if not lf & R.LWS_EXCLUSIVE_TOPOLOGY:
        flags |= R.SHR_NOT_EXCLUSIVE
    if ff & (R.LWSF_BAD_TABLE | R.LWSF_NOT_FORECAST):
        flags |= R.SHR_NOT_FORECAST
    if variant != "no_settled" and (
            not lf & R.LWS_STS_EXISTS or lf & R.LWS_UPDATED or r0 < 0 or int(lr["sts_replicas"]) != r0
            or int(lr["sts_partition"]) or int(lr["partition"]) or ff & NOT_SETTLED_FC
            or int(f["peak_sts_replicas"]) != r0 or int(f["final_replicas"]) != r0):
        flags |= R.SHR_NOT_SETTLED
    return flags


def n_extra(w, row, r):
    return len(extra_groups(w, row, r))


def r_pig(w, row):
    """The smallest R with |E(R)| = n_domains + 1."""
    gb, gc = int(w.lws["group_base"][row]), int(w.lws["group_count"][row])
    t, have = w.n_domains + 1, 0
    for g in range(gc):
        if not int(w.groups["flags"][gb + g]) & R.GRP_POD_PRESENT if gb + g < len(w.groups) else False:
            have += 1
            if have == t:
                return g + 1
    return gc + (t - have)


def triggers(o, constraints, variant=None):
    own = 0 if variant == "bumped_no_own" else int(o["own_lost"])
    return bool((constraints & R.RPW_STRANDED and int(o["stranded"]))
                or (constraints & R.RPW_BUMPED and (own or int(o["bumped"]))))


def probe_ns(w, row, ns, r, base):
    """lwse_resident_rollout_place's row of P(r) with only ns solved and E built from r."""
    o = np.zeros(1, R.ROLLOUT_PLACE)[0]
    x = extra_rows(w, row, w.lws[row], ns, extra_groups(w, row, r))
    a = solve(w, x, ns, base, "ns") if len(x) else base
    count_row(w, row, a[len(w.reqs):], a, base, o)
    o["flags"], o["peak"], o["surge"], o["namespaces_solved"] = R.RPL_SOLVED, r, len(x), 1 if len(x) else 0
    return o


def bounds(w, row, c):
    """→ (hi, ceiling bounds it): hi = min(c + 1, R_pig), at least r0 + 1."""
    r0, pig = int(w.lws["replicas"][row]), r_pig(w, row)
    ceil = c >= 0 and c + 1 <= pig
    hi = c + 1 if ceil else pig
    return max(hi, r0 + 1), ceil


def answer(o_flags, r0, h, probe, src):
    a = np.zeros(1, R.SCALE_HEADROOM)[0]
    flags = o_flags
    if int(src["stranded"]):
        flags |= R.SHR_STRANDS
    if int(src["own_lost"]) or int(src["bumped"]):
        flags |= R.SHR_BUMPS
    a["flags"], a["replicas"], a["max_replicas"], a["probe"] = flags, r0, h, probe
    for k in COUNTERS:
        a[k] = src[k]
    return a


def scale_headroom_ref(w, rows, ns, ceilings=None, constraints=R.RPW_STRANDED, mode="bisect", variant=None):
    """→ dict as ``Engine.resident_scale_headroom``: ``rows`` (SCALE_HEADROOM), the totals, ``current`` (the
    rollout placement rows of the resident rows) and, in literal mode, ``probes``: {entry: {R: ROLLOUT_PLACE row}}."""
    rows = np.asarray(rows, dtype=np.int64)
    ns = np.asarray(ns, dtype=np.int64)
    n = len(rows)
    ceil = np.full(n, -1, np.int64) if ceilings is None else np.asarray(ceilings, dtype=np.int64)
    go = oracle.sweep_lws(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, flags=w.flags)[1]
    fc = lws_forecast(w.lws, go, steps=False)["lws"]
    base = oracle.place(w.nodes, w.occ, w.n_domains, w.n_ns, w.reqs, threads=8)
    out = np.zeros(n, R.SCALE_HEADROOM)
    plan = []
    for i in range(n):
        r, r0 = int(rows[i]), int(w.lws["replicas"][rows[i]])
        flags = settled_flags(w, r, fc[r], variant)
        if flags:
            out[i]["flags"], out[i]["replicas"], out[i]["max_replicas"], out[i]["probe"] = flags, r0, -1, -1
            continue
        hi, by_ceil = bounds(w, r, int(ceil[i]))
        plan.append((i, r, r0, hi, by_ceil))
    probes = {}
    if mode == "literal":  # every R of every answered entry in one batched rollout placement, every namespace solved
        q = [(i, r, R_) for i, r, r0, hi, _ in plan for R_ in range(r0, hi + 1)]
        if q:
            recs = R.aligned_empty(len(q), R.LWS_REC)
            for j, (i, r, R_) in enumerate(q):
                recs[j] = w.lws[r]
                recs[j]["replicas"] = R_
            got = rollout_place_ref(w, [r for _, r, _ in q], [int(ns[i]) for i, _, _ in q], recs=recs, mode="literal")["rows"]
            for j, (i, r, R_) in enumerate(q):
                probes.setdefault(i, {})[R_] = got[j]
    for i, r, r0, hi, by_ceil in plan:
        if mode == "literal":
            p = probes[i]
            clean = [not triggers(p[R_], constraints, variant) for R_ in range(r0, hi)]
            k = clean.index(False) if False in clean else len(clean)
            assert not any(clean[k:]), f"entry {i}: the clean R are not an interval"
            get = p.__getitem__
        else:
            cache = {}

            def get(R_, r=r, i=i, cache=cache):
                if R_ not in cache:
                    cache[R_] = probe_ns(w, r, int(ns[i]), R_, base)
                return cache[R_]
        cur = get(r0)
        if triggers(cur, constraints, variant):
            out[i] = answer(R.SHR_SOLVED | R.SHR_BLOCKED, r0, -1, r0, cur)
            continue
        if mode == "literal":
            h = r0 + k - 1
        elif variant == "bound_once":
            top = hi - 1 if by_ceil else hi
            x = get(top)
            gs = extra_groups(w, r, top)
            xo = extra_rows(w, r, w.lws[r], int(ns[i]), gs)
            a = solve(w, xo, int(ns[i]), base, "ns") if len(xo) else base
            placed = (a[len(w.reqs):]["flags"] & R.PLACE_PLACED) != 0
            h = min(top, gs[int(np.flatnonzero(~placed)[0])] if (~placed).any() else top) if triggers(x, constraints) else top
            h = max(h, r0)
        else:
            lo, h_hi = r0, hi
            while h_hi - lo > 1:
                mid = lo + (h_hi - lo) // 2
                if triggers(get(mid), constraints, variant):
                    h_hi = mid
                else:
                    lo = mid
            h = lo
        if h == hi - 1 and by_ceil:
            out[i] = answer(R.SHR_SOLVED | R.SHR_AT_CEILING, r0, h, h, get(h))
        else:
            out[i] = answer(R.SHR_SOLVED, r0, h, h + 1, get(h + 1))
    solved = (out["flags"] & R.SHR_SOLVED) != 0
    blocked = (out["flags"] & R.SHR_BLOCKED) != 0
    ok = solved & ~blocked
    cur_rows = rollout_place_ref(w, rows, ns)["rows"]
    return {"rows": out, "current": cur_rows, "probes": probes, "n_solved": int(solved.sum()),
            "n_blocked": int(blocked.sum()), "n_at_ceiling": int(((out["flags"] & R.SHR_AT_CEILING) != 0).sum()),
            "headroom": int((out["max_replicas"][ok].astype(np.int64) - out["replicas"][ok]).sum())}


# ---- the worlds ----------------------------------------------------------------------------------------------------
# The rollout placement's edge world: stable exclusive objects of size 4, replicas 3, on 16 domains of which exactly 3
# (0, 5, 10) have 4 free slots; namespaces 0 and 1 hold the objects' own groups, 2 is empty, 3 holds three unpinned
# holders of the fitting domains that every extra row beats.  Namespaces 5 .. 9 are added here: each holds the three
# groups of one object (A, B, E1, E2, E3) as unpinned rows of its own priorities, holding the three fitting domains.

OWN_NS = {"A": 5, "B": 6, "E1": 7, "E2": 8, "E3": 9}


def headroom_world(fit_all=False):
    """→ (world, {name: LWS row}).  ``fit_all``: every domain has 4 free slots (a complete object in the empty
    namespace 2 reaches R_pig).  Named objects beyond the rollout edge world's: E1 .. E3 stable; D1 / D2 with
    replicas 2 below group_count 3 (group 2 with / without its leader pod); S1 .. S3 template changes with
    maxSurge 2: S1 UPDATED, S2 not yet flagged (rolling), S3 UPDATED with a held partition, S4 sts_replicas 5 != replicas 3; N not exclusive; IR not forecast."""
    w, rows = edge_world()
    lws, groups = w.lws.copy(), w.groups.copy()
    more = {"E1": 1, "E2": 3, "E3": 5, "D1": 7, "D2": 9, "S1": 11, "S2": 13, "S3": 15, "S4": 17}
    rows = {**rows, **more}
    gb = lambda r: int(lws["group_base"][r])
    for k in ("D1", "D2"):
        lws["replicas"][rows[k]] = lws["sts_replicas"][rows[k]] = 2
    groups["flags"][gb(rows["D2"]) + 2] &= ~np.uint32(R.GRP_POD_PRESENT)
    for k in ("S1", "S2", "S3"):  # template changes with a surge of 2
        lws["rev_hash"][rows[k]] ^= np.uint64(0x9E3779B97F4A7C15)
        lws["max_surge"][rows[k]] = 2
        lws["flags"][rows[k]] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT)
    lws["flags"][rows["S1"]] |= np.uint32(R.LWS_UPDATED)
    lws["flags"][rows["S3"]] |= np.uint32(R.LWS_UPDATED)
    lws["partition"][rows["S3"]] = 2
    lws["sts_replicas"][rows["S4"]] = 5
    nodes = w.nodes.copy()
    if fit_all:
        occ = w.occ.astype(np.int64)
        nodes["capacity"] = np.maximum(nodes["capacity"].astype(np.int64), occ + 4).astype(nodes["capacity"].dtype)
    x = []
    for k, v in OWN_NS.items():
        r = rows[k]
        own = extra_rows(type("W", (), {"lws": lws})(), r, lws[r], v, list(range(int(lws["group_count"][r]))))
        x.append(own)
    x = np.concatenate(x).view(R.PLACE_REQ)
    reqs = R.aligned_empty(len(w.reqs) + len(x), R.PLACE_REQ)
    reqs[: len(w.reqs)] = w.reqs
    reqs[len(w.reqs):] = x
    w.lws, w.groups, w.nodes, w.reqs, w.n_ns = lws, groups, nodes, reqs, 10
    w.occ = R.occupancy_of(w.pod_ident, len(nodes)).astype(np.uint32)
    return w, rows


def edge_queries(w, rows):
    """The edge entries → (rows, ns, ceilings, labels)."""
    q = []

    def e(label, name, ns, c=-1):
        q.append((label, rows[name], ns, c))

    e("k_fits", "A", 2)             # 3 fitting domains: H = r0 + 3
    e("k_fits_other", "B", 2)       # a second object alone takes the same last domains
    e("k_fits_twice_ceiling", "A", 2, 4)  # the same row again, a clean ceiling: AT_CEILING at 4
    e("ceiling_at_r0", "A", 2, 3)   # AT_CEILING at r0
    e("ceiling_below_r0", "A", 2, 1)
    e("ceiling_above_h", "A", 2, 9)  # the ceiling does not bind
    e("headroom_0", "A", 0)         # its own crowded namespace: r0 + 1 strands
    e("holders", "A", 3)            # bumps three holders: STRANDED 6, STRANDED|BUMPED 3
    e("missing_leader", "C", 2)     # group 1 lacks its leader: E(r0) = {1}
    e("blocked", "C", 0)            # ... and strands in the crowded namespace: BLOCKED
    e("below_gc_present", "D1", 2)  # group 2 present: E(3) empty
    e("below_gc_missing", "D2", 2)  # group 2 missing: E(3) = {2}
    for k, v in OWN_NS.items():
        e(f"own_{k}", k, v)         # the object's own unpinned rows hold the fitting domains
    e("updated", "S1", 2)
    e("rolling", "S2", 2)
    e("held", "S3", 2)
    e("scaling", "S4", 2)
    e("not_exclusive", "N", 2)
    e("not_forecast", "IR", 2)
    e("uf", "UF", 2)
    return (np.array([x[1] for x in q], np.uint32), np.array([x[2] for x in q], np.uint32),
            np.array([x[3] for x in q], np.int32), [x[0] for x in q])


def fuzz_query(w, seed, n=40):
    """Seeded entries over every object: the object's own namespace or the empty namespace 2, ceilings mixed."""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, len(w.lws), n).astype(np.uint32)
    ns = np.where(rng.random(n) < 0.5, rows.astype(np.int64) % 2, 2).astype(np.uint32)
    r0 = w.lws["replicas"][rows].astype(np.int64)
    ceil = np.where(rng.random(n) < 0.5, -1, r0 + rng.integers(-2, 8, n)).astype(np.int32)
    return rows, ns, ceil
