"""Rollout placement (lwse_resident_rollout_place) by its definition (lwse.h, "rollout placement"), without a GPU:

- ``mode="literal"``: per entry the forecast reference (``lws_forecast_ref.lws_forecast`` over the oracle's sweep, or
  ``rollout_whatif_ref.rollout_whatif`` for a proposal), then E_i, then ``test_place_whatif.whatif_ref`` with E_i as
  its extra rows over every namespace;
- ``mode="ns"``: the same rows when only ns_i is solved and every other row keeps its baseline row — what the
  device computes.

``variant`` names a wrong statement the tests show to be caught: ``"no_pod_present"`` (E_i only the groups at or
beyond group_count), ``"replicas_surge"`` (replicas + surge instead of the forecast's peak) and ``"together"``
(every entry's E_i in one round).  Worlds are ``types.SimpleNamespace`` objects with lws, groups, pod_state,
pod_ident, nodes, n_domains, flags, occ, reqs and n_ns."""
from __future__ import annotations

import types

import numpy as np

import oracle
from lws_b200 import informer, synth
from lws_b200 import records as R
from lws_forecast_ref import _scaled_surge, lws_forecast
from rollout_whatif_ref import rollout_whatif
from test_place_whatif import whatif_ref

EXCL = np.uint32(R.LWS_EXCLUSIVE_TOPOLOGY)


def world_of(t, n_ns=None, reqs=None):
    """A synth Tables (or any object with its fields) with its request rows, occupancy and namespace count."""
    reqs = t.place_requests() if reqs is None else reqs
    n_ns = max(int(t.n_namespaces), 1) if n_ns is None else n_ns
    occ = R.occupancy_of(t.pod_ident, len(t.nodes)).astype(np.uint32)
    return types.SimpleNamespace(lws=t.lws, groups=t.groups, pod_state=t.pod_state, pod_ident=t.pod_ident, nodes=t.nodes,
                                 n_domains=t.n_domains, flags=t.flags, occ=occ, reqs=reqs, n_ns=n_ns)


def forecasts(w, rows, recs=None):
    """F_i per entry: the resident forecast's row of L_i, or the rollout what-if's row of (L_i, P_i)."""
    if recs is None:
        go = oracle.sweep_lws(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, flags=w.flags)[1]
        return lws_forecast(w.lws, go, steps=False)["lws"][np.asarray(rows, dtype=np.int64)]
    return rollout_whatif(w, rows, recs, steps=False)["lws"]


def extra_groups(w, row, peak, variant=None):
    """E_i's group indices, ascending."""
    gb, gc = int(w.lws["group_base"][row]), int(w.lws["group_count"][row])
    gs = []
    for g in range(max(peak, 0)):
        if g >= gc:
            gs.append(g)
        elif variant != "no_pod_present" and not (int(w.groups["flags"][gb + g]) & R.GRP_POD_PRESENT):
            gs.append(g)
    return gs


def extra_rows(w, row, rec, ns, gs):
    """E_i's request rows: the informer's what-if rows (the encoder's mix) with the group rows of L_i's range."""
    x = informer.IncrementalEncoder._whatif_requests(int(rec["uid_hash"]), int(rec["size"]), ns, gs)
    x["group"] = (x["group"].astype(np.int64) + int(w.lws["group_base"][row])).astype(np.uint32)
    return x


def entry_flags(w, row, rec, f):
    lr = w.lws[row]
    flags = 0
    if not (int(lr["flags"]) & R.LWS_EXCLUSIVE_TOPOLOGY):
        flags |= R.RPL_NOT_EXCLUSIVE
    if int(f["flags"]) & (R.LWSF_BAD_TABLE | R.LWSF_NOT_FORECAST):
        flags |= R.RPL_NOT_FORECAST
    if int(rec["size"]) != int(lr["size"]) or (int(rec["flags"]) ^ int(lr["flags"])) & R.LWS_EXCLUSIVE_TOPOLOGY:
        flags |= R.RPL_NOT_MODELLED
    return flags


def solve(w, extra, ns, base, mode):
    """The what-if rows (resident rows then the extra rows) of one entry's composed query."""
    if mode == "literal":
        return whatif_ref(w.nodes, w.occ, w.n_domains, w.reqs, extra=extra, n_ns=w.n_ns)["after_all"]
    reqs = w.reqs.copy()
    other = (reqs["ns"] != ns) & (reqs["ns"] < w.n_ns)
    reqs["ns"][other] = w.n_ns  # out of the round: the baseline row stays
    all_reqs = R.aligned_empty(len(reqs) + len(extra), R.PLACE_REQ)
    all_reqs[: len(reqs)] = reqs
    all_reqs[len(reqs):] = extra
    after = oracle.place(w.nodes, w.occ, w.n_domains, w.n_ns, all_reqs, threads=8)
    after[: len(reqs)][other] = base[other]
    return after


def count_row(w, row, extra_out, after, base, out, n_extra_rows=None):
    n_res = len(w.reqs)
    res = after[:n_res]
    was = (base["flags"] & R.PLACE_PLACED) != 0
    now = (res["flags"] & R.PLACE_PLACED) != 0
    gb, gc = int(w.lws["group_base"][row]), int(w.lws["group_count"][row])
    grp = w.reqs["group"].astype(np.int64)
    own = (grp >= gb) & (grp < gb + gc)
    a = base.view(np.uint8).reshape(n_res, 16)
    b = res.view(np.uint8).reshape(n_res, 16)
    f = after["flags"]
    xp = (extra_out["flags"] & R.PLACE_PLACED) != 0
    out["placed"] = int(xp.sum())
    out["stranded"] = int((~xp).sum())
    out["own_lost"] = int((own & was & ~now).sum())
    out["bumped"] = int((~own & was & ~now).sum())
    out["n_changed"] = int((a != b).any(axis=1).sum())
    out["n_lost"] = int((was & ~now).sum())
    out["n_moved"] = int((was & now & (base["domain_id"] != res["domain_id"])).sum())
    out["n_gained"] = int((~was & now).sum())
    out["n_placed"] = int(((f & R.PLACE_PLACED) != 0).sum())
    out["n_unschedulable"] = int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum())
    out["n_conflict"] = int(((f & R.PLACE_CONFLICT) != 0).sum())


def rollout_place_ref(w, rows, ns, recs=None, mode="ns", variant=None):
    """→ dict as ``Engine.resident_rollout_place``: ``rows`` (ROLLOUT_PLACE), the totals, and ``extra`` (E_i's rows
    per entry, for the tests)."""
    rows = np.asarray(rows, dtype=np.int64)
    ns = np.asarray(ns, dtype=np.int64)
    n = len(rows)
    fc = forecasts(w, rows, recs)
    base = oracle.place(w.nodes, w.occ, w.n_domains, w.n_ns, w.reqs, threads=8)
    out = np.zeros(n, R.ROLLOUT_PLACE)
    extras = [R.aligned_empty(0, R.PLACE_REQ)] * n
    recs_of = [w.lws[r] if recs is None else recs[i] for i, r in enumerate(rows)]
    for i in range(n):
        r, rec, f = int(rows[i]), recs_of[i], fc[i]
        o = out[i]
        o["fc_flags"], o["peak"] = f["flags"], f["peak_sts_replicas"]
        flags = entry_flags(w, r, rec, f)
        if flags:
            o["flags"] = flags
            out[i] = o
            continue
        peak = int(f["peak_sts_replicas"])
        if variant == "replicas_surge":
            peak = int(rec["replicas"]) + int(_scaled_surge(np.array([rec], dtype=R.LWS_REC))[0])
        extras[i] = extra_rows(w, r, rec, int(ns[i]), extra_groups(w, r, peak, variant))
        o["flags"] = R.RPL_SOLVED
        o["surge"] = len(extras[i])
        out[i] = o
    solved = [i for i in range(n) if out[i]["flags"] & R.RPL_SOLVED]
    if variant == "together":
        allx = np.concatenate([extras[i] for i in solved]) if solved else R.aligned_empty(0, R.PLACE_REQ)
        allx = np.ascontiguousarray(allx).view(R.PLACE_REQ)
        after = whatif_ref(w.nodes, w.occ, w.n_domains, w.reqs, extra=allx, n_ns=w.n_ns)["after_all"]
    at = 0
    for i in solved:
        x = extras[i]
        o = out[i]
        if variant == "together":
            a_i = np.concatenate([after[: len(w.reqs)], after[len(w.reqs) + at: len(w.reqs) + at + len(x)]])
            at += len(x)
        elif len(x):
            a_i = solve(w, x, int(ns[i]), base, mode)
        else:
            a_i = base  # no extra row: nothing is solved, every row keeps its baseline row
        count_row(w, int(rows[i]), a_i[len(w.reqs):], a_i, base, o)
        o["namespaces_solved"] = 1 if len(x) else 0
        if o["stranded"]:
            o["flags"] |= R.RPL_STRANDS
        if o["bumped"]:
            o["flags"] |= R.RPL_BUMPS
        out[i] = o
    return {"rows": out, "extra": extras, "n_solved": len(solved),
            "n_strands": int(((out["flags"] & R.RPL_STRANDS) != 0).sum()),
            "n_surge": int(out["surge"].astype(np.int64).sum()),
            "n_stranded": int(out["stranded"].astype(np.int64).sum())}


def proposals(lws, rows, seed):
    """Proposals on ``rows``: replicas up and down, integer and percent maxSurge, template bumps, identity; a few
    that change size or the exclusive bit (flagged NOT_MODELLED)."""
    rng = np.random.default_rng(seed)
    rows = np.asarray(rows, dtype=np.int64)
    n = len(rows)
    recs = R.aligned_empty(n, R.LWS_REC)
    recs[:] = lws[rows]
    kind = rng.integers(0, 7, n)
    up = kind == 0
    recs["replicas"][up] += rng.integers(1, 6, int(up.sum())).astype(np.int32)
    dn = kind == 1
    recs["replicas"][dn] = np.maximum(recs["replicas"][dn] - rng.integers(1, 4, int(dn.sum())), 0)
    su = kind == 2
    pct = rng.random(n) < 0.5
    recs["max_surge"][su] = np.where(pct, rng.integers(0, 120, n), rng.integers(0, 4, n))[su]
    f = recs["flags"]
    f[su] = (f[su] & ~np.uint32(R.LWS_SURGE_IS_PERCENT)) | np.where(pct, R.LWS_SURGE_IS_PERCENT, 0).astype(np.uint32)[su]
    tm = kind == 3
    recs["rev_hash"][tm] = rng.integers(1, 2**63, int(tm.sum()), dtype=np.uint64)
    f[tm] |= np.uint32(R.LWS_UPDATED)
    sz = (kind == 4) & (rng.random(n) < 0.3)
    recs["size"][sz] += 1
    ex = (kind == 5) & (rng.random(n) < 0.3)
    f[ex] ^= EXCL
    recs["flags"] = f
    return rows.astype(np.uint32), recs


def fuzz_world(seed, scale=0.3):
    """A fuzz-profile world (40 % exclusive, mixed surge) with its objects dealt to three namespaces."""
    p = synth.profile("fuzz", scale)
    p.n_namespaces = 3
    return world_of(synth.make(p, seed=seed))


def edge_world():
    """A world with one case per edge of the definition.  Stable exclusive objects of size 4 with 3 groups (all
    present, scheduled and ready) in namespaces 0 and 1, on 16 domains of which exactly 3 have 4 free slots and the
    others 3 (size − 1).  Namespace 2 is empty; namespace 3 holds three unpinned rows of the lowest priority that
    hold the three fitting domains; namespace 4 holds 1 020 rows, 252 of them unpinned (and too big to fit), the
    rest pinned on node 0, so that 4 and 5 extra rows cross 1 024 / 1 025 rows and 256 / 257 unpinned rows.  Object
    C lacks the leader pod of group 1 and has group 0 unpinned; D is scaling down from 3 to 2 with group 2's pod
    missing; N is not exclusive; BT's range lies outside the group table; IR is IRREGULAR.  UF's forecast is
    UNFINISHED (the n' > C construction of the forecast edge tests): a pending template change with maxSurge =
    replicas = 3, maxUnavailable -1 and sts_replicas 6, so the first pass asks for n' = 7 > C = 6; its peak is the
    StatefulSet's 6 replicas, and groups 3 .. 5 are extra.
    → (world, {name: LWS row})."""
    p = synth.Profile("edge", 24, size_choices=(4,), replicas_choices=(3,), n_nodes=32, nodes_per_domain=2,
                      node_capacity=64, f_no_sts=0.0, f_mid_update=0.0, p_group_ready=1.0, p_exclusive=1.0,
                      p_leader_unscheduled=0.0, p_restarted=0.0, p_deleting=0.0, p_pending=0.0, p_short_group=0.0,
                      n_namespaces=2, conflict_free=True)
    t = synth.make(p, seed=5)
    lws, groups = t.lws.copy(), t.groups.copy()
    rows = {"A": 0, "B": 2, "C": 4, "D": 6, "N": 8, "BT": 10, "IR": 12, "UF": 14}
    gb = lambda r: int(lws["group_base"][r])
    groups["flags"][gb(rows["C"]) + 1] &= ~np.uint32(R.GRP_POD_PRESENT)
    groups["leader_node"][gb(rows["C"])] = R.NONE
    lws["replicas"][rows["D"]] = 2
    groups["flags"][gb(rows["D"]) + 2] &= ~np.uint32(R.GRP_POD_PRESENT)
    lws["flags"][rows["N"]] &= ~EXCL
    lws["group_base"][rows["BT"]] = len(groups)
    lws["flags"][rows["IR"]] |= np.uint32(R.LWS_IRREGULAR)
    uf = rows["UF"]
    lws["rev_hash"][uf] ^= np.uint64(0x9E3779B97F4A7C15)
    lws["flags"][uf] = (lws["flags"][uf] | np.uint32(R.LWS_UPDATED)) & ~np.uint32(R.LWS_SURGE_IS_PERCENT | R.LWS_UNAVAIL_IS_PERCENT)
    lws["max_surge"][uf], lws["max_unavailable"][uf], lws["sts_replicas"][uf] = 3, -1, 6
    t.lws, t.groups = lws, groups
    nodes = t.nodes.copy()
    occ = R.occupancy_of(t.pod_ident, len(nodes)).astype(np.int64)
    dom = nodes["domain_id"].astype(np.int64)
    free = np.zeros(len(nodes), np.int64)
    for d in range(t.n_domains):  # domain free slots: 4 for domains 0, 5, 10; 3 for the others
        on = np.flatnonzero(dom == d)
        want = 4 if d in (0, 5, 10) else 3
        free[on[0]] = want - (len(on) - 1)
        free[on[1:]] = 1
    nodes["capacity"] = (occ + free).astype(nodes["capacity"].dtype)
    t.nodes = nodes
    reqs = encoder_rows(t)
    rng = np.random.default_rng(7)
    raw = []
    for _ in range(3):  # namespace 3: holders every extra row beats
        raw.append((0xFFFFFFFFFFFFFFFF, int(rng.integers(0, 1 << 62)), R.NONE, 3, 4, R.NONE))
    for i in range(1020):  # namespace 4
        raw.append((int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 62)), R.NONE, 4, 100 if i < 252 else 1,
                    R.NONE if i < 252 else 0))
    x = R.aligned_empty(len(raw), R.PLACE_REQ)
    for i, r in enumerate(raw):
        x[i] = r
    all_reqs = R.aligned_empty(len(reqs) + len(x), R.PLACE_REQ)
    all_reqs[: len(reqs)] = reqs
    all_reqs[len(reqs):] = x
    return world_of(t, n_ns=5, reqs=all_reqs), rows


def encoder_rows(t):
    from lws_b200 import encoder

    return encoder.encode_place_requests(t.lws, t.groups, t.ns_of_lws)


def edge_queries(w, rows):
    """The edge world's resident query and proposal query → ((rows, ns), (rows, ns, recs), labels of the proposals)."""
    names = list(rows)
    res_rows = np.array([rows[k] for k in names], np.uint32)
    res_ns = w_ns(w, res_rows)
    A, B = rows["A"], rows["B"]
    props = []

    def prop(label, r, ns, **kw):
        rec = w.lws[r].copy()
        for k, v in kw.items():
            rec[k] = v
        props.append((label, r, ns, rec))

    prop("k_fits", A, 2, replicas=6)            # surge 3 into the 3 fitting domains of namespace 2
    prop("k_plus_1_strands", A, 2, replicas=7)  # surge 4: one stranded
    prop("other_k_fits", B, 2, replicas=6)      # a second object, answered on its own
    prop("bumps", A, 3, replicas=6)             # surge 3 beats the three holders of namespace 3
    prop("rows_1024", A, 4, replicas=7)         # 1 020 + 4 rows, 252 + 4 unpinned
    prop("rows_1025", A, 4, replicas=8)         # 1 020 + 5 rows, 252 + 5 unpinned
    bump = int(w.lws["flags"][A]) | R.LWS_UPDATED
    prop("surge_0", A, 2, rev_hash=12345, flags=bump, max_surge=0)
    prop("surge_2", A, 2, rev_hash=12345, flags=bump, max_surge=2)
    prop("size_edit", A, 2, size=5)
    prop("exclusive_edit", A, 2, flags=int(w.lws["flags"][A]) & ~R.LWS_EXCLUSIVE_TOPOLOGY)
    prop("identity_c", rows["C"], int(w_ns(w, [rows["C"]])[0]))
    prop("identity_uf", rows["UF"], int(w_ns(w, [rows["UF"]])[0]))
    recs = R.aligned_empty(len(props), R.LWS_REC)
    for i, pr in enumerate(props):
        recs[i] = pr[3]
    return ((res_rows, res_ns), (np.array([pr[1] for pr in props], np.uint32), np.array([pr[2] for pr in props], np.uint32),
                                 recs), [pr[0] for pr in props])


def w_ns(w, rows):
    """The namespace of each object's requests (synth deals objects to namespaces round-robin)."""
    return (np.asarray(rows, dtype=np.int64) % 2).astype(np.uint32)
