"""The drain budget by its definition (lwse.h, "drain budget"), without a GPU:

- ``drain_budget_ref``: the set form — the spec oracle's what-if (``drain_ref.drain_whatif_ref``) for the drained
  node rows, its restarted groups gathered per LWS row against the oracle's LWS results;
- ``drain_budget_cost_ref``: the per-key form — ``drain_ref.restart_pairs`` mapped to keys (the node, or its
  domain) and aggregated by (LWS, key) in numpy;
- ``budget_world``: tables whose objects have several replicas on shared nodes and domains, with maxUnavailable
  spread over its edges, so that floors bind."""
import numpy as np

from drain_ref import RESTART, drain_cost_ref, drain_whatif_ref, restart_pairs
from lws_b200 import records as R

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
EXCLUDED = R.LOUT_BAD_TABLE | R.LOUT_IRREGULAR | R.LOUT_RUP_ERROR | R.LOUT_STATUS_ERROR
COST_FIELDS = ("pods", "leaders", "groups_restarted", "ready_restarted", "pods_recreated")


def budgets(lws, lws_out, n_groups):
    """Per LWS row: (floor, ready_before, evaluated, available, group_base, group_count — 0 when the range
    leaves the group table)."""
    lflags = lws["flags"].astype(np.int64)
    oflags = lws_out["flags"].astype(np.int64)
    reps = lws["replicas"].astype(np.int64)
    mu = lws["max_unavailable"].astype(np.int64)
    mu = np.where((lflags & R.LWS_UNAVAIL_IS_PERCENT) != 0, (mu * reps) // 100, mu)  # rounded down (:302)
    evaluated = ((oflags & EXCLUDED) == 0) & ((lflags & R.LWS_INTSTR_INVALID) == 0)
    floor = np.where(evaluated, np.clip(reps - mu, 0, I32_MAX), 0)
    available = ((oflags & R.LOUT_COND_MASK) >> R.LOUT_COND_SHIFT) == R.COND_AVAILABLE
    gb = lws["group_base"].astype(np.int64)
    gc = np.where(gb + lws["group_count"].astype(np.int64) <= n_groups, lws["group_count"].astype(np.int64), 0)
    return floor, lws_out["ready_replicas"].astype(np.int64), evaluated, available, gb, gc


def owners(lws, groups):
    """Per group row: the LWS row it belongs to (in that row's range, inside the table, with lws_index naming
    it), or -1."""
    n_groups = len(groups)
    gb = lws["group_base"].astype(np.int64)
    gcount = lws["group_count"].astype(np.int64)
    li = groups["lws_index"].astype(np.int64)
    ok = li < len(lws)
    L = np.where(ok, li, 0)
    g = np.arange(n_groups)
    if len(lws) == 0:
        return np.full(n_groups, -1, np.int64)
    member = ok & (gb[L] + gcount[L] <= n_groups) & (g >= gb[L]) & (g < gb[L] + gcount[L])
    return np.where(member, li, -1)


def _verdicts(floor, ready_before, evaluated, available, restarted, lost, lost_nb):
    after = np.clip(ready_before - lost, I32_MIN, I32_MAX)
    below = evaluated & (ready_before < floor)
    breached = evaluated & (lost > 0) & (after < floor)
    loses = evaluated & available & (lost_nb > 0)
    flags = (np.where(~evaluated, R.DRAINB_NOT_EVALUATED, 0) | np.where(below, R.DRAINB_ALREADY_BELOW, 0)
             | np.where(breached, R.DRAINB_BREACHED, 0) | np.where(loses, R.DRAINB_LOSES_AVAILABLE, 0))
    return after, flags


def drain_budget_ref(lws, groups, pod_state, pod_ident, nodes, drain, flags=0, base=None):
    """The set form for node rows ``drain``: rows (DRAIN_BUDGET, sorted by LWS row) and the totals.  ``base``:
    the oracle's (lws_out, group_out) of the tables as they are."""
    import oracle

    if base is None:
        base = oracle.sweep_lws(lws, groups, pod_state, pod_ident, nodes, flags)[:2]
    lws_out, before = base
    wf = drain_whatif_ref(lws, groups, pod_state, pod_ident, nodes, drain, flags, base=base)
    after = wf["after_all"]
    hit = ((before["flags"] & RESTART) == 0) & ((after["flags"] & RESTART) != 0)
    own = owners(lws, groups)
    floor, ready, evaluated, available, gb, _ = budgets(lws, lws_out, len(groups))
    n = len(lws)
    sel = hit & (own >= 0)
    o = own[sel]
    ready_g = (before["flags"][sel] & R.GOUT_COND_READY) != 0
    idx = np.flatnonzero(sel) - gb[o]
    restarted = np.bincount(o, minlength=n)[:n]
    lost = np.bincount(o[ready_g], minlength=n)[:n]
    lost_nb = np.bincount(o[ready_g & (idx < lws["replicas"][o])], minlength=n)[:n]
    after_r, fl = _verdicts(floor, ready, evaluated, available, restarted, lost, lost_nb)
    touched = np.flatnonzero(restarted > 0)
    rows = np.zeros(len(touched), R.DRAIN_BUDGET)
    rows["lws"] = touched
    rows["flags"] = fl[touched]
    rows["replicas"] = lws["replicas"][touched]
    rows["floor"] = floor[touched]
    rows["ready_before"] = ready[touched]
    rows["ready_after"] = after_r[touched]
    rows["groups_restarted"] = restarted[touched]
    totals = {"n_touched": len(touched),
              "n_breached": int(((fl[touched] & R.DRAINB_BREACHED) != 0).sum()),
              "n_loses_available": int(((fl[touched] & R.DRAINB_LOSES_AVAILABLE) != 0).sum()),
              "n_already_below": int(((fl & R.DRAINB_ALREADY_BELOW) != 0).sum())}
    totals.update({k: wf[k] for k in ("n_pods_evicted", "n_leaders_evicted", "n_groups_restarted",
                                      "n_ready_restarted", "n_pods_recreated")})
    return rows, totals


def domain_nodes(nodes, n_domains, domains):
    """The node rows a drain of the domain ids ``domains`` drains: by domain_id alone."""
    d = nodes["domain_id"].astype(np.int64)
    return np.flatnonzero((d < n_domains) & np.isin(d, np.asarray(list(domains), dtype=np.int64)))


def key_of(nodes, n_domains, by_domain):
    """Per node row: its key (the row, or its domain id; -1 for a node in no domain)."""
    if not by_domain:
        return np.arange(len(nodes))
    d = nodes["domain_id"].astype(np.int64)
    return np.where(d < n_domains, d, -1)


def drain_budget_cost_ref(lws, lws_out, groups, pod_state, pod_ident, nodes, n_domains, base_out, by_domain=False):
    """The per-key form: one DRAIN_BUDGET_COST row per node (or per domain)."""
    n_nodes = len(nodes)
    n_keys = n_domains if by_domain else n_nodes
    out = np.zeros(n_keys, R.DRAIN_BUDGET_COST)
    key = key_of(nodes, n_domains, by_domain)
    node_cost = drain_cost_ref(lws, groups, pod_state, pod_ident, n_nodes, base_out)
    if not by_domain:
        for f in COST_FIELDS:
            out[f] = node_cost[f]
    else:
        has = key >= 0
        out["pods"] = np.bincount(key[has], weights=node_cost["pods"][has], minlength=n_keys)[:n_keys]
        out["leaders"] = np.bincount(key[has], weights=node_cost["leaders"][has], minlength=n_keys)[:n_keys]
    g, n = restart_pairs(lws, groups, pod_state, pod_ident, n_nodes, base_out)
    k = key[n]
    keep = k >= 0
    pairs = np.unique(np.stack([g[keep], k[keep]], axis=1), axis=0) if keep.any() else np.zeros((0, 2), np.int64)
    g, k = pairs[:, 0], pairs[:, 1]
    ready = (base_out["flags"][g] & R.GOUT_COND_READY) != 0
    if by_domain:
        out["groups_restarted"] = np.bincount(k, minlength=n_keys)[:n_keys]
        out["ready_restarted"] = np.bincount(k[ready], minlength=n_keys)[:n_keys]
        rec = np.zeros(n_keys, np.uint64)
        np.add.at(rec, k, groups["pod_count"][g].astype(np.uint64))
        out["pods_recreated"] = rec
    # (LWS, key) entries of the groups that belong to their LWS row
    own = owners(lws, groups)
    m = own[g] >= 0
    L, k, ready, g = own[g][m], k[m], ready[m], g[m]
    floor, rb, evaluated, available, gb, _ = budgets(lws, lws_out, len(groups))
    ready_nb = ready & ((g - gb[L]) < lws["replicas"][L])
    out["min_margin"] = I32_MAX
    if len(L) == 0:
        return out
    ent, inv = np.unique(np.stack([L, k], axis=1), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    lost = np.bincount(inv, weights=ready, minlength=len(ent)).astype(np.int64)
    lost_nb = np.bincount(inv, weights=ready_nb, minlength=len(ent)).astype(np.int64)
    EL, EK = ent[:, 0], ent[:, 1]
    after, fl = _verdicts(floor[EL], rb[EL], evaluated[EL], available[EL], np.ones(len(ent)), lost, lost_nb)
    out["lws_touched"] = np.bincount(EK, minlength=n_keys)[:n_keys]
    out["lws_breached"] = np.bincount(EK[(fl & R.DRAINB_BREACHED) != 0], minlength=n_keys)[:n_keys]
    out["lws_loses_available"] = np.bincount(EK[(fl & R.DRAINB_LOSES_AVAILABLE) != 0], minlength=n_keys)[:n_keys]
    ev = evaluated[EL]
    margin = np.clip(after - floor[EL], I32_MIN, I32_MAX)
    mm = np.full(n_keys, I32_MAX, np.int64)
    np.minimum.at(mm, EK[ev], margin[ev])
    out["min_margin"] = mm
    return out


def budget_world(n_lws=4000, n_nodes=512, seed=17):
    """synth tables where floors bind: 4-16 replicas of 4-8 pods, groups packed onto shared nodes of 8-node
    domains, maxUnavailable over 0, 1, 2, 25 %, 50 %, 100 % and 33 %, most objects with a restart policy."""
    from lws_b200 import synth

    p = synth.Profile("breach", n_lws, size_choices=(4, 8), replicas_choices=(3, 4, 6, 8, 16), n_nodes=n_nodes,
                      nodes_per_domain=8, node_capacity=4096, max_surge=((0, False), (1, False), (2, False)),
                      max_unavailable=((0, False), (1, False), (2, False), (20, False), (0, True), (25, True),
                                       (33, True), (50, True), (100, True)),
                      f_mid_update=0.1, p_group_ready=0.9, p_leader_unscheduled=0.02, restart_policy_p=(0.1, 0.7, 0.2))
    return synth.make(p, seed=seed)


def budget_row_of_cost(row):
    """The set-form totals a per-key row stands for: {total name: value}."""
    return {"n_pods_evicted": int(row["pods"]), "n_leaders_evicted": int(row["leaders"]),
            "n_groups_restarted": int(row["groups_restarted"]), "n_ready_restarted": int(row["ready_restarted"]),
            "n_pods_recreated": int(row["pods_recreated"]), "n_touched": int(row["lws_touched"]),
            "n_breached": int(row["lws_breached"]), "n_loses_available": int(row["lws_loses_available"])}


def min_margin_of(rows):
    ev = (rows["flags"] & R.DRAINB_NOT_EVALUATED) == 0
    if not ev.any():
        return I32_MAX
    return int(np.clip(rows["ready_after"][ev].astype(np.int64) - rows["floor"][ev], I32_MIN, I32_MAX).min())
