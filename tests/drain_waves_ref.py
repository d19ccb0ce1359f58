"""Drain waves (lwse_resident_drain_waves) by its definition (lwse.h, "drain waves"), without a GPU:

- ``plan_literal``: first-fit where every probe is the set form ``drain_budget_ref`` over the candidate node set
  (the spec oracle's what-if each time) — the definition as written;
- ``plan_fast``: the same plan from ``drain_ref.restart_pairs`` and per-(LWS, wave) lost counters — what the
  device computes, and fast enough for the breach world and C3;
- ``waves_edges_world``: a hand-built world with one object per edge of the plan (see its docstring).

Both planners return (keys: DRAIN_WAVE_KEY rows in query order, waves: DRAIN_WAVE rows, totals dict)."""
import os
import re

import numpy as np

from drain_budget_ref import (I32_MAX, I32_MIN, budgets, domain_nodes, drain_budget_cost_ref, drain_budget_ref, key_of,
                              min_margin_of, owners)
from drain_ref import restart_pairs
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = R.NONE


def plan_threads() -> int:
    """(pair, wave) items the plan kernel takes per pass, read from the kernel source."""
    src = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_drain_wave_kernels.cu")).read()
    return int(re.search(r"constexpr uint32_t kPlanThreads = (\d+);", src).group(1))


def _key_nodes(nodes, n_domains, by_domain, ids):
    return domain_nodes(nodes, n_domains, ids) if by_domain else np.asarray(list(ids), dtype=np.int64)


def _totals(keys, n_waves):
    st = keys["status"]
    return {"n_waves": n_waves, "n_planned": int((st == R.DRAINW_PLANNED).sum()),
            "n_breaches_alone": int((st == R.DRAINW_BREACHES_ALONE).sum()), "n_no_wave": int((st == R.DRAINW_NO_WAVE).sum())}


def wave_row_of_set(rows, totals, n_keys):
    """A DRAIN_WAVE row from the set form's rows and totals over a wave's ids."""
    w = np.zeros(1, R.DRAIN_WAVE)[0]
    w["n_keys"] = n_keys
    w["lws_touched"] = totals["n_touched"]
    w["lws_loses_available"] = totals["n_loses_available"]
    for f in ("n_pods_evicted", "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted", "n_pods_recreated"):
        w[f] = totals[f]
    w["min_margin"] = min_margin_of(rows)
    return w


def plan_literal(lws, groups, pst, pid, nodes, n_domains, ids, by_domain=False, max_waves=64, flags=0, base=None):
    """First-fit by the definition: each probe is ``drain_budget_ref`` over W ∪ {k}."""
    import oracle

    if base is None:
        base = oracle.sweep_lws(lws, groups, pst, pid, nodes, flags)[:2]
    cost = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, n_domains, base[1], by_domain)
    probe = lambda ks: drain_budget_ref(lws, groups, pst, pid, nodes, _key_nodes(nodes, n_domains, by_domain, ks),
                                        flags, base=base)
    keys = np.zeros(len(ids), R.DRAIN_WAVE_KEY)
    waves = []
    for i, k in enumerate(int(x) for x in ids):
        row = keys[i]
        row["id"], row["wave"] = k, NONE
        for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
            row[f] = cost[k][f]
        if probe([k])[1]["n_breached"] > 0:
            row["status"] = R.DRAINW_BREACHES_ALONE
            continue
        for w, W in enumerate(waves):
            if probe(W + [k])[1]["n_breached"] == 0:
                W.append(k)
                row["wave"] = w
                break
        else:
            if len(waves) < max_waves:
                waves.append([k])
                row["wave"] = len(waves) - 1
            else:
                row["status"] = R.DRAINW_NO_WAVE
    out = np.zeros(len(waves), R.DRAIN_WAVE)
    for w, W in enumerate(waves):
        rows, tot = probe(W)
        assert tot["n_breached"] == 0
        out[w] = wave_row_of_set(rows, tot, len(W))
    return keys, out, _totals(keys, len(waves))


def plan_fast(lws, lws_out, groups, pst, pid, nodes, n_domains, base_out, ids, by_domain=False, max_waves=64):
    """First-fit from the restart pairs: per wave the set of its groups and lost(L, W) per LWS row."""
    n_keys = n_domains if by_domain else len(nodes)
    cost = drain_budget_cost_ref(lws, lws_out, groups, pst, pid, nodes, n_domains, base_out, by_domain)
    g, n = restart_pairs(lws, groups, pst, pid, len(nodes), base_out)
    k = key_of(nodes, n_domains, by_domain)[n]
    pairs = np.unique(np.stack([k[k >= 0], g[k >= 0]], axis=1), axis=0) if (k >= 0).any() else np.zeros((0, 2), np.int64)
    starts = np.searchsorted(pairs[:, 0], np.arange(n_keys + 1))
    own = owners(lws, groups)
    floor, rb, evaluated, available, gb, _ = budgets(lws, lws_out, len(groups))
    slack = rb - floor
    ready = (base_out["flags"] & R.GOUT_COND_READY) != 0
    member = own >= 0
    o = np.where(member, own, 0)
    nb = ready & member & ((np.arange(len(groups)) - gb[o]) < lws["replicas"][o].astype(np.int64))
    bound = ready & member & evaluated[o]
    keys = np.zeros(len(ids), R.DRAIN_WAVE_KEY)
    waves = []  # [ids, groups (set), lost {L: n}]
    for i, key in enumerate(int(x) for x in ids):
        gs = pairs[starts[key]:starts[key + 1], 1]
        row = keys[i]
        row["id"], row["wave"] = key, NONE
        row["groups_restarted"] = len(gs)
        row["ready_restarted"] = int(ready[gs].sum())
        row["lws_touched"] = len(np.unique(own[gs][member[gs]]))
        b = gs[bound[gs]]
        Ls, cnt = np.unique(own[b], return_counts=True)
        row["lws_breached"] = int((cnt > slack[Ls]).sum())
        if row["lws_breached"]:
            row["status"] = R.DRAINW_BREACHES_ALONE
            continue
        chosen = None
        for w, (W_ids, W_groups, W_lost) in enumerate(waves):
            new = [x for x in b.tolist() if x not in W_groups]
            Ls, cnt = np.unique(own[np.asarray(new, dtype=np.int64)], return_counts=True)
            if all(W_lost.get(int(L), 0) + int(c) <= slack[L] for L, c in zip(Ls, cnt)):
                chosen = w
                break
        if chosen is None:
            if len(waves) >= max_waves:
                row["status"] = R.DRAINW_NO_WAVE
                continue
            waves.append(([], set(), {}))
            chosen = len(waves) - 1
        W_ids, W_groups, W_lost = waves[chosen]
        for x in b.tolist():
            if x not in W_groups:
                W_lost[int(own[x])] = W_lost.get(int(own[x]), 0) + 1
        W_groups.update(gs.tolist())
        W_ids.append(key)
        row["wave"] = chosen
    out = np.zeros(len(waves), R.DRAIN_WAVE)
    for w, (W_ids, W_groups, W_lost) in enumerate(waves):
        G = np.asarray(sorted(W_groups), dtype=np.int64)
        row = out[w]
        row["n_keys"] = len(W_ids)
        row["n_pods_evicted"] = int(cost["pods"][W_ids].sum())
        row["n_leaders_evicted"] = int(cost["leaders"][W_ids].sum())
        row["n_groups_restarted"] = len(G)
        row["n_ready_restarted"] = int(ready[G].sum()) if len(G) else 0
        row["n_pods_recreated"] = int(groups["pod_count"][G].astype(np.int64).sum()) if len(G) else 0
        Gm = G[member[G]] if len(G) else G
        touched = np.unique(own[Gm])
        row["lws_touched"] = len(touched)
        row["lws_loses_available"] = len(np.unique(own[Gm[nb[Gm] & evaluated[own[Gm]] & available[own[Gm]]]]))
        margin = I32_MAX
        for L in touched[evaluated[touched]]:
            after = int(np.clip(rb[L] - W_lost.get(int(L), 0), I32_MIN, I32_MAX))
            margin = min(margin, int(np.clip(after - floor[L], I32_MIN, I32_MAX)))
        row["min_margin"] = margin
        out[w] = row
    return keys, out, _totals(keys, len(waves))


def orders(ids, cost, seed=3):
    """The key orders the tests compare: as given, reversed, by drain cost (largest min_margin first, then fewest
    groups restarted), and a seeded shuffle."""
    ids = np.asarray(ids, dtype=np.int64)
    c = cost[ids]
    by_cost = ids[np.lexsort((ids, c["groups_restarted"], -c["min_margin"].astype(np.int64)))]
    return {"given": ids, "reversed": ids[::-1].copy(), "by_cost": by_cost,
            "random": np.random.default_rng(seed).permutation(ids)}


# --------------------------------------------------------------------------- #
# the edges world
# --------------------------------------------------------------------------- #
def waves_edges_world():
    """One object per edge, each on nodes of its own (one node per domain, so both scopes name the same keys):

    - ``pair_exact`` / ``pair_over``: keys restarting exactly ``plan_threads()`` ready groups (slack equal to it)
      and one more than that (slack one below it: the last pair, in the second pass, breaches) — first in the
      given order, when the plan has one column;
    - ``below``: an object already below its floor (4 replicas, maxUnavailable 0, 3 of 4 groups ready): the key of
      a ready group breaches alone, the key of its not-ready group does not;
    - ``shared`` / ``third``: two keys restarting the same single group of an object with slack 1 (the group's
      leader on one node, its worker on the other), and a key restarting another group of it;
    - ``foreign``: a group inside one object's range naming an object with slack 0: a non-member, counted in
      the totals and never a constraint;
    - ``unevaluated``: an object with LWSE_LWS_INTSTR_INVALID and slack 0 (NOT_EVALUATED): never a constraint;
    - ``pct``: replicas 2^30 at maxUnavailable 300 %: mu passes int32, the floor is 0 in 64 bits;
    - ``cap``: 65 keys each restarting a different ready group of an object with slack 1: waves 0-63, then
      NO_WAVE at the cap;
    - ``empty``: a node with no pods.
    → (EdgeWorld, ids in the given order, notes {label: ids})."""
    from drain_edges_world import ON, Builder, node_table

    T = plan_threads()
    n_nodes = 96
    nodes, n_domains = node_table(n_nodes, 1)
    b = Builder(nodes, n_domains)
    nxt = iter(range(n_nodes))
    notes = {}
    # pair_exact: T groups, slack T; pair_over: T + 1 groups, slack T
    k_exact, k_over = next(nxt), next(nxt)
    o = b.obj(ON, size=1, replicas=T, mu=T)
    for _ in range(T):
        b.group(o, [], leader=k_exact)
    o = b.obj(ON, size=1, replicas=T + 1, mu=T)
    for _ in range(T + 1):
        b.group(o, [], leader=k_over)
    notes["pair_exact"], notes["pair_over"] = [k_exact], [k_over]
    # below: 4 replicas, mu 0, the last group not ready
    k_b0, k_b3 = next(nxt), next(nxt)
    o = b.obj(ON, size=1, replicas=4, mu=0)
    b.group(o, [], leader=k_b0)
    b.group(o, [], leader=next(nxt))
    b.group(o, [], leader=next(nxt))
    b.group(o, [], leader=k_b3, ready=False)
    notes["below"] = [k_b0, k_b3]
    # shared: slack 1 (3 replicas, mu 1), group 0 on two keys, group 1 on a third
    k_s1, k_s2, k_s3 = next(nxt), next(nxt), next(nxt)
    o = b.obj(ON, size=2, replicas=3, mu=1)
    b.group(o, [k_s2], leader=k_s1)
    b.group(o, [next(nxt)], leader=k_s3)
    b.group(o, [next(nxt)], leader=next(nxt))
    notes["shared"], notes["third"] = [k_s1, k_s2], [k_s3]
    # foreign: the host's third group names `other` (2 replicas, mu 0, slack 0)
    k_f = next(nxt)
    host = b.obj(ON, size=1, replicas=3, mu=3)
    hg = [b.group(host, [], leader=k_f if i == 2 else next(nxt)) for i in range(3)]
    other = b.obj(ON, size=1, replicas=2, mu=0)
    for _ in range(2):
        b.group(other, [], leader=next(nxt))
    notes["foreign"] = [k_f]
    # unevaluated: slack 0 but INTSTR_INVALID
    k_u = next(nxt)
    unev = b.obj(ON, size=1, replicas=2, mu=0)
    b.group(unev, [], leader=k_u)
    b.group(unev, [], leader=next(nxt))
    notes["unevaluated"] = [k_u]
    # pct: replicas 2^30, 300 %
    k_p = next(nxt)
    o = b.obj(ON, size=1, replicas=1 << 30, mu=300, pct=True)
    b.group(o, [], leader=k_p)
    b.group(o, [], leader=next(nxt))
    notes["pct"] = [k_p]
    k_empty = next(nxt)
    notes["empty"] = [k_empty]
    # cap: 65 groups, slack 1
    cap = [next(nxt) for _ in range(R.DRAIN_WAVES_MAX + 1)]
    o = b.obj(ON, size=1, replicas=len(cap), mu=1)
    for k in cap:
        b.group(o, [], leader=k)
    notes["cap"] = cap
    w = b.tables("waves_edges")
    w.groups[hg[2]]["lws_index"] = other  # inside host's range, naming `other`: a member of neither
    w.lws[unev]["flags"] |= R.LWS_INTSTR_INVALID
    w.notes = notes
    ids = [k_exact, k_over, k_b0, k_b3, k_s1, k_s2, k_s3, k_f, k_u, k_p, k_empty] + cap
    return w, ids, notes


def waves_world(n_lws=120, n_nodes=96, seed=5):
    """A variant of ``budget_world`` with slack: maxUnavailable 1-3, 50 % or 75 % and 97 % of groups ready, so that
    keys breach alone, share waves and fill several."""
    from lws_b200 import synth

    p = synth.Profile("waves", n_lws, size_choices=(2, 4), replicas_choices=(3, 4, 6, 8), n_nodes=n_nodes,
                      nodes_per_domain=4, node_capacity=4096, max_surge=((0, False), (1, False)),
                      max_unavailable=((1, False), (2, False), (3, False), (50, True), (75, True)),
                      f_mid_update=0.05, p_group_ready=0.97, p_leader_unscheduled=0.02, restart_policy_p=(0.1, 0.7, 0.2))
    return synth.make(p, seed=seed)
