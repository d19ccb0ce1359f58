"""Drain placement waves (lwse_resident_drain_place_waves) by its definition (lwse.h, "drain placement waves"),
without a GPU.  ``plan`` is the sequential first-fit where every probe S = W ∪ {k} is the set-form composition —
``drain_ref.drain_whatif_ref`` over N_S, U_S, the spec oracle's round with N_S cordoned and U_S unpinned, diffed
against the baseline — and the set form ``drain_budget_ref``:

- ``clause=None``: the literal plan, every namespace solved;
- ``clause="exact"``: only the namespaces of the set locality rule (a) / (b) solved, every other row keeping its
  baseline row — what the device computes, namespaces_solved included;
- ``clause="per_node"`` / ``"key_only"``: wrong rules (each node's free[n] tested alone; only k's own clause, as
  the per-key rule states it) that the tests show give wrong plans.

→ (keys: DRAIN_PLACE_WAVE_KEY rows in query order, waves: DRAIN_PLACE_WAVE rows, totals dict)."""
import numpy as np

from drain_budget_ref import drain_budget_cost_ref, drain_budget_ref
from drain_place_ref import drain_place_ref, key_nodes, node_free, unpinned_rows
from drain_ref import RESTART, drain_whatif_ref
from drain_waves_ref import wave_row_of_set
from lws_b200 import records as R

NONE = R.NONE
PLACE_FIELDS = ("unpinned", "stranded", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed",
                "n_unschedulable", "n_conflict", "namespaces_solved")


def set_namespaces(reqs, base_place, nodes, occ, n_domains, n_ns, by_domain, keys, drained, u, clause="exact"):
    """NS(S) by the set locality rule: (a) the namespaces of U_S; (b) those with a row that is not pinned and is
    PLACED in a domain d that S touches, where S holds d, or the row's chosen node is in N_S, or
    dom_free[d] - sum of free[n] over usable n in N_S ∩ d < size."""
    ns = reqs["ns"].astype(np.int64)
    out = {int(v) for v in ns[u] if v < n_ns}
    usable, free = node_free(nodes, occ, n_domains)
    dom = nodes["domain_id"].astype(np.int64)
    dom_free = np.bincount(dom[usable], weights=free[usable], minlength=n_domains)[:n_domains].astype(np.int64)
    in_s = np.zeros(len(nodes), bool)
    in_s[drained] = True
    touched = set(int(x) for x in dom[drained] if x < n_domains)
    drained_free = {d: int(free[in_s & usable & (dom == d)].sum()) for d in touched}
    placed = ((base_place["flags"] & R.PLACE_PLACED) != 0) & (reqs["leader_node"] == R.NONE) & (ns < n_ns)
    placed &= base_place["domain_id"].astype(np.int64) < n_domains
    last = keys[-1]
    for r in np.flatnonzero(placed):
        d, m, size = int(base_place["domain_id"][r]), int(base_place["leader_node"][r]), int(reqs["size"][r])
        if d not in touched:
            continue
        if by_domain:
            hit = True
        elif clause == "key_only":  # the per-key rule for the last key only, the rest of S's clause dropped
            hit = in_s[m] if m < len(nodes) else False
            hit = hit or (usable[last] and dom[last] == d and dom_free[d] - free[last] < size)
        elif clause == "per_node":  # each drained node's free slots tested alone
            hit = (m < len(nodes) and in_s[m]) or any(dom_free[d] - free[n] < size for n in drained
                                                      if usable[n] and dom[n] == d)
        else:
            hit = (m < len(nodes) and in_s[m]) or dom_free[d] - drained_free[d] < size
        if hit:
            out.add(int(ns[r]))
    return out


def probe(world, base_groups, base_place, keys, by_domain, clause):
    """The set-form composition over the keys: (DRAIN_PLACE_COST-like dict of PLACE_FIELDS, budget rows, totals)."""
    import oracle

    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = world
    drained = np.unique(np.concatenate([key_nodes(nodes, nd, by_domain, k) for k in keys])).astype(np.int64)
    wf = drain_whatif_ref(lws, groups, pst, pid, nodes, drained, 0, base=base_groups)
    hit = ((base_groups[1]["flags"] & RESTART) == 0) & ((wf["after_all"]["flags"] & RESTART) != 0)
    u = unpinned_rows(reqs, groups, set(np.flatnonzero(hit).tolist()), drained)
    p_nodes, p_reqs = nodes.copy(), reqs.copy()
    p_nodes["flags"][drained] &= ~np.uint16(R.NODE_SCHEDULABLE)
    p_reqs["leader_node"][u] = R.NONE
    solve = None
    if clause is not None:
        solve = set_namespaces(reqs, base_place, nodes, occ, nd, n_ns, by_domain, list(keys), drained, u, clause)
        keep = np.isin(p_reqs["ns"].astype(np.int64), np.asarray(sorted(solve), dtype=np.int64))
        p_reqs["ns"][~keep & (p_reqs["ns"] < n_ns)] = n_ns
    after = oracle.place(p_nodes, occ, nd, n_ns, p_reqs, threads=4)
    if clause is not None:
        other = ~keep & (reqs["ns"] < n_ns)
        after[other] = base_place[other]
    was, now = (base_place["flags"] & R.PLACE_PLACED) != 0, (after["flags"] & R.PLACE_PLACED) != 0
    in_u = np.zeros(len(reqs), bool)
    in_u[u] = True
    a = base_place.view(np.uint8).reshape(len(reqs), 16)
    b = after.view(np.uint8).reshape(len(reqs), 16)
    f = after["flags"]
    pl = {"unpinned": len(u), "stranded": int((in_u & ~now).sum()), "bumped": int((~in_u & was & ~now).sum()),
          "n_changed": int((a != b).any(axis=1).sum()), "n_lost": int((was & ~now).sum()),
          "n_moved": int((was & now & (base_place["domain_id"] != after["domain_id"])).sum()),
          "n_gained": int((~was & now).sum()), "n_placed": int(((f & R.PLACE_PLACED) != 0).sum()),
          "n_unschedulable": int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum()),
          "n_conflict": int(((f & R.PLACE_CONFLICT) != 0).sum()), "namespaces_solved": len(solve) if solve else 0}
    rows, tot = drain_budget_ref(lws, groups, pst, pid, nodes, drained, 0, base=base_groups)
    return pl, rows, tot


def triggers(pl, tot):
    return ((R.DPW_LWS_FLOOR if tot["n_breached"] > 0 else 0) | (R.DPW_STRANDED if pl["stranded"] else 0)
            | (R.DPW_BUMPED if pl["bumped"] else 0))


def plan(world, ids, by_domain=False, max_waves=64, constraints=R.DPW_LWS_FLOOR | R.DPW_STRANDED, clause="exact",
         base_place=None):
    import oracle

    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = world
    base_groups = oracle.sweep_lws(lws, groups, pst, pid, nodes, 0)[:2]
    if base_place is None:
        base_place = oracle.place(nodes, occ, nd, n_ns, reqs, threads=4)
    cost = drain_budget_cost_ref(lws, base_groups[0], groups, pst, pid, nodes, nd, base_groups[1], by_domain)
    alone_pl = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, by_domain, base_groups=base_groups,
                               base_place=base_place, keys=[int(k) for k in ids])
    keys = np.zeros(len(ids), R.DRAIN_PLACE_WAVE_KEY)
    waves, last = [], []  # the key lists, and each wave's last probe
    for i, k in enumerate(int(x) for x in ids):
        row = keys[i]
        row["id"], row["wave"] = k, NONE
        for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
            row[f] = cost[k][f]
        for f in ("unpinned", "stranded", "bumped"):
            row[f] = alone_pl[k][f]
        pl1, _, tot1 = probe(world, base_groups, base_place, [k], by_domain, clause)
        row["alone"] = triggers(pl1, tot1)
        if row["alone"] & constraints:
            row["status"] = R.DRAINW_BREACHES_ALONE
            continue
        for w, W in enumerate(waves):
            got = probe(world, base_groups, base_place, W + [k], by_domain, clause)
            if not triggers(got[0], got[2]) & constraints:
                W.append(k)
                last[w] = got[0]
                row["wave"] = w
                break
        else:
            if len(waves) < max_waves:
                waves.append([k])
                last.append(pl1)
                row["wave"] = len(waves) - 1
            else:
                row["status"] = R.DRAINW_NO_WAVE
    out = np.zeros(len(waves), R.DRAIN_PLACE_WAVE)
    for w, W in enumerate(waves):
        pl = last[w]
        rows, tot = drain_budget_ref(lws, groups, pst, pid, nodes,
                                     np.unique(np.concatenate([key_nodes(nodes, nd, by_domain, k) for k in W])),
                                     0, base=base_groups)
        fw = wave_row_of_set(rows, tot, len(W))
        for f in R.DRAIN_WAVE.names:
            if f != "reserved":
                out[w][f] = fw[f]
        out[w]["lws_breached"] = tot["n_breached"]
        for f in PLACE_FIELDS:
            out[w][f] = pl[f]
    st = keys["status"]
    totals = {"n_waves": len(waves), "n_planned": int((st == R.DRAINW_PLANNED).sum()),
              "n_breaches_alone": int((st == R.DRAINW_BREACHES_ALONE).sum()), "n_no_wave": int((st == R.DRAINW_NO_WAVE).sum())}
    return keys, out, totals


# --------------------------------------------------------------------------- #
# the edge worlds
# --------------------------------------------------------------------------- #
def _nodes(domains, free):
    nodes = R.aligned_empty(len(domains), R.NODE_REC)
    nodes["domain_id"] = np.asarray(domains, dtype=np.uint32)
    nodes["topo_value_hash"] = (np.asarray(domains, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(1)
    nodes["capacity"] = np.asarray(free, dtype=np.uint16)
    nodes["flags"] = R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE
    return nodes


def _world(b, nodes, nd, rows, n_ns):
    """(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns) from a Builder and request tuples
    (priority, group_key, group, ns, size, leader).  Capacities are raised by each node's pods, so ``free`` holds."""
    t = b.tables("place_waves_edges")
    occ = R.occupancy_of(t.pod_ident, len(nodes)).astype(np.uint32)
    nodes = nodes.copy()
    nodes["capacity"] = nodes["capacity"].astype(np.uint32) + occ
    reqs = R.aligned_empty(len(rows), R.PLACE_REQ)
    for i, r in enumerate(rows):
        reqs[i] = r
    return t.lws, t.groups, t.pod_state, t.pod_ident, nodes, nd, occ, reqs, n_ns


def _chosen(nodes, occ, nd, n_ns, rows, r, want, seed):
    """Re-draw row r's group_key until the round places it on node ``want`` (its domain has other nodes)."""
    import oracle

    rng = np.random.default_rng(seed)
    for _ in range(4096):
        reqs = R.aligned_empty(len(rows), R.PLACE_REQ)
        for i, x in enumerate(rows):
            reqs[i] = x
        out = oracle.place(nodes, occ, nd, n_ns, reqs, threads=1)
        if out["leader_node"][r] == want:
            return rows
        rows[r] = (rows[r][0], int(rng.integers(0, 1 << 62))) + tuple(rows[r][2:])
    raise AssertionError("no group key places the row on the node")


def sum_world():
    """Node scope, the capacity clause of rule (b) summed over a wave's nodes.  Domain 0 is nodes 0, 1, 2 with 2, 2
    and 4 free slots (dom_free 8); domain 1 is nodes 3, 4, 5 with one each; so a request of size 4 or 5 fits
    domain 0 only.  Namespace 0: ``A`` (size 4) and namespace 1: ``B`` (size 5), both on node 2.  Nodes 0 and 1
    drained together leave dom_free - (2 + 2) - size = 0 for A (kept: its namespace is not solved) and -1 for B
    (bumped, not stranded); each node alone leaves 2 and 1 (each node's clause alone, and the last key's, never
    names B's namespace).  Namespace 2: ``pinned`` on node 0 with no group (unpinned by the leader clause only,
    placed again in domain 1).  A pinned row of no namespace on node 5 (UNSCHEDULABLE once unpinned: stranded).
    An object of 2 replicas and maxUnavailable 1 with its leaders on nodes 3 and 4 (slack 1).
    → (world, ids, notes)."""
    from drain_edges_world import ON, Builder

    nodes = _nodes([0, 0, 0, 1, 1, 1], [2, 2, 4, 1, 1, 1])
    b = Builder(nodes, 2)
    o = b.obj(ON, size=1, replicas=2, mu=1)
    b.group(o, [], leader=3)
    b.group(o, [], leader=4)
    n_ns = 3
    rows = [(10, 1, NONE, 0, 4, NONE), (20, 2, NONE, 1, 5, NONE), (5, 3, NONE, 2, 1, 0), (6, 4, NONE, n_ns, 1, 5)]
    occ = np.zeros(len(nodes), np.uint32)
    rows = _chosen(nodes, occ, 2, n_ns, rows, 0, 2, 1)
    rows = _chosen(nodes, occ, 2, n_ns, rows, 1, 2, 2)
    return _world(b, nodes, 2, rows, n_ns), [0, 1, 2, 3, 4, 5], {"A": 0, "B": 1, "pinned": 2, "no_ns": 3}


def strand_world():
    """Domain scope, one node per domain.  Namespace 0 has ``P1`` and ``P2`` (size 4) pinned on domains 1 and 2
    and one spare domain that fits them (3; its pinned rows on 4 and 7, never drained, hold the others): each
    domain drained alone moves its row to 3, both together strand one, so the second opens a new wave.
    Namespace 1: ``P3`` (size 9, first in key order) pinned on domain 5 and ``H`` (size 5) pinned on domain 4 —
    the only domain that fits P3 — by a group whose worker runs on domain 6; domain 7 fits H only.  Domain 5
    alone strands P3 (H holds 4).  Domain 6 restarts H's group and unpins H without cordoning 4, and with 5 added
    P3 takes 4 and H takes 7: {6, 5} strands nothing, yet 5 is BREACHES_ALONE.  → (world, ids, notes)."""
    from drain_edges_world import ON, Builder

    nodes = _nodes(range(8), [1, 4, 4, 4, 10, 1, 1, 6])
    b = Builder(nodes, 8)
    o = b.obj(ON, size=2, replicas=1, mu=1)
    g = b.group(o, [6], leader=4)
    rows = [(100, 1, NONE, 0, 4, 1), (101, 2, NONE, 0, 4, 2), (1, 3, NONE, 1, 9, 5), (50, 4, g, 1, 5, 4),
            (102, 5, NONE, 0, 1, 4), (103, 6, NONE, 0, 1, 7)]
    return _world(b, nodes, 8, rows, 2), [1, 2, 6, 5], {"P1": 0, "P2": 1, "P3": 2, "H": 3}


def cap_world():
    """65 node keys (one node per domain) each restarting one ready group of an object of slack 1, and a request
    per namespace on every node: LWS floor fills waves 0-63, then NO_WAVE.  → (world, ids, notes)."""
    from drain_edges_world import ON, Builder

    n = R.DRAIN_WAVES_MAX + 1
    nodes = _nodes(range(n + 1), [4] * (n + 1))
    b = Builder(nodes, n + 1)
    o = b.obj(ON, size=1, replicas=n, mu=1)
    for k in range(n):
        b.group(o, [], leader=k)
    rows = [(7, 9, NONE, 0, 2, NONE)]
    return _world(b, nodes, n + 1, rows, 1), list(range(n)), {}


EDGE_WORLDS = {"sum": sum_world, "strand": strand_world, "cap": cap_world}
