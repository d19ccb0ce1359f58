"""The drain placement (lwse_resident_drain_place_cost) by its definition (lwse.h, "drain placement"), without a
GPU:

- ``drain_place_ref``: per key, the set-form composition — the drain what-if of the key's nodes
  (``drain_ref.drain_whatif_ref``), U_k from its restarted groups and the leaders on the key, then the spec
  oracle's round over the cordoned node rows and the unpinned request rows, diffed against the baseline;
- ``pruned=True``: the same rows when only the namespaces of the locality rule (a) / (b) are solved and every
  other row keeps its baseline row — what the device computes."""
import numpy as np

from drain_budget_ref import key_of
from drain_ref import RESTART, drain_whatif_ref
from lws_b200 import records as R


def key_nodes(nodes, n_domains, by_domain, k):
    """N_k: the node row k, or every node row whose domain_id is k."""
    if not by_domain:
        return np.array([k], dtype=np.int64)
    d = nodes["domain_id"].astype(np.int64)
    return np.flatnonzero((d < n_domains) & (d == k))


def node_free(nodes, occ, n_domains):
    """(usable, free slots) per node row, as the placement round's node index sees them."""
    f = nodes["flags"].astype(np.int64)
    usable = ((f & R.NODE_SCHEDULABLE) != 0) & ((f & R.NODE_HAS_TOPOLOGY) != 0) & (nodes["domain_id"].astype(np.int64) < n_domains)
    cap, o = nodes["capacity"].astype(np.int64), np.asarray(occ, dtype=np.int64)
    return usable, np.where(usable, np.maximum(cap - o, 0), 0)


def unpinned_rows(reqs, groups, restarted, drained):
    """U_k: pinned request rows whose leader node is drained or whose group row is restarted."""
    leader = reqs["leader_node"].astype(np.int64)
    g = reqs["group"].astype(np.int64)
    pinned = leader != R.NONE
    in_group = (g < len(groups)) & np.isin(g, np.asarray(sorted(restarted), dtype=np.int64))
    return np.flatnonzero(pinned & (np.isin(leader, drained) | in_group))


def solved_namespaces(reqs, base_place, nodes, occ, n_domains, n_ns, by_domain, k, drained, u, capacity_clause="exact"):
    """The namespaces the locality rule solves for key k.  ``capacity_clause`` "dropped" / "tight" (the node clause
    left out, or ``< size - 1``) are wrong rules the tests show to be caught."""
    ns = reqs["ns"].astype(np.int64)
    out = {int(v) for v in ns[u] if v < n_ns}
    usable, free = node_free(nodes, occ, n_domains)
    dom = nodes["domain_id"].astype(np.int64)
    dom_free = np.bincount(dom[usable], weights=free[usable], minlength=n_domains)[:n_domains].astype(np.int64)
    placed = ((base_place["flags"] & R.PLACE_PLACED) != 0) & (reqs["leader_node"] == R.NONE) & (ns < n_ns)
    placed &= base_place["domain_id"].astype(np.int64) < n_domains
    for r in np.flatnonzero(placed):
        d, m, size = int(base_place["domain_id"][r]), int(base_place["leader_node"][r]), int(reqs["size"][r])
        if by_domain:
            hit = d == k
        else:
            slack = {"exact": 0, "tight": 1, "dropped": None}[capacity_clause]
            hit = m == k or (slack is not None and usable[k] and dom[k] == d and dom_free[d] - free[k] < size - slack)
        if hit:
            out.add(int(ns[r]))
    return out


def drain_place_ref(lws, groups, pst, pid, nodes, n_domains, occ, reqs, n_ns, by_domain=False, flags=0,
                    base_groups=None, base_place=None, pruned=False, keys=None, threads=4, capacity_clause="exact"):
    """DRAIN_PLACE_COST rows for ``keys`` (default every key).  ``base_groups``: the oracle's (lws_out, group_out);
    ``base_place``: the oracle's placement rows of the tables as they are."""
    import oracle

    if base_groups is None:
        base_groups = oracle.sweep_lws(lws, groups, pst, pid, nodes, flags)[:2]
    if base_place is None:
        base_place = oracle.place(nodes, occ, n_domains, n_ns, reqs, threads=threads)
    n_keys = n_domains if by_domain else len(nodes)
    keys = range(n_keys) if keys is None else keys
    out = np.zeros(n_keys, R.DRAIN_PLACE_COST)
    was = (base_place["flags"] & R.PLACE_PLACED) != 0
    for k in keys:
        drained = key_nodes(nodes, n_domains, by_domain, k)
        wf = drain_whatif_ref(lws, groups, pst, pid, nodes, drained, flags, base=base_groups)
        hit = ((base_groups[1]["flags"] & RESTART) == 0) & ((wf["after_all"]["flags"] & RESTART) != 0)
        u = unpinned_rows(reqs, groups, set(np.flatnonzero(hit).tolist()), drained)
        p_nodes, p_reqs = nodes.copy(), reqs.copy()
        p_nodes["flags"][drained] &= ~np.uint16(R.NODE_SCHEDULABLE)
        p_reqs["leader_node"][u] = R.NONE
        solve = None
        if pruned:
            solve = solved_namespaces(reqs, base_place, nodes, occ, n_domains, n_ns, by_domain, k, drained, u,
                                      capacity_clause)
            keep = np.isin(p_reqs["ns"].astype(np.int64), np.asarray(sorted(solve), dtype=np.int64))
            p_reqs["ns"][~keep & (p_reqs["ns"] < n_ns)] = n_ns  # (out of the round: the baseline row stays)
        after = oracle.place(p_nodes, occ, n_domains, n_ns, p_reqs, threads=threads)
        if pruned:
            other = ~keep & (reqs["ns"] < n_ns)
            after[other] = base_place[other]
        a = base_place.view(np.uint8).reshape(len(reqs), 16)
        b = after.view(np.uint8).reshape(len(reqs), 16)
        now = (after["flags"] & R.PLACE_PLACED) != 0
        in_u = np.zeros(len(reqs), bool)
        in_u[u] = True
        f = after["flags"]
        row = out[k]
        row["groups_restarted"] = int(hit.sum())
        row["unpinned"] = len(u)
        row["stranded"] = int((in_u & ~now).sum())
        row["bumped"] = int((~in_u & was & ~now).sum())
        row["n_changed"] = int((a != b).any(axis=1).sum())
        row["n_lost"] = int((was & ~now).sum())
        row["n_moved"] = int((was & now & (base_place["domain_id"] != after["domain_id"])).sum())
        row["n_gained"] = int((~was & now).sum())
        row["n_placed"] = int(((f & R.PLACE_PLACED) != 0).sum())
        row["n_unschedulable"] = int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum())
        row["n_conflict"] = int(((f & R.PLACE_CONFLICT) != 0).sum())
        row["namespaces_solved"] = len(solve) if pruned else 0
        out[k] = row
    return out


def composition_ref(enc, by_domain, keys=None, flags=0, threads=4):
    """Per key, the informer's own composition: ``drain_place_query`` (with the oracle's drain what-if of the key's
    nodes) and ``test_place_whatif.whatif_ref`` over its segments → DRAIN_PLACE_COST rows (namespaces_solved 0)."""
    import oracle
    from test_place_whatif import whatif_ref

    lws, groups, pst, pid, reqs = enc.full_tables()
    nodes, nd = enc.node_rec, enc.n_domains
    occ = R.occupancy_of(pid, len(nodes))
    base = oracle.sweep_lws(lws, groups, pst, pid, nodes, flags)[:2]
    names = {row: name for name, row in enc.node_index.items()}
    n_keys = nd if by_domain else len(nodes)
    out = np.zeros(n_keys, R.DRAIN_PLACE_COST)
    for k in (range(n_keys) if keys is None else keys):
        drained = key_nodes(nodes, nd, by_domain, k)
        node_names = [names[int(n)] for n in drained if int(n) in names]
        if not node_names:
            continue
        wf = drain_whatif_ref(lws, groups, pst, pid, nodes, drained, flags, base=base)
        segs = enc.drain_place_query(wf, node_names)
        ref = whatif_ref(nodes, occ, nd, reqs, segs, n_ns=enc.n_namespaces, threads=threads)
        u = segs[1][1][reqs["leader_node"][segs[1][1]] != R.NONE]
        before = oracle.place(nodes, occ, nd, enc.n_namespaces, reqs, threads=threads)
        after = ref["after_all"]
        now = (after["flags"] & R.PLACE_PLACED) != 0
        was = (before["flags"] & R.PLACE_PLACED) != 0
        in_u = np.zeros(len(reqs), bool)
        in_u[u] = True
        row = out[k]
        row["groups_restarted"] = wf["n_groups_restarted"]
        row["unpinned"] = len(u)
        row["stranded"] = int((in_u & ~now).sum())
        row["bumped"] = int((~in_u & was & ~now).sum())
        for f in ("n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict"):
            row[f] = ref[f]
        out[k] = row
    return out
