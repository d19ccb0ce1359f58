"""The drain what-if and the drain cost by their definitions (lwse.h, "drain what-if"), without a GPU:

- ``drain_whatif_ref``: the spec oracle's sweep of the tables with the pods of the drained nodes deleting,
  diffed against the oracle's sweep of the tables as they are;
- ``restart_pairs`` / ``drain_cost_ref``: a numpy restatement of the one-pass argument — the (group, node)
  pairs through which draining the node restarts the group — and the per-node totals it gives;
- ``special_tables``: a small table built to reach every branch of the restart verdict."""
import numpy as np

from lws_b200 import records as R

RESTART = R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING
CHAIN = R.GRP_WSTS_FOUND | R.GRP_WSTS_OWNER_IS_POD | R.GRP_WSTS_OWNER_NAME_MATCH
TOTALS = ("n_pods_evicted", "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted", "n_pods_recreated")
COST_OF = dict(zip(TOTALS, ("pods", "leaders", "groups_restarted", "ready_restarted", "pods_recreated")))


def drain_tables(groups, pod_state, pod_ident, drain):
    """Copies of the group rows and the state column with the what-if's two changes for node rows ``drain``
    → (groups, pod_state, pods evicted, leaders evicted)."""
    d = np.asarray(list(drain), dtype=np.int64)
    place = pod_ident["place"]
    evict = ((place & R.PODID_SCHEDULED) != 0) & np.isin((place >> R.PODID_NODE_SHIFT).astype(np.int64), d)
    pst = pod_state.copy()
    pst[evict] |= np.uint8(R.POD_DELETING)
    g = groups.copy()
    lead = np.isin(g["leader_node"].astype(np.int64), d)
    g["flags"][lead] |= np.uint32(R.GRP_POD_DELETING)
    return g, pst, int(evict.sum()), int(lead.sum())


def drain_whatif_ref(lws, groups, pod_state, pod_ident, nodes, drain, flags=0, base=None):
    """The what-if by its definition.  ``base``: the oracle's (lws_out, group_out) of the tables as they are."""
    import oracle

    if base is None:
        base = oracle.sweep_lws(lws, groups, pod_state, pod_ident, nodes, flags)[:2]
    g, pst, n_pods, n_leaders = drain_tables(groups, pod_state, pod_ident, drain)
    lws_out, after, _ = oracle.sweep_lws(lws, g, pst, pod_ident, nodes, flags)
    before = base[1]
    a = before.view(np.uint8).reshape(len(before), 16)
    b = after.view(np.uint8).reshape(len(after), 16)
    rows = np.flatnonzero((a != b).any(axis=1)).astype(np.uint32)
    hit = ((before["flags"] & RESTART) == 0) & ((after["flags"] & RESTART) != 0)
    return {
        "rows": rows, "before": before[rows], "after": after[rows], "after_all": after, "lws_out": lws_out,
        "n_changed": len(rows), "n_pods_evicted": n_pods, "n_leaders_evicted": n_leaders,
        "n_groups_restarted": int(hit.sum()),
        "n_ready_restarted": int((hit & ((before["flags"] & R.GOUT_COND_READY) != 0)).sum()),
        "n_pods_recreated": int(groups["pod_count"][hit].astype(np.int64).sum()),
    }


def restart_pairs(lws, groups, pod_state, pod_ident, n_nodes, base_out):
    """(group rows, node rows): every distinct pair where draining the node restarts the group — a group whose
    baseline row has no restart bit, whose policy and pending gate let its pods be visited, and one of whose
    pods, scheduled on the node, passes the per-pod verdict with its deleting bit set."""
    n_pods, n_lws = len(pod_state), len(lws)
    li = groups["lws_index"].astype(np.int64)
    pb = groups["pod_base"].astype(np.int64)
    pc = groups["pod_count"].astype(np.int64)
    ok = (li < n_lws) & (pb + pc <= n_pods) & (pc > 0) & ((base_out["flags"] & RESTART) == 0)
    L = lws[np.where(ok, li, 0)] if n_lws else np.zeros(len(groups), R.LWS_REC)
    lflags = L["flags"].astype(np.int64)
    policy = (lflags & R.LWS_RESTART_MASK) >> R.LWS_RESTART_SHIFT
    cs = np.concatenate([[0], np.cumsum((pod_state & R.POD_PHASE_MASK) == R.POD_PHASE_PENDING)])
    any_pending = np.where(ok, cs[np.clip(pb + pc, 0, n_pods)] - cs[np.clip(pb, 0, n_pods)], 0) > 0
    pending = (L["size"].astype(np.int64) != pc) | any_pending
    suppressed = pending & ((policy == R.RESTART_AFTER_START) | ((lflags & R.LWS_RECREATE_AFTER_START_ANNOT) != 0))
    gate = ok & ((policy == R.RESTART_ON_POD_RESTART) | (policy == R.RESTART_AFTER_START)) & ~suppressed
    gi = np.repeat(np.flatnonzero(gate), pc[gate])
    if len(gi) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    start = np.repeat(np.cumsum(pc[gate]) - pc[gate], pc[gate])
    p = pb[gi] + (np.arange(len(gi)) - start)
    st = pod_state[p].astype(np.int64) | R.POD_DELETING
    ident = pod_ident[p]
    place = ident["place"].astype(np.int64)
    node = place >> R.PODID_NODE_SHIFT
    g = groups[gi]
    gflags = g["flags"].astype(np.int64)
    found = (gflags & (R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH)) == (R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH)
    chain = ((gflags & CHAIN) == CHAIN) & (g["wsts_owner_uid_hash"] == g["leader_uid_hash"])
    kind = (st & R.POD_OWNER_MASK) >> R.POD_OWNER_SHIFT
    owner = ident["owner_uid_hash"]
    belongs = ((st & R.POD_OWNER_NAME_MATCH) != 0) & (
        ((kind == R.POD_OWNER_POD) & (owner == g["leader_uid_hash"]))
        | ((kind == R.POD_OWNER_STS) & (owner == g["wsts_uid_hash"]) & chain))
    worker = ((place & R.PODID_NAME_OK) != 0) & found & (ident["rev_hash"] == g["leader_rev_hash"]) & belongs
    cand = ((st & R.POD_IS_LEADER) != 0) | worker
    on = cand & ((place & R.PODID_SCHEDULED) != 0) & (node < n_nodes)
    pairs = np.unique(np.stack([gi[on], node[on]], axis=1), axis=0)
    return pairs[:, 0], pairs[:, 1]


def drain_cost_ref(lws, groups, pod_state, pod_ident, n_nodes, base_out):
    """One DRAIN_COST row per node: the totals of the what-if of that node alone, from ``restart_pairs``."""
    cost = np.zeros(n_nodes, R.DRAIN_COST)
    place = pod_ident["place"].astype(np.int64)
    node = place >> R.PODID_NODE_SHIFT
    on = ((place & R.PODID_SCHEDULED) != 0) & (node < n_nodes)
    cost["pods"] = np.bincount(node[on], minlength=n_nodes)[:n_nodes]
    ln = groups["leader_node"].astype(np.int64)
    cost["leaders"] = np.bincount(ln[ln < n_nodes], minlength=n_nodes)[:n_nodes]
    g, n = restart_pairs(lws, groups, pod_state, pod_ident, n_nodes, base_out)
    ready = (base_out["flags"][g] & R.GOUT_COND_READY) != 0
    cost["groups_restarted"] = np.bincount(n, minlength=n_nodes)[:n_nodes]
    cost["ready_restarted"] = np.bincount(n[ready], minlength=n_nodes)[:n_nodes]
    rec = np.zeros(n_nodes, np.uint64)
    np.add.at(rec, n, groups["pod_count"][g].astype(np.uint64))
    cost["pods_recreated"] = rec
    return cost


def set_totals_ref(lws, groups, pod_state, pod_ident, n_nodes, base_out, drain):
    """The restart totals of a what-if over the node set ``drain``, from ``restart_pairs``: a group restarts
    when any of its pairs names a drained node."""
    g, n = restart_pairs(lws, groups, pod_state, pod_ident, n_nodes, base_out)
    hit = np.unique(g[np.isin(n, np.asarray(list(drain), dtype=np.int64))])
    return {"n_groups_restarted": len(hit),
            "n_ready_restarted": int(((base_out["flags"][hit] & R.GOUT_COND_READY) != 0).sum()),
            "n_pods_recreated": int(groups["pod_count"][hit].astype(np.int64).sum())}


def _ident(rev, owner, node=None, name_ok=True):
    place = (R.PODID_NAME_OK if name_ok else 0)
    if node is not None:
        place |= R.PODID_SCHEDULED | (node << R.PODID_NODE_SHIFT)
    return (rev, owner, place)


def special_tables(n_nodes=8):
    """(lws, groups, pod_state, pod_ident, nodes): one group per case of the restart verdict.  Every group has
    the leader pod first (owner = the set) and workers owned by its worker StatefulSet; running unless said."""
    REV, OTHER = 0x1111, 0x2222
    RUN, PEND = R.POD_PHASE_RUNNING, R.POD_PHASE_PENDING
    lws_rows, groups, pods = [], [], []

    def obj(policy, size, annot=False):
        lws_rows.append((policy, size, annot))
        return len(lws_rows) - 1

    def group(o, workers, leader=0, leader_node=None, gflags=None, chain_ok=True, restarting=False, pod_count=None):
        """workers: [(node, phase, extra state bits, name_ok, owner ok)]; leader: node of the leader pod."""
        gi = len(groups)
        luid, wuid = 1000 + gi, 2000 + gi
        base = len(pods)
        lstate = RUN | R.POD_IS_LEADER | (R.POD_OWNER_STS << R.POD_OWNER_SHIFT)
        if restarting:
            lstate |= R.POD_ANY_RESTART
        pods.append((lstate, _ident(REV, 9, leader)))
        for node, phase, extra, name_ok, owner_ok in workers:
            st = phase | extra | (R.POD_OWNER_STS << R.POD_OWNER_SHIFT) | R.POD_OWNER_NAME_MATCH
            pods.append((st, _ident(REV, wuid if owner_ok else 77, node, name_ok)))
        f = (R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH | R.GRP_POD_RUNNING | R.GRP_POD_READY | R.GRP_WSTS_LABEL_NAME_MATCH
             | R.GRP_WSTS_FOUND | R.GRP_WSTS_REV_SETTLED | R.GRP_WSTS_OWNER_IS_POD | R.GRP_WSTS_OWNER_NAME_MATCH
             | R.GRP_REVISION_EXISTS) if gflags is None else gflags
        ln = leader if leader_node is None else leader_node
        groups.append(dict(o=o, luid=luid, wuid=wuid, owner=luid if chain_ok else 5, node=R.NONE if ln is None else ln,
                           base=base, count=len(pods) - base if pod_count is None else pod_count, flags=f,
                           workers=len(workers)))

    on, after, none = R.RESTART_ON_POD_RESTART, R.RESTART_AFTER_START, R.RESTART_NONE
    w = lambda node, phase=RUN, extra=0, name_ok=True, owner_ok=True: (node, phase, extra, name_ok, owner_ok)
    o_on3, o_after3, o_annot3, o_none3 = obj(on, 3), obj(after, 3), obj(on, 3, annot=True), obj(none, 3)
    o_on5 = obj(on, 5)
    group(o_on3, [w(1), w(2)], leader=0)                    # spread over three nodes
    group(o_on3, [w(3), w(3)], leader=4)                    # two pods of the group on one node
    group(o_on3, [w(5), w(5)], leader=5)                    # leader and workers on one node
    group(o_on3, [w(None), w(None)], leader=6)              # leader on the node, no workers there
    group(o_none3, [w(1), w(2)], leader=0)                  # policy None
    group(o_after3, [w(1), w(2)], leader=0)                 # AfterStart, gate open
    group(o_after3, [w(1, PEND), w(2)], leader=0)           # AfterStart, a pending pod closes the gate
    group(o_annot3, [w(1), w(2, PEND)], leader=0)           # annotation, gate closed
    group(o_annot3, [w(1), w(2)], leader=0)                 # annotation, gate open
    group(o_on5, [w(1), w(2)], leader=0)                    # size != pod count: pending, open for OnPodRestart
    group(o_after3, [w(7), w(7), w(1)], leader=0, pod_count=3)  # AfterStart, open; its last worker is in no range
    group(o_on3, [w(1), w(2)], leader=0, restarting=True)   # already restarting
    group(o_on3, [w(1, name_ok=False), w(2)], leader=3)     # worker name fails to parse: RESTART_ERROR
    group(o_on3, [w(1), w(2)], leader=3, chain_ok=False)    # stale owner chain: workers do not belong
    group(o_on3, [w(1, owner_ok=False), w(2)], leader=3)    # a worker owned by another set
    group(o_on3, [w(1), w(2)], leader=None, leader_node=R.NODE_NOT_FOUND)  # leader unscheduled, Node missing
    group(o_on3, [w(1), w(2)], leader=None, leader_node=R.NONE)            # leader unscheduled
    group(o_on3, [w(4), w(4)], leader=2, gflags=R.GRP_POD_PRESENT)         # leader not found by name
    group(o_on3, [w(6), w(6)], leader=6, gflags=R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH | R.GRP_POD_DELETING)
    n_good = len(groups)
    pods.append((RUN, _ident(REV, 1, 2)))                   # scheduled pod rows no group references
    pods.append((RUN, _ident(REV, 1, 3)))
    pods.append((RUN, _ident(REV, 1, None)))                # unscheduled

    P = len(pods)
    lws = R.aligned_empty(len(lws_rows), R.LWS_REC)
    for i, (policy, size, annot) in enumerate(lws_rows):
        lws[i]["rev_hash"] = REV
        lws[i]["size"] = size
        lws[i]["replicas"] = lws[i]["sts_replicas"] = lws[i]["sts_replicas_annotation"] = 4
        lws[i]["flags"] = (R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID | (policy << R.LWS_RESTART_SHIFT)
                           | (R.LWS_RECREATE_AFTER_START_ANNOT if annot else 0))
    g = R.aligned_empty(n_good + 2, R.GROUP_REC)
    for i, d in enumerate(groups):
        g[i]["leader_rev_hash"] = g[i]["wsts_rev_hash"] = REV
        g[i]["wsts_spec_replicas"] = g[i]["wsts_avail_replicas"] = 2
        g[i]["leader_uid_hash"], g[i]["wsts_uid_hash"], g[i]["wsts_owner_uid_hash"] = d["luid"], d["wuid"], d["owner"]
        g[i]["leader_node"], g[i]["pod_base"], g[i]["pod_count"] = d["node"], d["base"], d["count"]
        g[i]["lws_index"], g[i]["flags"] = d["o"], d["flags"]
    # BAD_TABLE rows: an owner beyond the LWS table, a pod range beyond the pod columns (leaders on node 1)
    g[n_good]["lws_index"], g[n_good]["leader_node"], g[n_good]["pod_count"] = len(lws) + 3, 1, 2
    g[n_good + 1]["lws_index"], g[n_good + 1]["leader_node"] = 0, 1
    g[n_good + 1]["pod_base"], g[n_good + 1]["pod_count"] = P - 1, 5
    pst = R.aligned_empty(P, R.POD_STATE)
    pst[:] = [s for s, _ in pods]
    pid = R.pod_ident_table(np.array([i[0] for _, i in pods], np.uint64), np.array([i[1] for _, i in pods], np.uint32),
                            np.array([i[2] for _, i in pods], np.uint32))
    nodes = R.aligned_empty(n_nodes, R.NODE_REC)
    nodes["flags"] = R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE
    nodes["capacity"] = 16
    nodes["domain_id"] = np.arange(n_nodes) // 2
    return lws, g, pst, pid, nodes
