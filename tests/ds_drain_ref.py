"""The DS drain by its definition (lwse.h, "DS drain"), without a GPU:

- ``lost_ref``: lost(L, D) of the drain budget — the spec oracle's what-if for the drained node rows, its restarted
  ready groups gathered per LWS row (as ``drain_budget_ref``);
- ``link_targets``: the LWS row each revision-role row takes its ready count from (the rule of
  ``ds_link_world.linked_revroles``), or -1;
- ``ds_drain_ref``: the set form — the before and the after linked sweep through ``oracle.sweep_ds`` and the
  verdicts of every touched DS;
- ``ds_drain_cost_ref``: the per-key form restated from (row, key) facts, as the device computes it;
- ``ds_drain_world``: child LeaderWorkerSets of 2-8 pod groups bound to nodes in several domains, and C4-style DS
  tables linked to them, with ready, stable, rolling and BAD_TABLE DS and every fall-back cause."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from drain_budget_ref import domain_nodes, key_of, owners
from drain_ref import RESTART, drain_whatif_ref, restart_pairs
from ds_link_world import LOUT_NO_UPDATE, none_links
from lws_b200 import records as R

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
COST_FIELDS = ("ds_touched", "ds_service_lost", "ds_old_service_lost", "ds_stalled", "rows_touched", "rows_zeroed")
TOTALS = R.DS_DRAIN_TOTALS


@dataclass
class World:
    lws: np.ndarray
    groups: np.ndarray
    pod_state: np.ndarray
    pod_ident: np.ndarray
    nodes: np.ndarray
    n_domains: int
    flags: int
    ds: np.ndarray
    roles: np.ndarray
    revroles: np.ndarray
    links: np.ndarray
    base: tuple = None  # the oracle's (lws_out, group_out)

    @property
    def sweep_flags(self):
        return self.flags & R.SWEEP_GANG


def lost_ref(w: World, drain) -> np.ndarray:
    """lost(L, D) for every LWS row: restarted groups of L whose baseline row is COND_READY."""
    lws_out, before = w.base
    wf = drain_whatif_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, drain, w.sweep_flags, base=w.base)
    hit = ((before["flags"] & RESTART) == 0) & ((wf["after_all"]["flags"] & RESTART) != 0)
    own = owners(w.lws, w.groups)
    sel = hit & (own >= 0) & ((before["flags"] & R.GOUT_COND_READY) != 0)
    return np.bincount(own[sel], minlength=len(w.lws))[: len(w.lws)].astype(np.int64)


def link_targets(revroles, links, lws, lws_out) -> np.ndarray:
    """Per revision-role row: the LWS row whose ready count it takes, or -1 (it falls back)."""
    L = links["lws_row"].astype(np.int64)
    ok = (L != R.NONE) & ((revroles["flags"] & R.RR_EXISTS) != 0) & (L < len(lws))
    at = np.where(ok, L, 0)
    if len(lws):
        ok &= lws["uid_hash"][at] == links["lws_uid_hash"]
        ok &= (lws_out["flags"][at] & LOUT_NO_UPDATE) == 0
    return np.where(ok, L, -1)


def ds_ok(ds, n_roles_table, n_revroles_table) -> np.ndarray:
    """Per DS: its table checks pass (not BAD_TABLE)."""
    n, S, V = ds["n_roles"].astype(np.int64), ds["n_spec_roles"].astype(np.int64), ds["n_old_revs"].astype(np.int64)
    return ((n <= R.DS_MAX_ROLES) & (S <= n) & (V <= R.DS_MAX_OLD_REVS)
            & (ds["role_base"].astype(np.int64) + n <= n_roles_table)
            & (ds["rev_base"].astype(np.int64) + (V + 1) * n <= n_revroles_table))


def read_rows(ds, n_roles_table, n_revroles_table):
    """(DS row, revision slot, role, spec) of every revision-role row the sweep reads, by row: -1 elsewhere."""
    nrr = n_revroles_table
    owner, slot, role, spec = (np.full(nrr, -1, np.int64) for _ in range(4))
    for d in np.flatnonzero(ds_ok(ds, n_roles_table, n_revroles_table)):
        n, V, S, vb = int(ds["n_roles"][d]), int(ds["n_old_revs"][d]), int(ds["n_spec_roles"][d]), int(ds["rev_base"][d])
        k = np.arange((V + 1) * n)
        owner[vb + k], slot[vb + k], role[vb + k], spec[vb + k] = d, k // n, k % n, (k % n) < S
    return owner, slot, role, spec


def _sweep(w: World, ready):
    import oracle

    rr = w.revroles.copy()
    rr["ready_replicas"] = ready
    ds_out, role_out, revrole_out = oracle.sweep_ds(w.ds, w.roles, rr)
    # rows no DS's sweep writes read 0
    ok = ds_ok(w.ds, len(w.roles), len(w.revroles))
    rmask = np.zeros(len(w.roles), bool)
    for d in np.flatnonzero(ok):
        rmask[int(w.ds["role_base"][d]): int(w.ds["role_base"][d]) + int(w.ds["n_roles"][d])] = True
    role_out[~rmask] = 0
    revrole_out[read_rows(w.ds, len(w.roles), len(w.revroles))[0] < 0] = 0
    return ds_out, role_out, revrole_out


def ready_columns(w: World, lost):
    """(targets, ready_before, ready_after) per revision-role row."""
    lws_out = w.base[0]
    L = link_targets(w.revroles, w.links, w.lws, lws_out)
    before = np.where(L >= 0, lws_out["ready_replicas"][np.maximum(L, 0)].astype(np.int64),
                      w.revroles["ready_replicas"].astype(np.int64))
    after = np.where(L >= 0, np.clip(before - lost[np.maximum(L, 0)], I32_MIN, I32_MAX), before)
    return L, before, after


def ds_drain_ref(w: World, drain):
    """The set form for node rows ``drain``: rows (DS_DRAIN, sorted by DS row), totals, and the after sweep's
    (role_out, revrole_out)."""
    lost = lost_ref(w, drain)
    L, rb, ra = ready_columns(w, lost)
    b = _sweep(w, rb)
    a = _sweep(w, ra)
    owner, slot, role, spec = read_rows(w.ds, len(w.roles), len(w.revroles))
    take = (L >= 0) & (owner >= 0)
    lost_r = np.where(take, lost[np.maximum(L, 0)], 0)
    touched_r = take & (lost_r > 0)
    zeroed_r = touched_r & (rb >= 1) & (ra < 1)
    n_ds = len(w.ds)
    rows_touched = np.bincount(owner[touched_r], minlength=n_ds)[:n_ds]
    rows_zeroed = np.bincount(owner[zeroed_r], minlength=n_ds)[:n_ds]
    # the zeroed spec roles: of the new revision, and of the old revisions whose ready bit falls
    fell = b[0]["ready_revs"].astype(np.int64) & ~a[0]["ready_revs"].astype(np.int64)
    new_z, old_z = np.zeros(n_ds, np.int64), np.zeros(n_ds, np.int64)
    for r in np.flatnonzero(zeroed_r & (spec == 1)):
        d, v = int(owner[r]), int(slot[r])
        if v == int(w.ds["n_old_revs"][d]):
            new_z[d] |= 1 << int(role[r])
        elif (fell[d] >> v) & 1:
            old_z[d] |= 1 << int(role[r])
    out = []
    for d in np.flatnonzero(rows_touched > 0):
        bo, ao = b[0][d], a[0][d]
        fl = R.DSD_TOUCHED
        if bo["flags"] & R.DOUT_NEW_READY and not ao["flags"] & R.DOUT_NEW_READY:
            fl |= R.DSD_SERVICE_LOST
        if int(bo["ready_revs"]) & ~int(ao["ready_revs"]):
            fl |= R.DSD_OLD_SERVICE_LOST
        if bo["flags"] & R.DOUT_STABLE and not ao["flags"] & R.DOUT_STABLE:
            fl |= R.DSD_STALLS
        changed = bo.tobytes() != ao.tobytes()
        if not bo["flags"] & R.DOUT_BAD_TABLE:
            rbase, n = int(w.ds["role_base"][d]), int(w.ds["n_roles"][d])
            vb, nrr = int(w.ds["rev_base"][d]), (int(w.ds["n_old_revs"][d]) + 1) * n
            changed |= b[1][rbase: rbase + n].tobytes() != a[1][rbase: rbase + n].tobytes()
            changed |= b[2][vb: vb + nrr].tobytes() != a[2][vb: vb + nrr].tobytes()
        if changed:
            fl |= R.DSD_CHANGED
        out.append((d, fl, rows_touched[d], rows_zeroed[d], new_z[d], old_z[d], (0, 0), tuple(bo), tuple(ao)))
    rows = np.array(out, dtype=R.DS_DRAIN) if out else np.zeros(0, R.DS_DRAIN)
    f = rows["flags"]
    totals = {"n_touched": len(rows), "n_service_lost": int(((f & R.DSD_SERVICE_LOST) != 0).sum()),
              "n_old_service_lost": int(((f & R.DSD_OLD_SERVICE_LOST) != 0).sum()),
              "n_stalled": int(((f & R.DSD_STALLS) != 0).sum()), "n_changed": int(((f & R.DSD_CHANGED) != 0).sum()),
              "rows_touched": int(rows_touched.sum()), "rows_zeroed": int(rows_zeroed.sum()),
              "rows_linked": int(take.sum())}
    return rows, totals, a[1], a[2]


def ds_drain_domains_ref(w: World, domains):
    return ds_drain_ref(w, domain_nodes(w.nodes, w.n_domains, domains))


def lost_pairs(w: World, by_domain):
    """{(L, key): lost(L, key)} over the keys whose drain restarts a ready group of L."""
    lws_out, base_out = w.base
    key = key_of(w.nodes, w.n_domains, by_domain)
    g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base_out)
    k = key[n]
    keep = k >= 0
    if not keep.any():
        return {}
    pairs = np.unique(np.stack([g[keep], k[keep]], axis=1), axis=0)
    own = owners(w.lws, w.groups)
    g, k = pairs[:, 0], pairs[:, 1]
    m = (own[g] >= 0) & ((base_out["flags"][g] & R.GOUT_COND_READY) != 0)
    out: dict = {}
    for L, kk in zip(own[g][m].tolist(), k[m].tolist()):
        out[(L, kk)] = out.get((L, kk), 0) + 1
    return out


def ds_drain_cost_ref(w: World, by_domain=False) -> np.ndarray:
    """The per-key form restated: per key, OR the (row, key) facts into (DS, key) bits and gate them with the DS's
    flags in the before sweep (lwse.h, "Exact in one pass")."""
    n_keys = w.n_domains if by_domain else len(w.nodes)
    out = np.zeros(n_keys, R.DS_DRAIN_COST)
    lws_out = w.base[0]
    L, rb, _ = ready_columns(w, np.zeros(len(w.lws), np.int64))
    owner, slot, _, spec = read_rows(w.ds, len(w.roles), len(w.revroles))
    take = (L >= 0) & (owner >= 0)
    rows_of: dict = {}
    for r in np.flatnonzero(take):
        rows_of.setdefault(int(L[r]), []).append(int(r))
    before = _sweep(w, rb)[0]
    entries: dict = {}  # (DS, key) → [new zeroed, new changed, old mask]
    for (Lr, k), lost in lost_pairs(w, by_domain).items():
        for r in rows_of.get(Lr, []):
            b = int(rb[r])
            a = int(np.clip(b - lost, I32_MIN, I32_MAX))
            zero = b >= 1 and a < 1
            out["rows_touched"][k] += 1
            out["rows_zeroed"][k] += zero
            d = int(owner[r])
            e = entries.setdefault((d, k), [False, False, 0])
            if spec[r]:
                if slot[r] == int(w.ds["n_old_revs"][d]):
                    e[0] |= zero
                    e[1] |= a != b
                elif zero:
                    e[2] |= 1 << int(slot[r])
    for (d, k), (nz, nc, om) in entries.items():
        f, rr = int(before["flags"][d]), int(before["ready_revs"][d])
        out["ds_touched"][k] += 1
        out["ds_service_lost"][k] += bool(nz and f & R.DOUT_NEW_READY)
        out["ds_old_service_lost"][k] += bool(om & rr)
        out["ds_stalled"][k] += bool(nc and f & R.DOUT_STABLE)
    return out


def cost_row_of(totals) -> dict:
    """The per-key columns a set-form answer stands for."""
    return {"ds_touched": totals["n_touched"], "ds_service_lost": totals["n_service_lost"],
            "ds_old_service_lost": totals["n_old_service_lost"], "ds_stalled": totals["n_stalled"],
            "rows_touched": totals["rows_touched"], "rows_zeroed": totals["rows_zeroed"]}


# --------------------------------------------------------------------------------------------------
# worlds
# --------------------------------------------------------------------------------------------------
def _children(n_lws, n_nodes, seed, nodes_per_domain=8):
    from lws_b200 import synth

    p = synth.Profile("ds-drain", n_lws, size_choices=(2, 4, 8), replicas_choices=(1, 2, 3, 4, 6), n_nodes=n_nodes,
                      nodes_per_domain=nodes_per_domain, node_capacity=4096, f_mid_update=0.1, p_group_ready=0.9,
                      p_leader_unscheduled=0.02, restart_policy_p=(0.1, 0.7, 0.2))
    return synth.make(p, seed=seed)


def ds_drain_world(n_ds=200, n_lws=None, n_nodes=48, seed=3, nodes_per_domain=8, fallbacks=True, bad=True,
                   roles=(2, 3)) -> World:
    """C4-style DS tables (2 or 3 spec roles, some removed roles, 1-3 old revisions) whose existing revision-role
    rows link to child LWS rows with pods on nodes.  New-revision rows of half the DS take their child's ready count
    as replicas, so those DS are stable (or ready) before the drain.  With ``fallbacks``, some rows fall back: no
    link, a stale uid, a row past the LWS table, or a child whose result is excluded; some pairs of rows share a
    child.  With ``bad``, a few DS are BAD_TABLE (n_spec_roles > n_roles)."""
    import oracle
    from lws_b200 import synth

    rng = np.random.default_rng(seed)
    dst = synth.make_ds(n_ds, n_roles_choices=roles, seed=seed)
    ds, roles, rr = dst.ds, dst.roles, dst.revroles
    ex = np.flatnonzero(rr["flags"] & R.RR_EXISTS)
    t = _children(n_lws or max(len(ex) + 8, 16), n_nodes, seed + 1, nodes_per_domain)
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.flags & R.SWEEP_GANG)[:2]
    lws_out = base[0]
    links = none_links(len(rr))
    child = rng.permutation(len(t.lws))[: len(ex)] if len(t.lws) >= len(ex) else rng.integers(0, len(t.lws), len(ex))
    links["lws_row"][ex] = child
    links["lws_uid_hash"][ex] = t.lws["uid_hash"][child]
    if fallbacks and len(ex) > 8:
        pick = rng.permutation(ex)
        q = max(1, len(ex) // 40)
        links["lws_row"][pick[:q]] = R.NONE                                          # not linked
        links["lws_uid_hash"][pick[q: 2 * q]] ^= np.uint64(1)                         # stale uid
        links["lws_row"][pick[2 * q: 3 * q]] = len(t.lws) + np.arange(q)             # past the LWS table
        shared = pick[3 * q: 5 * q]                                                   # two rows, one child
        links["lws_row"][shared[1::2]] = links["lws_row"][shared[0::2][: len(shared[1::2])]]
        links["lws_uid_hash"][shared[1::2]] = links["lws_uid_hash"][shared[0::2][: len(shared[1::2])]]
    # half the DS: new-revision rows with replicas = their child's ready count (stable before the drain)
    n = ds["n_roles"].astype(np.int64)
    d_of = np.repeat(np.arange(n_ds), (ds["n_old_revs"].astype(np.int64) + 1) * n)
    k = np.arange(len(rr)) - ds["rev_base"][d_of].astype(np.int64)
    is_new = k // n[d_of] == ds["n_old_revs"][d_of]
    L = link_targets(rr, links, t.lws, lws_out)
    stable_ds = rng.random(n_ds) < 0.5
    sel = is_new & stable_ds[d_of] & (L >= 0)
    rr["replicas"][sel] = lws_out["ready_replicas"][L[sel]]
    rr["flags"][sel] &= ~np.uint32(R.RR_REPLICAS_NIL)
    if bad:
        for d in rng.choice(n_ds, size=max(1, n_ds // 50), replace=False):
            ds["n_spec_roles"][d] = ds["n_roles"][d] + 1
    return World(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags, ds, roles, rr, links, base)


def single_row_world(keys: dict, n_nodes=64, nodes_per_domain=4) -> World:
    """DS rows {d: node} (nodes below n_nodes - 1): DS d has one spec role and no old revision, its one revision-role row linked to a child
    LWS of one ready group whose two pods are on that node; every other DS row is vacant (zeroed).  Draining the
    node restarts the group, so each listed DS gives exactly one (row, key) pair of the per-key form, on (d, node)."""
    import oracle
    from lws_b200 import synth

    ds_rows = sorted(keys)
    n = len(ds_rows)
    p = synth.Profile("single-row", 2 * n + 16, size_choices=(2,), replicas_choices=(1,), n_nodes=n_nodes,
                      nodes_per_domain=nodes_per_domain, node_capacity=4096, f_mid_update=0.0, p_group_ready=1.0,
                      p_leader_unscheduled=0.0, restart_policy_p=(0.0, 1.0, 0.0))
    t = synth.make(p, seed=5)
    fl = t.flags & R.SWEEP_GANG
    go = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl)[1]
    # children: LWS rows of one group that is ready and not restarting, each its own ranges' only member
    own = owners(t.lws, t.groups)
    ok_g = (own >= 0) & ((go["flags"] & R.GOUT_COND_READY) != 0) & ((go["flags"] & RESTART) == 0)
    good = [L for L in range(len(t.lws)) if int(t.lws["group_count"][L]) == 1
            and ok_g[int(t.lws["group_base"][L])] and own[int(t.lws["group_base"][L])] == L]
    low = np.uint32((1 << R.PODID_NODE_SHIFT) - 1)
    pod_ident0, groups0 = t.pod_ident.copy(), t.groups.copy()
    roles = R.aligned_empty(n, R.DS_ROLE_REC)
    roles[:] = (1, 1, 0, R.ROLE_IN_SPEC | R.ROLE_HAS_ROLLING_CONFIG)
    rr = R.aligned_empty(n, R.DS_REVROLE_REC)
    rr[:] = (1, -1, 1, R.RR_EXISTS | (1 << R.RR_TS_SHIFT))
    ds = R.aligned_empty(ds_rows[-1] + 1 if n else 0, R.DS_REC)
    ds[:] = 0
    for j, d in enumerate(ds_rows):
        ds[d] = (100 + d, j, 1, 1, j, 0, R.DS_HAS_NEW_REVISION)
    while True:  # (a candidate whose drain restarts nothing, e.g. behind the pending gate, is dropped)
        assert len(good) >= n
        child = np.array(good[:n], np.int64)
        node_of = np.full(len(t.lws), n_nodes - 1, np.int64)  # (other LWS rows: the last node, drained by no case)
        node_of[child] = [keys[d] for d in ds_rows]
        t.pod_ident[:], t.groups[:] = pod_ident0, groups0
        for g in range(len(t.groups)):
            L = int(t.groups["lws_index"][g])
            node = int(node_of[L]) if L < len(t.lws) else n_nodes - 1
            pb, pc = int(t.groups["pod_base"][g]), int(t.groups["pod_count"][g])
            t.groups["leader_node"][g] = node
            t.pod_ident["place"][pb: pb + pc] = (t.pod_ident["place"][pb: pb + pc] & low) | np.uint32(node << R.PODID_NODE_SHIFT)
        base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl)[:2]
        links = R.aligned_empty(n, R.DS_LINK)
        links["lws_row"] = child
        links["lws_uid_hash"] = t.lws["uid_hash"][child]
        links["reserved"] = 0
        w = World(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags, ds, roles, rr, links, base)
        pairs = lost_pairs(w, False)
        bad = [int(child[j]) for j, d in enumerate(ds_rows) if pairs.get((int(child[j]), keys[d])) != 1]
        if not bad:
            return w
        good = [L for L in good if L not in bad]


def linked_ds(w: World) -> int:
    """The first DS that passes the table checks and has a row that takes an LWS value."""
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    owner = read_rows(w.ds, len(w.roles), len(w.revroles))[0]
    return int(owner[(L >= 0) & (owner >= 0)][0])


def overlap_worlds(w: World, copies: int):
    """(shared, copied): ``w`` with ``copies`` more DS rows, each a copy of the record of DS ``linked_ds(w)``.  In
    ``shared`` the copies keep its role and revision-role ranges, so ``copies + 1`` DS read the same rows (accepted
    input: the tables do not require disjoint ranges).  In ``copied`` each copy points at a copy of those rows and of
    their links, so every DS reads rows of its own with the same values.  Both give every DS the same inputs."""
    d0 = linked_ds(w)
    rec = w.ds[d0]
    n, V = int(rec["n_roles"]), int(rec["n_old_revs"])
    rb, vb, nrr = int(rec["role_base"]), int(rec["rev_base"]), (V + 1) * n
    extra = R.aligned_empty(copies, R.DS_REC)
    extra[:] = rec
    shared_ds = np.concatenate([w.ds, extra])
    copied_ds = np.concatenate([w.ds, extra])
    copied_ds["role_base"][len(w.ds):] = len(w.roles) + n * np.arange(copies)
    copied_ds["rev_base"][len(w.ds):] = len(w.revroles) + nrr * np.arange(copies)
    roles = np.concatenate([w.roles] + [w.roles[rb: rb + n]] * copies)
    revroles = np.concatenate([w.revroles] + [w.revroles[vb: vb + nrr]] * copies)
    links = np.concatenate([w.links] + [w.links[vb: vb + nrr]] * copies)

    def world(ds, ro, rr, lk):
        return World(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, w.flags,
                     np.ascontiguousarray(ds), np.ascontiguousarray(ro), np.ascontiguousarray(rr),
                     np.ascontiguousarray(lk), w.base)

    return world(shared_ds, w.roles, w.revroles, w.links), world(copied_ds, roles, revroles, links)


def index_entries(w: World) -> int:
    """The per-key form's reverse-index entries: rows that take an LWS value, once per DS whose ranges hold them."""
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    total = 0
    for d in np.flatnonzero(ds_ok(w.ds, len(w.roles), len(w.revroles))):
        vb, nrr = int(w.ds["rev_base"][d]), (int(w.ds["n_old_revs"][d]) + 1) * int(w.ds["n_roles"][d])
        total += int((L[vb: vb + nrr] >= 0).sum())
    return total


def table_slot(k, mask):
    """table_slot of lwse_drain_kernels.cu: the home slot of a 64-bit table key."""
    M = (1 << 64) - 1
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M
    k ^= k >> 33
    return k & mask


def table_slots(pairs):
    """The engine's sizing of a (DS, key) table: a power of two >= 2 * pairs, at least 256."""
    slots = 256
    while slots < 2 * pairs:
        slots <<= 1
    return slots


def wrap_keys(n_pairs=128, n_wrap=12, n_nodes=64):
    """{DS row: node} for single_row_world with n_pairs pairs: the first n_wrap have (DS, node) keys whose home is
    the last slot of a table sized for n_pairs, so that inserting them probes past it to slot 0 and on."""
    mask = table_slots(n_pairs) - 1
    keys, d = {}, 0
    while len(keys) < n_wrap:
        for node in range(n_nodes - 1):
            if table_slot((d << 32) | node, mask) == mask:
                keys[d] = node
                break
        d += 1
    while len(keys) < n_pairs:
        keys[d] = d % (n_nodes - 1)
        d += 1
    return keys
