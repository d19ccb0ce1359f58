"""DS drain waves (lwse_resident_ds_drain_waves) by its definition (lwse.h, "DS drain waves"), without a GPU:

- ``plan_literal``: first-fit where every probe is the set forms ``drain_budget_ref`` and ``ds_drain_ref`` over
  W ∪ {k} — the definition as written;
- ``plan_fast``: the same plan from ``drain_ref.restart_pairs``, per-(LWS, wave) lost counters and one cap per LWS
  row (the exactness argument) — what the device computes;
- ``slack_world``: ``ds_drain_world`` with the children's maxUnavailable set to 1, 2, 50 % or 100 % (or one of
  them for every child), so that the LWS floors leave room and the DS verdicts decide.

Both planners return (keys: DS_DRAIN_WAVE_KEY rows in query order, waves: DS_DRAIN_WAVE rows, totals dict)."""
import numpy as np

from drain_budget_ref import (I32_MAX, I32_MIN, budgets, domain_nodes, drain_budget_cost_ref, drain_budget_ref, key_of,
                              min_margin_of, owners)
from drain_ref import restart_pairs
from ds_drain_edges_world import entries_of
from ds_drain_ref import World, _sweep, ds_drain_cost_ref, ds_drain_ref, lost_pairs, ready_columns
from lws_b200 import records as R

NONE = R.NONE
DEFAULT = R.DSW_LWS_FLOOR | R.DSW_DS_SERVICE | R.DSW_DS_OLD_SERVICE
CONSTRAINTS = (R.DSW_LWS_FLOOR, R.DSW_DS_SERVICE, R.DSW_DS_OLD_SERVICE, R.DSW_DS_STALL, DEFAULT, R.DSW_ALL)
DS_WAVE_FIELDS = ("ds_touched", "ds_service_lost", "ds_old_service_lost", "ds_stalled", "rows_touched", "rows_zeroed")


def _totals(keys, n_waves):
    st = keys["status"]
    return {"n_waves": n_waves, "n_planned": int((st == R.DRAINW_PLANNED).sum()),
            "n_breaches_alone": int((st == R.DRAINW_BREACHES_ALONE).sum()), "n_no_wave": int((st == R.DRAINW_NO_WAVE).sum())}


def _key_nodes(w: World, by_domain, ids):
    return domain_nodes(w.nodes, w.n_domains, ids) if by_domain else np.asarray(list(ids), dtype=np.int64)


def triggers(budget_totals, ds_totals) -> int:
    """The DSW_* bits a drain set triggers, from its two set-form answers."""
    return ((R.DSW_LWS_FLOOR if budget_totals["n_breached"] else 0)
            | (R.DSW_DS_SERVICE if ds_totals["n_service_lost"] else 0)
            | (R.DSW_DS_OLD_SERVICE if ds_totals["n_old_service_lost"] else 0)
            | (R.DSW_DS_STALL if ds_totals["n_stalled"] else 0))


def alone_bits(bcost, dcost) -> np.ndarray:
    """Per key: the DSW_* bits it triggers alone, from the two per-key forms."""
    return ((bcost["lws_breached"] > 0) * R.DSW_LWS_FLOOR | (dcost["ds_service_lost"] > 0) * R.DSW_DS_SERVICE
            | (dcost["ds_old_service_lost"] > 0) * R.DSW_DS_OLD_SERVICE
            | (dcost["ds_stalled"] > 0) * R.DSW_DS_STALL).astype(np.uint32)


def _key_row(row, k, bcost, dcost, alone):
    row["id"], row["wave"], row["alone"] = k, NONE, alone[k]
    for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        row[f] = bcost[k][f]
    for f in ("ds_touched", "ds_service_lost", "ds_old_service_lost", "ds_stalled"):
        row[f] = dcost[k][f]


def wave_row_of_sets(brows, btot, dtot, n_keys):
    """A DS_DRAIN_WAVE row from the two set forms' answers over a wave's ids."""
    w = np.zeros(1, R.DS_DRAIN_WAVE)[0]
    w["n_keys"] = n_keys
    w["lws_touched"] = btot["n_touched"]
    w["lws_breached"] = btot["n_breached"]
    w["lws_loses_available"] = btot["n_loses_available"]
    for f in ("n_pods_evicted", "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted", "n_pods_recreated"):
        w[f] = btot[f]
    w["min_margin"] = min_margin_of(brows)
    w["ds_touched"] = dtot["n_touched"]
    w["ds_service_lost"] = dtot["n_service_lost"]
    w["ds_old_service_lost"] = dtot["n_old_service_lost"]
    w["ds_stalled"] = dtot["n_stalled"]
    w["rows_touched"] = dtot["rows_touched"]
    w["rows_zeroed"] = dtot["rows_zeroed"]
    return w


def plan_literal(w: World, ids, by_domain=False, max_waves=64, constraints=DEFAULT):
    """First-fit by the definition: each probe is ``drain_budget_ref`` and ``ds_drain_ref`` over W ∪ {k}."""
    lws_out, base_out = w.base
    bcost = drain_budget_cost_ref(w.lws, lws_out, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, base_out,
                                  by_domain)
    dcost = ds_drain_cost_ref(w, by_domain)
    alone = alone_bits(bcost, dcost)

    def probe(ks):
        drain = _key_nodes(w, by_domain, ks)
        b = drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, drain, w.sweep_flags, base=w.base)
        d = ds_drain_ref(w, drain)
        return b, d, triggers(b[1], d[1])

    keys = np.zeros(len(ids), R.DS_DRAIN_WAVE_KEY)
    waves = []
    for i, k in enumerate(int(x) for x in ids):
        row = keys[i]
        _key_row(row, k, bcost, dcost, alone)
        got = probe([k])[2]
        assert got == alone[k], (k, got, alone[k])
        if got & constraints:
            row["status"] = R.DRAINW_BREACHES_ALONE
            continue
        for v, W in enumerate(waves):
            if not probe(W + [k])[2] & constraints:
                W.append(k)
                row["wave"] = v
                break
        else:
            if len(waves) < max_waves:
                waves.append([k])
                row["wave"] = len(waves) - 1
            else:
                row["status"] = R.DRAINW_NO_WAVE
    out = np.zeros(len(waves), R.DS_DRAIN_WAVE)
    for v, W in enumerate(waves):
        b, d, trig = probe(W)
        assert not trig & constraints
        out[v] = wave_row_of_sets(b[0], b[1], d[1], len(W))
    return keys, out, _totals(keys, len(waves))


def linked_entries(w: World):
    """Every revision-role row a DS sweep reads that takes an LWS value, once per DS whose range holds it (as the
    device walks them: DS ranges may overlap): (DS, row, slot, spec, L) arrays, slot = V for the new revision."""
    d, row, slot, spec = entries_of(w)
    L = ready_columns(w, np.zeros(len(w.lws), np.int64))[0]
    keep = L[row] >= 0
    return d[keep], row[keep], slot[keep], spec[keep], L[row][keep]


def caps(w: World, gates=True):
    """Per LWS row: (linked, service, old_service, stall) — a row the DS sweep reads takes its value, and such a
    row is gated for that verdict by its DS's flags in the before sweep.  ``gates`` off is a mutation: every linked
    spec row caps, whatever its DS's flags."""
    n = len(w.lws)
    rb = ready_columns(w, np.zeros(n, np.int64))[1]
    before = _sweep(w, rb)[0]
    linked, service, old, stall = (np.zeros(n, bool) for _ in range(4))
    for d, _, v, spec, Lr in zip(*linked_entries(w)):
        linked[Lr] = True
        if not spec:
            continue
        f = int(before["flags"][d])
        if v == int(w.ds["n_old_revs"][d]):
            service[Lr] |= bool(f & R.DOUT_NEW_READY) or not gates
            stall[Lr] |= bool(f & R.DOUT_STABLE) or not gates
        else:
            old[Lr] |= bool((int(before["ready_revs"][d]) >> int(v)) & 1) or not gates
    return linked, service, old, stall


def ds_cost_per_ds(w: World, by_domain=False) -> np.ndarray:
    """The DS per-key form restated over ``linked_entries`` (a row read by k DS counts k times, as on the device);
    equal to ``ds_drain_cost_ref`` where DS ranges do not overlap."""
    n_keys = w.n_domains if by_domain else len(w.nodes)
    out = np.zeros(n_keys, R.DS_DRAIN_COST)
    rb_r = ready_columns(w, np.zeros(len(w.lws), np.int64))[1]
    before = _sweep(w, rb_r)[0]
    by_L: dict = {}
    for e in zip(*linked_entries(w)):
        by_L.setdefault(int(e[4]), []).append(e)
    facts: dict = {}  # (DS, key) → [new zeroed, new changed, old mask]
    for (Lr, k), lost in lost_pairs(w, by_domain).items():
        for d, row, v, spec, _ in by_L.get(Lr, []):
            b = int(rb_r[row])
            a = int(np.clip(b - lost, I32_MIN, I32_MAX))
            zero = b >= 1 and a < 1
            out["rows_touched"][k] += 1
            out["rows_zeroed"][k] += zero
            f = facts.setdefault((int(d), k), [False, False, 0])
            if spec:
                if v == int(w.ds["n_old_revs"][d]):
                    f[0] |= zero
                    f[1] |= a != b
                elif zero:
                    f[2] |= 1 << int(v)
    for (d, k), (nz, nc, om) in facts.items():
        fl, rr = int(before["flags"][d]), int(before["ready_revs"][d])
        out["ds_touched"][k] += 1
        out["ds_service_lost"][k] += bool(nz and fl & R.DOUT_NEW_READY)
        out["ds_old_service_lost"][k] += bool(om & rr)
        out["ds_stalled"][k] += bool(nc and fl & R.DOUT_STABLE)
    return out


def slacks(w: World, constraints, linked_bind=True, gates=True):
    """(bound per group, slack per LWS row — None for no bound) under ``constraints``.  ``linked_bind`` and ``gates``
    off are the mutations the tests show to be wrong: only evaluated rows bind pairs; every linked spec row caps,
    whatever its DS's flags."""
    lws_out, base_out = w.base
    floor, rb, evaluated, _, _, _ = budgets(w.lws, lws_out, len(w.groups))
    linked, service, old, stall = caps(w, gates)
    slack = [None] * len(w.lws)
    for L in range(len(w.lws)):
        c = []
        if constraints & R.DSW_LWS_FLOOR and evaluated[L]:
            c.append(int(rb[L]) - int(floor[L]))
        if (constraints & R.DSW_DS_SERVICE and service[L]) or (constraints & R.DSW_DS_OLD_SERVICE and old[L]):
            c.append(int(rb[L]) - 1)
        if constraints & R.DSW_DS_STALL and stall[L]:
            c.append(0)
        slack[L] = min(c) if c else None
    own = owners(w.lws, w.groups)
    ready = (base_out["flags"] & R.GOUT_COND_READY) != 0
    member = own >= 0
    o = np.where(member, own, 0)
    bound = ready & member & (evaluated[o] | (linked[o] if linked_bind else False))
    return bound, slack


def plan_fast(w: World, ids, by_domain=False, max_waves=64, constraints=DEFAULT, linked_bind=True, gates=True):
    """First-fit from the restart pairs: per wave the set of its groups and lost(L, W) per LWS row, checked against
    one slack per row."""
    lws_out, base_out = w.base
    n_keys = w.n_domains if by_domain else len(w.nodes)
    bcost = drain_budget_cost_ref(w.lws, lws_out, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, base_out,
                                  by_domain)
    dcost = ds_cost_per_ds(w, by_domain)
    alone = alone_bits(bcost, dcost)
    g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base_out)
    k = key_of(w.nodes, w.n_domains, by_domain)[n]
    pairs = np.unique(np.stack([k[k >= 0], g[k >= 0]], axis=1), axis=0) if (k >= 0).any() else np.zeros((0, 2), np.int64)
    starts = np.searchsorted(pairs[:, 0], np.arange(n_keys + 1))
    own = owners(w.lws, w.groups)
    floor, rb, evaluated, available, gb, _ = budgets(w.lws, lws_out, len(w.groups))
    bound, slack = slacks(w, constraints, linked_bind, gates)
    ready = (base_out["flags"] & R.GOUT_COND_READY) != 0
    member = own >= 0
    o = np.where(member, own, 0)
    nb = ready & member & ((np.arange(len(w.groups)) - gb[o]) < w.lws["replicas"][o].astype(np.int64))

    def fits(lost_of, b):
        Ls, cnt = np.unique(own[np.asarray(b, dtype=np.int64)], return_counts=True)
        return all(slack[L] is None or lost_of.get(int(L), 0) + int(c) <= slack[L] for L, c in zip(Ls, cnt))

    keys = np.zeros(len(ids), R.DS_DRAIN_WAVE_KEY)
    waves = []  # [ids, groups (set), lost {L: n}]
    for i, key in enumerate(int(x) for x in ids):
        gs = pairs[starts[key]:starts[key + 1], 1]
        row = keys[i]
        _key_row(row, key, bcost, dcost, alone)
        b = gs[bound[gs]]
        if not fits({}, b):
            row["status"] = R.DRAINW_BREACHES_ALONE
            continue
        chosen = None
        for v, (W_ids, W_groups, W_lost) in enumerate(waves):
            if fits(W_lost, [x for x in b.tolist() if x not in W_groups]):
                chosen = v
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
    # the DS columns of a wave: its lost(L, W) through every linked row, gated by the before sweep
    rb_r = ready_columns(w, np.zeros(len(w.lws), np.int64))[1]
    before = _sweep(w, rb_r)[0]
    entries = list(zip(*linked_entries(w)))
    out = np.zeros(len(waves), R.DS_DRAIN_WAVE)
    for v, (W_ids, W_groups, W_lost) in enumerate(waves):
        G = np.asarray(sorted(W_groups), dtype=np.int64)
        row = out[v]
        row["n_keys"] = len(W_ids)
        row["n_pods_evicted"] = int(bcost["pods"][W_ids].sum())
        row["n_leaders_evicted"] = int(bcost["leaders"][W_ids].sum())
        row["n_groups_restarted"] = len(G)
        row["n_ready_restarted"] = int(ready[G].sum()) if len(G) else 0
        row["n_pods_recreated"] = int(w.groups["pod_count"][G].astype(np.int64).sum()) if len(G) else 0
        Gm = G[member[G]] if len(G) else G
        touched = np.unique(own[Gm])
        row["lws_touched"] = len(touched)
        row["lws_loses_available"] = len(np.unique(own[Gm[nb[Gm] & evaluated[own[Gm]] & available[own[Gm]]]]))
        margin, breached = I32_MAX, 0
        for L in touched[evaluated[touched]]:
            lost = W_lost.get(int(L), 0)
            after = int(np.clip(rb[L] - lost, I32_MIN, I32_MAX))
            margin = min(margin, int(np.clip(after - floor[L], I32_MIN, I32_MAX)))
            breached += lost > 0 and int(rb[L]) - lost < int(floor[L])
        row["min_margin"] = margin
        row["lws_breached"] = breached
        facts = {}  # DS → [touched, new zeroed, new changed, old fell]
        for d, r, slot, spec, Lr in entries:
            lost = W_lost.get(int(Lr), 0)
            if lost == 0:
                continue
            d = int(d)
            b0 = int(rb_r[r])
            a0 = int(np.clip(b0 - lost, I32_MIN, I32_MAX))
            zero = b0 >= 1 and a0 < 1
            row["rows_touched"] += 1
            row["rows_zeroed"] += zero
            f = facts.setdefault(d, [False, False, 0])
            if spec:
                if int(slot) == int(w.ds["n_old_revs"][d]):
                    f[0] |= zero
                    f[1] |= a0 != b0
                elif zero:
                    f[2] |= 1 << int(slot)
        for d, (nz, nc, om) in facts.items():
            fl, rr = int(before["flags"][d]), int(before["ready_revs"][d])
            row["ds_touched"] += 1
            row["ds_service_lost"] += bool(nz and fl & R.DOUT_NEW_READY)
            row["ds_old_service_lost"] += bool(om & rr)
            row["ds_stalled"] += bool(nc and fl & R.DOUT_STABLE)
        out[v] = row
    return keys, out, _totals(keys, len(waves))


def orders(ids, bcost, seed=3):
    """The key orders the tests compare: as given, reversed, by drain cost (largest min_margin first, then fewest
    groups restarted), and a seeded shuffle."""
    ids = np.asarray(ids, dtype=np.int64)
    c = bcost[ids]
    by_cost = ids[np.lexsort((ids, c["groups_restarted"], -c["min_margin"].astype(np.int64)))]
    return {"given": ids, "reversed": ids[::-1].copy(), "by_cost": by_cost,
            "random": np.random.default_rng(seed).permutation(ids)}


MU_CHOICES = ((1, False), (2, False), (50, True), (100, True))


def slack_world(mu=None, seed=3, **kw) -> World:
    """``ds_drain_world(**kw)`` with every child's maxUnavailable set to ``mu`` ((value, is_percent)), or each to a
    seeded choice of 1, 2, 50 % and 100 %; the baseline swept again."""
    import oracle
    from ds_drain_ref import ds_drain_world

    w = ds_drain_world(seed=seed, **kw)
    lws = w.lws.copy()
    rng = np.random.default_rng(seed + 100)
    pick = [mu] * len(lws) if mu is not None else [MU_CHOICES[i] for i in rng.integers(0, len(MU_CHOICES), len(lws))]
    for L, (v, pct) in enumerate(pick):
        lws["max_unavailable"][L] = v
        if pct:
            lws["flags"][L] |= np.uint32(R.LWS_UNAVAIL_IS_PERCENT)
        else:
            lws["flags"][L] &= ~np.uint32(R.LWS_UNAVAIL_IS_PERCENT)
    base = oracle.sweep_lws(lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.flags & R.SWEEP_GANG)[:2]
    return World(lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, w.flags, w.ds, w.roles, w.revroles,
                 w.links, base)


# --------------------------------------------------------------------------- #
# the edges world
# --------------------------------------------------------------------------- #
def ds_waves_edges_world():
    """One case per edge of the cap argument, each on nodes of its own (one node per domain, so both scopes name the
    same keys).  Children have maxUnavailable = replicas (floor 0) unless a case says otherwise; DS rows come from
    ``ds_drain_edges_world._ds`` (every row present, ready 1 until a link says otherwise):

    - ``ready2``: a service child (one spec role, no old revision) of 2 ready groups: cap 1, two keys of one group
      each — the second opens a wave of its own;
    - ``service_ready1``: a service child of 1 ready group: cap 0, the key breaches alone;
    - ``stable``: a STABLE rolling DS whose new-revision child has 2 ready groups: the key stalls it, nothing else;
    - ``old_rev``: the child of an old revision's spec row (its ready_revs bit set): OLD_SERVICE only;
    - ``removed``: the child of a removed role's row: rows zeroed, no verdict;
    - ``bad_table``: the child of a BAD_TABLE DS: nothing;
    - ``fb_unlinked`` / ``fb_stale_uid`` / ``fb_past_table`` / ``fb_excluded`` / ``fb_not_exists``: a row that falls
      back (no link, a stale uid, an LWS row past the table, a child whose result is excluded, a row that does not
      exist): nothing;
    - ``shared``: one child of 2 ready groups read by two DS: cap 1, two DS touched per key;
    - ``below``: a service child already below its LWS floor (3 replicas, maxUnavailable 0, 2 ready): the LWS floor
      breaches alone, the DS cap (1) does not;
    - ``unevaluated``: a service child with LWSE_LWS_INTSTR_INVALID and no StatefulSet (re-swept: linked, not
      EVALUATED) of 1 ready group: cap 0 — it binds only because linked pairs are bound;
    - ``cap``: 65 keys, each one ready group of a child of slack 1 (65 replicas, maxUnavailable 1) that a DS links:
      waves 0-63, then NO_WAVE, under the LWS floor.
    → (World, ids in the given order, notes {label: keys})."""
    import drain_edges_world as DW
    import ds_limits_world as LW
    from ds_drain_edges_world import _ds, world_of

    n_nodes = 96
    nodes, n_domains = DW.node_table(n_nodes, 1)
    b = DW.Builder(nodes, n_domains)
    nxt = iter(range(n_nodes))
    items, tg, notes, at = [], [], {}, {}

    def child(n_ready, n_not=0, replicas=None, mu=None):
        reps = n_ready + n_not if replicas is None else replicas
        o = b.obj(DW.ON, size=1, replicas=reps, mu=reps if mu is None else mu)
        ks = [next(nxt) for _ in range(n_ready + n_not)]
        for j, k in enumerate(ks):
            b.group(o, [], leader=k, ready=j < n_ready)
        return o, ks

    def ds(x, targets, label=None):
        items.append(x)
        tg.append(np.asarray(targets, np.int64))
        if label:
            at[label] = len(items) - 1
        return len(items) - 1

    c, notes["ready2"] = child(2)
    ds(_ds(1, 0, 0), [c])
    c, notes["service_ready1"] = child(1)
    ds(_ds(1, 0, 0), [c])
    c, ks = child(2)
    co, _ = child(1)
    ds(_ds(1, 0, 1, new_replicas=2), [co, c], "stable")
    notes["stable"] = ks[:1]
    co, notes["old_rev"] = child(1)
    cn, _ = child(2)
    ds(_ds(1, 0, 1, new_replicas=2), [co, cn])
    cr, notes["removed"] = child(1)
    cs, _ = child(1)
    ds(_ds(1, 1, 0), [cs, cr])
    c, notes["bad_table"] = child(1)
    ds(_ds(1, 0, 0), [c], "bad_table")
    fb = {}
    for label in ("fb_unlinked", "fb_stale_uid", "fb_past_table", "fb_excluded", "fb_not_exists"):
        c, notes[label] = child(1)
        ds(_ds(1, 0, 0), [-1 if label == "fb_unlinked" else c], label)
        fb[label] = c
    c, notes["shared"] = child(2)
    ds(_ds(1, 0, 0), [c])
    ds(_ds(1, 0, 0), [c])
    c, ks = child(2, n_not=1, replicas=3, mu=0)
    ds(_ds(1, 0, 0), [c])
    notes["below"] = ks[:1]
    unev, notes["unevaluated"] = child(1)
    ds(_ds(1, 0, 0), [unev])
    c, notes["cap"] = child(65, replicas=65, mu=1)
    ds(_ds(1, 0, 0), [c])
    e = b.tables("ds_waves_edges")
    e.lws[unev]["flags"] = (e.lws[unev]["flags"] | np.uint32(R.LWS_INTSTR_INVALID)) & ~np.uint32(R.LWS_STS_EXISTS)
    e.lws[fb["fb_excluded"]]["flags"] |= np.uint32(R.LWS_INTSTR_INVALID)  # (with a StatefulSet: RUP_ERROR)
    dsr, roles, rr = LW.assemble(items)
    vb = dsr["rev_base"].astype(np.int64)
    targets = np.full(len(rr), -1, np.int64)
    for d, t in enumerate(tg):
        targets[vb[d]: vb[d] + len(t)] = t
    dsr["n_spec_roles"][at["bad_table"]] = dsr["n_roles"][at["bad_table"]] + 1
    rr["flags"][vb[at["fb_not_exists"]]] &= ~np.uint32(R.RR_EXISTS)
    w = world_of(e, dsr, roles, rr, targets)  # (the baseline swept after every edit above)
    w.links["lws_uid_hash"][vb[at["fb_stale_uid"]]] ^= np.uint64(1)
    w.links["lws_row"][vb[at["fb_past_table"]]] = len(w.lws) + 5
    order = ("ready2", "service_ready1", "stable", "old_rev", "removed", "bad_table", "fb_unlinked", "fb_stale_uid",
             "fb_past_table", "fb_excluded", "fb_not_exists", "shared", "below", "unevaluated", "cap")
    ids = [k for label in order for k in notes[label]]
    notes["children"] = dict(unevaluated=unev, fb_excluded=fb["fb_excluded"], stable_ds=at["stable"])
    return w, ids, notes
