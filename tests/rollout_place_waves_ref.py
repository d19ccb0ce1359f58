"""Rollout placement waves (lwse_resident_rollout_place_waves) by their definition (lwse.h, "rollout placement
waves"), without a GPU.  The plan is stated twice:

- ``mode="literal"``: the global first-fit in query order; every probe W ∪ {k} is the set form — the placement
  what-if over every namespace with extra = the E_i of the set concatenated in query order, numbered over the whole
  concatenation;
- ``mode="ns"``: the decomposition of DESIGN.md §3.5: an independent first-fit per namespace, each probe solving the
  namespace alone with the column's rows then E_k, numbered per (wave, namespace) — what the device computes.

``variant`` names a statement the tests show to be wrong or equivalent: ``"alone_only"`` (a key clean alone joins
wave 0), ``"drop_earlier"`` (a probe leaves out the wave's earlier entries of k's namespace), ``"reverse_ns"`` (the
concatenation reversed within each namespace) and ``"by_ns"`` (the concatenation grouped by namespace: the same
plan, argument (1)).  E_i and the alone rows come from ``rollout_place_ref``."""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import records as R
from rollout_place_ref import edge_world, rollout_place_ref, solve
from test_place_whatif import whatif_ref

ALL_MASKS = (R.RPW_STRANDED, R.RPW_BUMPED, R.RPW_ALL)
COUNTS = ("placed", "stranded", "own_lost", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed",
          "n_unschedulable", "n_conflict")


def alone_bits(row) -> int:
    return (R.RPW_STRANDED if int(row["stranded"]) else 0) | (
        R.RPW_BUMPED if int(row["own_lost"]) or int(row["bumped"]) else 0)


def _cat(xs):
    xs = [x for x in xs if len(x)]
    out = R.aligned_empty(sum(len(x) for x in xs), R.PLACE_REQ)
    at = 0
    for x in xs:
        out[at: at + len(x)] = x
        at += len(x)
    return out


def counts(w, after, base, x_out, ranges):
    """The set form's counts: ``after`` the rows of the resident requests, ``x_out`` those of the extra rows,
    ``ranges`` per namespace the group ranges of the set's entries with that ns."""
    was = (base["flags"] & R.PLACE_PLACED) != 0
    now = (after["flags"] & R.PLACE_PLACED) != 0
    lost = was & ~now
    own = np.zeros(len(base), bool)
    grp = w.reqs["group"].astype(np.int64)
    rns = w.reqs["ns"].astype(np.int64)
    for v, rs in ranges.items():
        for gb, gc in rs:
            own |= (rns == v) & (grp >= gb) & (grp < gb + gc)
    xp = (x_out["flags"] & R.PLACE_PLACED) != 0
    a = base.view(np.uint8).reshape(len(base), 16)
    b = after.view(np.uint8).reshape(len(after), 16)
    f = np.concatenate([after["flags"], x_out["flags"]])
    return {"placed": int(xp.sum()), "stranded": int((~xp).sum()), "own_lost": int((lost & own).sum()),
            "bumped": int((lost & ~own).sum()), "n_changed": int((a != b).any(axis=1).sum()), "n_lost": int(lost.sum()),
            "n_moved": int((was & now & (base["domain_id"] != after["domain_id"])).sum()),
            "n_gained": int((~was & now).sum()), "n_placed": int(((f & R.PLACE_PLACED) != 0).sum()),
            "n_unschedulable": int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum()),
            "n_conflict": int(((f & R.PLACE_CONFLICT) != 0).sum())}


def verdicts(c) -> int:
    return (R.RPW_STRANDED if c["stranded"] else 0) | (R.RPW_BUMPED if c["own_lost"] or c["bumped"] else 0)


class _Plan:
    def __init__(self, w, rows, ns, recs):
        self.w = w
        self.rows = np.asarray(rows, dtype=np.int64)
        self.ns = np.asarray(ns, dtype=np.int64)
        rp = rollout_place_ref(w, rows, ns, recs=recs)
        self.alone = rp["rows"]
        self.extra = rp["extra"]
        self.base = oracle.place(w.nodes, w.occ, w.n_domains, w.n_ns, w.reqs, threads=8)

    def rng(self, i):
        r = int(self.rows[i])
        return int(self.w.lws["group_base"][r]), int(self.w.lws["group_count"][r])

    def ranges(self, S):
        out = {}
        for i in S:
            out.setdefault(int(self.ns[i]), []).append(self.rng(i))
        return out

    def order(self, S, variant):
        """The concatenation order of a set (query order unless a variant changes it)."""
        S = sorted(S)
        if variant == "by_ns":
            S = sorted(S, key=lambda i: (int(self.ns[i]), i))
        elif variant == "reverse_ns":
            by = {}
            for i in S:
                by.setdefault(int(self.ns[i]), []).append(i)
            rev = {v: list(reversed(l)) for v, l in by.items()}
            S = [rev[int(self.ns[i])].pop(0) for i in S]
        return S

    def literal(self, S, variant=None):
        """The set form over every namespace."""
        S = self.order(S, variant)
        x = _cat([self.extra[i] for i in S])
        w = self.w
        after = whatif_ref(w.nodes, w.occ, w.n_domains, w.reqs, extra=x, n_ns=w.n_ns)["after_all"]
        n = len(w.reqs)
        return counts(w, after[:n], self.base, after[n:], self.ranges(S))

    def column(self, S, v, variant=None):
        """Namespace v solved alone with the set's rows of v, numbered per (wave, namespace)."""
        S = self.order([i for i in S if int(self.ns[i]) == v], variant)
        x = _cat([self.extra[i] for i in S])
        w = self.w
        n = len(w.reqs)
        after = solve(w, x, v, self.base, "ns") if len(x) else np.concatenate([self.base, x.view(R.PLACE_OUT)])
        c = counts(w, after[:n], self.base, after[n:], self.ranges(S))
        base_tot = [int(((self.base["flags"] & b) != 0).sum()) for b in (R.PLACE_PLACED, R.PLACE_UNSCHEDULABLE, R.PLACE_CONFLICT)]
        for k, b in zip(("n_placed", "n_unschedulable", "n_conflict"), base_tot):
            c[k] -= b  # a delta against the baseline
        return c


def rollout_place_waves_ref(w, rows, ns, recs=None, max_waves=R.DRAIN_WAVES_MAX, constraints=R.RPW_STRANDED,
                            mode="literal", variant=None):
    """→ dict as ``Engine.resident_rollout_place_waves(..., alone=True)``."""
    pl = _Plan(w, rows, ns, recs)
    n = len(pl.rows)
    keys = np.zeros(n, R.ROLLOUT_WAVE_KEY)
    keys["wave"] = R.NONE
    part = []
    for i in range(n):
        row = pl.alone[i]
        solved = int(row["flags"]) & R.RPL_SOLVED
        keys[i]["alone"] = alone_bits(row) if solved else 0
        if not solved:
            keys[i]["status"] = R.ROLLW_NOT_SOLVED
        elif alone_bits(row) & constraints:
            keys[i]["status"] = R.ROLLW_TRIGGERS_ALONE
        else:
            keys[i]["status"] = R.ROLLW_PLANNED
            part.append(i)
    sets = []
    if mode == "literal":
        for k in part:
            wave = None
            for c, S in enumerate(sets):
                if variant == "alone_only":
                    ok = True
                else:
                    T = [i for i in S if variant != "drop_earlier" or int(pl.ns[i]) != int(pl.ns[k])]
                    ok = not (verdicts(pl.literal(T + [k], variant)) & constraints)
                if ok:
                    wave = c
                    break
            if wave is None and len(sets) < max_waves:
                wave = len(sets)
                sets.append([])
            if wave is None:
                keys[k]["status"] = R.ROLLW_NO_WAVE
            else:
                sets[wave].append(k)
                keys[k]["wave"] = wave
        totals = [pl.literal(S, variant) for S in sets]
    else:
        cols = {}  # namespace -> its columns (lists of keys)
        for k in part:
            v = int(pl.ns[k])
            cs = cols.setdefault(v, [])
            wave = None
            for c, S in enumerate(cs):
                if not (verdicts(pl.column(S + [k], v, variant)) & constraints):
                    wave = c
                    break
            if wave is None and len(cs) < max_waves:
                wave = len(cs)
                cs.append([])
            if wave is None:
                keys[k]["status"] = R.ROLLW_NO_WAVE
            else:
                cs[wave].append(k)
                keys[k]["wave"] = wave
        n_waves = max((len(cs) for cs in cols.values()), default=0)
        sets = [[i for cs in cols.values() if c < len(cs) for i in cs[c]] for c in range(n_waves)]
        base_tot = [int(((pl.base["flags"] & b) != 0).sum()) for b in (R.PLACE_PLACED, R.PLACE_UNSCHEDULABLE, R.PLACE_CONFLICT)]
        totals = []
        for c in range(n_waves):
            t = dict.fromkeys(COUNTS, 0)
            for v, cs in cols.items():
                if c < len(cs):
                    for k2, x in pl.column(cs[c], v, variant).items():
                        t[k2] += x
            for k2, b in zip(("n_placed", "n_unschedulable", "n_conflict"), base_tot):
                t[k2] += b
            totals.append(t)
    waves = np.zeros(len(sets), R.ROLLOUT_WAVE)
    for c, (S, t) in enumerate(zip(sets, totals)):
        o = waves[c]
        o["n_keys"] = len(S)
        for k2 in COUNTS:
            o[k2] = t[k2]
        o["surge"] = t["placed"] + t["stranded"]
        o["namespaces"] = len({int(pl.ns[i]) for i in S})
        waves[c] = o
    st = keys["status"]
    return {"keys": keys, "waves": waves, "alone_rows": pl.alone, "n_waves": len(sets),
            "n_planned": int((st == R.ROLLW_PLANNED).sum()), "n_triggers_alone": int((st == R.ROLLW_TRIGGERS_ALONE).sum()),
            "n_no_wave": int((st == R.ROLLW_NO_WAVE).sum()), "n_not_solved": int((st == R.ROLLW_NOT_SOLVED).sum())}


def same_plan(a, b) -> bool:
    return (a["keys"].tobytes() == b["keys"].tobytes() and a["waves"].tobytes() == b["waves"].tobytes()
            and all(a[k] == b[k] for k in R.ROLLOUT_WAVES_TOTALS))


def key_orders(n, surge, seed):
    """The four key orders of the tests: given, reversed, shuffled and by surge (largest first)."""
    idx = np.arange(n)
    return {"given": idx, "reversed": idx[::-1].copy(), "shuffled": np.random.default_rng(seed).permutation(n),
            "by_surge": np.argsort(-np.asarray(surge, dtype=np.int64), kind="stable")}


# ---- the edge world ---------------------------------------------------------------------------------------------
EXTRA_NS = 3  # namespaces 5, 6 and 7: empty, for the edges that need a namespace of their own


def waves_world():
    """``rollout_place_ref.edge_world`` (exactly 3 fitting domains for a size-4 group; namespace 3 holds three
    unpinned lowest-priority rows on them; A has no extra row; C lacks a leader pod and has its group 0 unpinned; N,
    BT and IR are not solved; UF is UNFINISHED) with namespaces 5 .. 7 empty.  → (world, {name: LWS row})."""
    w, rows = edge_world()
    w.n_ns = 5 + EXTRA_NS
    # two of the holders of namespace 3 carry groups of object O's range: O's surge rows there lose its own rows
    w.reqs = w.reqs.copy()
    held = np.flatnonzero(w.reqs["ns"] == 3)[:2]
    w.reqs["group"][held] = int(w.lws["group_base"][OWN_OBJECT]) + np.arange(2, dtype=np.uint32)
    return w, rows


OWN_OBJECT = 21  # a stable object of namespace 1


def _prop(w, r, **kw):
    rec = w.lws[r].copy()
    for k, v in kw.items():
        rec[k] = v
    return rec


def edge_queries(w, rows):
    """The waves edge queries → {label: (rows, ns, recs or None, expected names per entry)}.  Stable objects 1, 3,
    5, ... of the edge world carry the proposals (rows must be distinct)."""
    free = [r for r in range(len(w.lws)) if r not in rows.values() and r % 2 == 1 and r != OWN_OBJECT]
    q = {}

    def props(label, entries):
        rs = np.array([e[0] for e in entries], np.uint32)
        vs = np.array([e[1] for e in entries], np.uint32)
        recs = R.aligned_empty(len(entries), R.LWS_REC)
        for i, e in enumerate(entries):
            recs[i] = _prop(w, e[0], **e[2])
        q[label] = (rs, vs, recs)

    f = free
    # two objects that each need the last 3 domains: one namespace, then two
    props("pair_one_ns", [(f[0], 5, {"replicas": 6}), (f[1], 5, {"replicas": 6})])
    props("pair_two_ns", [(f[0], 5, {"replicas": 6}), (f[1], 6, {"replicas": 6})])
    # three such objects in namespace 5 under a cap of 2, and one in namespace 6
    props("cap", [(f[0], 5, {"replicas": 6}), (f[1], 5, {"replicas": 6}), (f[2], 5, {"replicas": 6}),
                  (f[3], 6, {"replicas": 6})])
    # an object that strands alone next to an open wave of its namespace
    props("strands_alone", [(f[0], 5, {"replicas": 4}), (f[1], 5, {"replicas": 7}), (f[2], 5, {"replicas": 4})])
    # surge rows that bump the holders of namespace 3: another object's, then two of O's own and one other
    props("bumps", [(f[0], 3, {"replicas": 6}), (f[1], 5, {"replicas": 4})])
    props("own", [(OWN_OBJECT, 3, {"replicas": 6}), (f[1], 5, {"replicas": 4})])
    # no extra row, the flagged entries, an edit that is not modelled, UNFINISHED
    props("flags", [(rows["A"], 0, {}), (rows["N"], 0, {}), (rows["BT"], 0, {}), (rows["IR"], 0, {}),
                    (f[0], 5, {"size": 5}), (rows["UF"], 0, {}), (f[1], 0, {"replicas": 4})])
    # the resident form over every named object
    names = list(rows)
    q["resident"] = (np.array([rows[k] for k in names], np.uint32),
                     (np.array([rows[k] for k in names], np.int64) % 2).astype(np.uint32), None)
    return q


# ---- the tie world (argument (1)) ---------------------------------------------------------------------------------
_C1, _C2, _C3 = 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
_M = (1 << 64) - 1


def _mix(uid, g):
    pr = ((uid ^ ((g * _C1) & _M)) * _C2) & _M
    pr ^= pr >> 31
    k = ((uid + g) * _C3) & _M
    k ^= k >> 29
    return pr, k


def _unmix_priority(pr, g):
    """The uid_hash whose group g has priority ``pr`` under the encoder's mix."""
    x = pr
    x ^= x >> 31
    x ^= x >> 62  # (the inverse of x ^= x >> 31 on 64 bits)
    x = (x * pow(_C2, -1, 1 << 64)) & _M
    return x ^ ((g * _C1) & _M)


def _score(key, d):
    x = ((key & 0xFFFFFFFF) ^ ((d * 0x9E3779B1) & 0xFFFFFFFF)) & 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & 0xFFFFFFFF
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & 0xFFFFFFFF
    x ^= x >> 16
    return x | 1


def tie_world():
    """Two proposals P (size 8) and Q (size 4), one surge group each, in the empty namespace 5 of a world whose
    domains all hold 3 free slots except two: d1, Q's favourite domain, with 8, and d2 with 4.  Their extra rows
    carry the same priority, so the row index decides between them: with P first in the concatenation P takes d1 and
    Q moves to d2; with Q first Q takes d1 and P, which fits nowhere else, strands.  → (world, rows, ns, recs)."""
    w, _ = waves_world()
    w.nodes = w.nodes.copy()
    dom = w.nodes["domain_id"].astype(np.int64)
    occ = w.occ.astype(np.int64)
    rp, rq = 1, 3
    g = int(w.lws["group_count"][rp])
    uid_p = 0x1234567
    pr, _ = _mix(uid_p, g)
    uid_q = _unmix_priority(pr, g)
    assert _mix(uid_q, g)[0] == pr
    key_q = _mix(uid_q, g)[1]
    order = sorted(range(int(w.n_domains)), key=lambda d: (-_score(key_q, d), d))
    d1, d2 = order[0], order[1]
    cap = occ.copy()
    for d in range(int(w.n_domains)):
        on = np.flatnonzero(dom == d)
        want = 8 if d == d1 else 4 if d == d2 else 3
        cap[on] = occ[on]
        cap[on[0]] += want - (len(on) - 1)
        cap[on[1:]] += 1
    w.nodes["capacity"] = cap.astype(w.nodes["capacity"].dtype)
    recs = R.aligned_empty(2, R.LWS_REC)
    recs[0] = _prop(w, rp, uid_hash=uid_p, size=int(w.lws["size"][rp]), replicas=g + 1)
    recs[1] = _prop(w, rq, uid_hash=uid_q, replicas=g + 1)
    # P is size 8: a resident object of that size, its proposal keeps its size
    w.lws = w.lws.copy()
    w.lws["size"][rp] = 8
    recs[0]["size"] = 8
    return w, np.array([rp, rq], np.uint32), np.array([5, 5], np.uint32), recs
