"""Placement explanation (lwse_resident_place_explain) by its definition (lwse.h, "placement explanation"), without a
GPU: the round from the spec oracle (``oracle.place`` for the baseline, ``test_place_whatif.whatif_ref`` for a what-if
round), then the per-domain class table stated in its order for every explained row.

``variant`` names a wrong statement the tests show to be caught: ``"held_before_fit"`` (the held classes tested before
no_usable / too_small), ``"later_blocks"`` (a holder with a larger key counted as held ahead) and
``"capacity_not_free"`` (dom_free from node capacities, occupancy ignored).

Worlds are ``types.SimpleNamespace`` objects with nodes, occ, n_domains, reqs and n_ns."""
from __future__ import annotations

import types

import numpy as np

import oracle
from lws_b200 import records as R
from test_place_whatif import apply_segments, whatif_ref

M32 = 0xFFFFFFFF
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
OWN, NO_USABLE, TOO_SMALL, HELD_PINNED, HELD_EARLIER, HELD_LATER, OPEN = range(7)
# (a tie of the level-1 hash: key_lo, d1 < d2 with hi(key_lo, d1) == hi(key_lo, d2); tests/golden/find_place_ties.py)
TIE = (0x5DD5FF0E, 24, 56)


def mix32(x):
    x = np.asarray(x, dtype=np.uint64) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85EBCA6B)) & np.uint64(M32)
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xC2B2AE35)) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return x


def hi_of(key_lo, d):
    """The spec's level-1 hash of domains ``d`` for a request whose group key's low word is ``key_lo``."""
    d = np.asarray(d, dtype=np.uint64)
    return mix32(np.uint64(key_lo) ^ ((d * np.uint64(0x9E3779B1)) & np.uint64(M32))) | np.uint64(1)


def spec_keys(reqs):
    """The spec's key of every request row."""
    rows = np.arange(len(reqs), dtype=np.uint64)
    pinned = reqs["leader_node"] != R.NONE
    prio = (reqs["priority"].astype(np.uint64) >> np.uint64(25)) & np.uint64(0x7FFFFFFFFF)
    return (np.where(pinned, np.uint64(0), np.uint64(1)) << np.uint64(63)) | (prio << np.uint64(24)) | (rows & np.uint64(0xFFFFFF))


def domain_stats(nodes, occ, n_domains, variant=None):
    """dom_free, usable and free_all per domain (uint32 sums, as the spec's)."""
    flags = nodes["flags"].astype(np.int64)
    dom = nodes["domain_id"].astype(np.int64)
    labelled = ((flags & R.NODE_HAS_TOPOLOGY) != 0) & (dom < n_domains)
    sched = (flags & R.NODE_SCHEDULABLE) != 0
    cap = nodes["capacity"].astype(np.int64)
    o = np.zeros(len(nodes), np.int64) if occ is None else np.asarray(occ, dtype=np.int64)[: len(nodes)]
    fr = cap if variant == "capacity_not_free" else np.maximum(cap - o, 0)
    use = labelled & sched
    dom_free = np.bincount(dom[use], weights=fr[use], minlength=n_domains).astype(np.int64) % (1 << 32)
    usable = np.bincount(dom[use], minlength=n_domains).astype(np.int64)
    free_all = np.bincount(dom[labelled], weights=fr[labelled], minlength=n_domains).astype(np.int64) % (1 << 32)
    return dom_free, usable, free_all


def holders(reqs, out, n_ns, n_domains):
    """{namespace: [n_domains] the holder's key, EMPTY where nobody holds}; at most one PLACED row per (ns, d)."""
    keys = spec_keys(reqs)
    hold = {}
    placed = np.flatnonzero(((out["flags"] & R.PLACE_PLACED) != 0) & (reqs["ns"] < n_ns))
    for i in placed.tolist():
        v, d = int(reqs["ns"][i]), int(out["domain_id"][i])
        h = hold.setdefault(v, np.full(n_domains, EMPTY, dtype=np.uint64))
        assert h[d] == EMPTY, f"(ns {v}, domain {d}) has two holders"
        h[d] = keys[i]
    return hold


def round_of(w, segs=(), extra=None, n_ns=0):
    """The round explained → (nodes, reqs, out, n_ns, whatif)."""
    extra = R.aligned_empty(0, R.PLACE_REQ) if extra is None else extra
    if not len(segs) and not len(extra) and n_ns in (0, w.n_ns):
        return w.nodes, w.reqs, oracle.place(w.nodes, w.occ, w.n_domains, w.n_ns, w.reqs, threads=8), w.n_ns, False
    n_ns = n_ns or w.n_ns
    after = whatif_ref(w.nodes, w.occ, w.n_domains, w.reqs, segs, extra, n_ns=n_ns, base_n_ns=w.n_ns, threads=8)["after_all"]
    nodes, reqs = apply_segments(w.nodes, w.reqs, segs)
    all_reqs = R.aligned_empty(len(reqs) + len(extra), R.PLACE_REQ)
    all_reqs[: len(reqs)] = reqs
    all_reqs[len(reqs):] = extra
    return nodes, all_reqs, after, n_ns, True


def explain_row(r, nodes, reqs, out, n_ns, n_domains, stats, hold, keys, variant=None):
    """One PLACE_EXPLAIN row by the table of lwse.h."""
    row = np.zeros(1, R.PLACE_EXPLAIN)[0]
    row["row"], row["place_flags"] = r, out["flags"][r]
    for f in ("best_domain", "blocker_domain", "blocker_row", "shortfall_domain"):
        row[f] = R.NONE
    q = reqs[r]
    if int(q["ns"]) >= n_ns:
        row["flags"] = R.PEX_NO_NAMESPACE
        return row
    dom_free, usable, free_all = stats
    d = np.arange(n_domains, dtype=np.int64)
    s = int(q["size"])
    k = keys[r]
    pinned = int(q["leader_node"]) != R.NONE
    own = int(out["domain_id"][r]) if out["flags"][r] & R.PLACE_PLACED else -1
    hk = hold.get(int(q["ns"]), np.full(n_domains, EMPTY, dtype=np.uint64))
    held = hk != EMPTY
    ahead = held & (hk < k)
    if variant == "later_blocks":
        ahead = held
    by_pin = (hk >> np.uint64(63)) == 0
    fits = (usable > 0) & (dom_free >= s)
    conds = [d == own, usable == 0, dom_free < s, ahead & by_pin, ahead & ~by_pin, held & ~ahead, ~held]
    if variant == "held_before_fit":
        conds = [d == own, ahead & by_pin, ahead & ~by_pin, held & ~ahead, usable == 0, dom_free < s, ~held]
        cls = np.select(conds, [OWN, HELD_PINNED, HELD_EARLIER, HELD_LATER, NO_USABLE, TOO_SMALL, OPEN], -1)
    else:
        cls = np.select(conds, [OWN, NO_USABLE, TOO_SMALL, HELD_PINNED, HELD_EARLIER, HELD_LATER, OPEN], -1)
    assert (cls >= 0).all()
    for c, f in enumerate(R.PLACE_EXPLAIN_CLASSES[:7]):
        row[f] = int((cls == c).sum())
    row["n_fit_uncordoned"] = int((((cls == NO_USABLE) | (cls == TOO_SMALL)) & (free_all >= s)).sum())
    hi = hi_of(int(q["group_key"]) & M32, d).astype(np.int64)

    def argmax_in(mask):
        return int(np.argmax(np.where(mask, hi, -1))) if mask.any() else None  # (first maximum: the lower domain)

    b = argmax_in((cls == OWN) | (cls == HELD_LATER) | (cls == OPEN))
    if b is not None:
        row["best_domain"] = b
    b = argmax_in((cls == HELD_PINNED) | (cls == HELD_EARLIER))
    if b is not None:
        row["blocker_domain"], row["blocker_row"] = b, int(hk[b]) & 0xFFFFFF
    small = cls == TOO_SMALL
    if small.any():
        gap = np.where(small, s - dom_free, np.iinfo(np.int64).max)
        b = int(np.argmin(gap))
        row["shortfall"], row["shortfall_domain"] = int(gap[b]), b
    flags = 0
    n_fit = int(fits.sum())
    if n_fit == 0:
        flags |= R.PEX_CAPACITY
    if n_fit > 0 and int(row["n_held_pinned"]) + int(row["n_held_earlier"]) == n_fit:
        flags |= R.PEX_EXCLUSIVE
    if row["n_fit_uncordoned"] > 0:
        flags |= R.PEX_CORDONED
    if not pinned and s < 1:
        flags |= R.PEX_BAD_SIZE
    if pinned:
        ln = int(q["leader_node"])
        ld = None
        if ln < len(nodes):
            nd = nodes[ln]
            if (int(nd["flags"]) & R.NODE_HAS_TOPOLOGY) and int(nd["domain_id"]) < n_domains:
                ld = int(nd["domain_id"])
        if ld is None:
            flags |= R.PEX_NO_CLAIM
        elif hk[ld] != EMPTY and hk[ld] < k and (hk[ld] >> np.uint64(63)) == 0:
            flags |= R.PEX_CONFLICT
            row["blocker_domain"], row["blocker_row"] = ld, int(hk[ld]) & 0xFFFFFF
    row["flags"] = flags
    return row


def explain_ref(w, rows=None, mask=R.PLACE_UNSCHEDULABLE | R.PLACE_CONFLICT, segs=(), extra=None, n_ns=0, capacity=None,
                variant=None):
    """The answer of ``Engine.resident_place_explain`` with the same arguments (its dict, without ``form``)."""
    nodes, reqs, out, n_ns, whatif = round_of(w, segs, extra, n_ns)
    if rows is None:
        sel = np.flatnonzero((out["flags"] & np.uint32(mask)) != 0)
    else:
        sel = np.asarray(rows, dtype=np.int64)
        assert (sel < len(reqs)).all()
    stats = domain_stats(nodes, w.occ, w.n_domains, variant)
    marked = set(int(v) for v in reqs["ns"][sel])
    hold = {v: h for v, h in holders(reqs, out, n_ns, w.n_domains).items() if v in marked}
    keys = spec_keys(reqs)
    got = R.aligned_empty(len(sel), R.PLACE_EXPLAIN)
    for j, r in enumerate(sel.tolist()):
        got[j] = explain_row(r, nodes, reqs, out, n_ns, w.n_domains, stats, hold, keys, variant)
    cap = len(sel) if capacity is None else capacity
    return {"rows": got[:cap], "all_rows": got, "round": out, "reqs": reqs, "nodes": nodes, "n_explained": len(sel),
            "round_rows": len(reqs), "n_domains": w.n_domains, "whatif": whatif,
            "classes": {f: int(got[f].astype(np.int64).sum()) for f in R.PLACE_EXPLAIN_CLASSES},
            "flags": {name: int(((got["flags"] & b) != 0).sum()) for b, name in R.PEX_NAMES.items()}}


def certificate(ans, n_ns, n_domains):
    """The serial-order certificate over the explained rows of a round → list of violations (empty when it holds)."""
    bad = []
    out, reqs = ans["round"], ans["reqs"]
    keys = spec_keys(reqs)
    for e in ans["all_rows"]:
        r = int(e["row"])
        q, o = reqs[r], out[r]
        if int(q["ns"]) >= n_ns:
            continue
        cls = sum(int(e[f]) for f in R.PLACE_EXPLAIN_CLASSES[:7])
        if cls != n_domains:
            bad.append((r, "classes do not sum to n_domains"))
        unpinned = int(q["leader_node"]) == R.NONE
        if unpinned and o["flags"] & R.PLACE_UNSCHEDULABLE and int(q["size"]) >= 1:
            if int(e["n_open"]) + int(e["n_held_later"]) != 0 or int(e["best_domain"]) != R.NONE:
                bad.append((r, "unschedulable with an open domain"))
        if unpinned and o["flags"] & R.PLACE_PLACED:
            if int(e["best_domain"]) != int(o["domain_id"]):
                bad.append((r, "placed outside its best domain"))
            elif int(hi_of(int(q["group_key"]) & M32, int(e["best_domain"]))) != int(o["score"]):
                bad.append((r, "score is not the best domain's hash"))
        if e["flags"] & R.PEX_CONFLICT:
            b = int(e["blocker_row"])
            ln = int(q["leader_node"])
            if not (out[b]["flags"] & R.PLACE_PLACED and int(out[b]["domain_id"]) == int(e["blocker_domain"])
                    and int(ans["nodes"]["domain_id"][ln]) == int(e["blocker_domain"])
                    and int(reqs[b]["leader_node"]) != R.NONE and int(reqs[b]["ns"]) == int(q["ns"])
                    and keys[b] < keys[r]):
                bad.append((r, "conflict without a smaller pinned holder of its leader's domain"))
    return bad


# --------------------------------------------------------------------------- #
# the edge world
# --------------------------------------------------------------------------- #
def _req(ns, size, prio, key=None, leader=R.NONE, group=0):
    x = np.zeros(1, R.PLACE_REQ)[0]
    x["priority"] = np.uint64(prio) << np.uint64(25)
    x["group_key"] = key if key is not None else (0x9E3779B97F4A7C15 * (group + 7)) & 0xFFFFFFFFFFFFFFFF
    x["group"], x["ns"], x["size"], x["leader_node"] = group, ns, size, leader
    return x


def edge_world(n_domains=64):
    """One case per edge, on 64 domains of two nodes each (nodes 2d, 2d + 1), capacity 1 each unless named:
    domain 1 has dom_free 5 (= s for the size-5 rows), 2 has 4 (s − 1), 3 has 4 with a cordoned node of 4 beside it
    (free_all 8), 4 has both nodes cordoned (no usable node, free_all 8), 5 has a node with occupancy 9 above its
    capacity 2 next to a node of 8, 24 and 56 (the tie pair of TIE) have 16 each; node 128 is unlabelled and node 129
    labelled beyond the domains.  Namespace 0: two size-9 rows of key TIE (only 24 and 56 fit): the first takes 24 by
    the tie.  Namespace 1: two high-priority size-9 rows take 24 and 56; a TIE row is left with a tied blocker.
    Namespace 2: pinned P1 holds 1 and P2 conflicts with it, three unpinned rows take 5, 24 and 56, F5 is left
    EXCLUSIVE and CORDONED, then NO_CLAIM leaders (missing, unlabelled, out of range) and sizes 0 and −3.
    Namespace 3: a pinned row on a cordoned node of 4 (PLACED: pinned claims ignore capacity) and one on 5, an
    unpinned row of higher priority and one of lower, and a size-17 row no domain fits.  One row of namespace 7 (the world has 4).
    → (world, {name: row})."""
    K, d1, d2 = TIE
    nodes = R.aligned_empty(130, R.NODE_REC)
    nodes["topo_value_hash"] = 0
    nodes["domain_id"] = np.arange(130) // 2
    nodes["capacity"] = 1
    nodes["flags"] = R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE
    occ = np.zeros(130, np.uint32)
    nodes["capacity"][2], nodes["capacity"][3] = 3, 2          # domain 1: 5
    nodes["capacity"][4], nodes["capacity"][5] = 2, 2          # domain 2: 4
    nodes["capacity"][6], nodes["capacity"][7] = 4, 4          # domain 3: 4 + a cordoned 4
    nodes["flags"][7] = R.NODE_HAS_TOPOLOGY
    nodes["capacity"][8], nodes["capacity"][9] = 4, 4          # domain 4: all cordoned
    nodes["flags"][8] = nodes["flags"][9] = R.NODE_HAS_TOPOLOGY
    nodes["capacity"][10], nodes["capacity"][11] = 2, 8        # domain 5: occupancy above capacity, then 8
    occ[10] = 9
    for d in (d1, d2):
        nodes["capacity"][2 * d] = nodes["capacity"][2 * d + 1] = 8
    nodes["domain_id"][128], nodes["flags"][128], nodes["capacity"][128] = 5, R.NODE_SCHEDULABLE, 50
    nodes["domain_id"][129], nodes["capacity"][129] = 99, 50
    rows, reqs = {}, []

    def add(name, x):
        rows[name] = len(reqs)
        reqs.append(x)

    add("T0", _req(0, 9, 10, key=K, group=1))
    add("T1", _req(0, 9, 11, key=K, group=2))
    add("H1", _req(1, 9, 1, group=3))
    add("H2", _req(1, 9, 2, group=4))
    add("B", _req(1, 9, 20, key=K, group=5))
    add("P1", _req(2, 5, 30, leader=2, group=6))
    add("P2", _req(2, 5, 31, leader=3, group=7))
    add("U1", _req(2, 5, 1, group=8))
    add("U2", _req(2, 5, 2, group=9))
    add("U3", _req(2, 5, 3, group=10))
    add("F5", _req(2, 5, 9, group=11))
    add("NC_MISSING", _req(2, 5, 40, leader=R.NODE_NOT_FOUND, group=12))
    add("NC_UNLABELLED", _req(2, 5, 41, leader=128, group=13))
    add("NC_RANGE", _req(2, 5, 42, leader=129, group=14))
    add("Z0", _req(2, 0, 5, group=15))
    add("ZN", _req(2, -3, 5, group=16))
    add("PC", _req(3, 5, 50, leader=9, group=17))
    add("P5", _req(3, 5, 51, leader=11, group=18))
    add("E1", _req(3, 5, 1, group=19))
    add("Q", _req(3, 5, 60, group=20))
    add("CAP", _req(3, 17, 61, group=22))
    add("NS", _req(7, 5, 1, group=21))
    t = R.aligned_empty(len(reqs), R.PLACE_REQ)
    for i, x in enumerate(reqs):
        t[i] = x
    return types.SimpleNamespace(nodes=nodes, occ=occ, n_domains=n_domains, reqs=t, n_ns=4), rows


def cordon_seg(nodes, node_rows, cordon):
    """A NODES segment that cordons (or uncordons) ``node_rows``."""
    rows = np.asarray(sorted(node_rows), dtype=np.uint32)
    vals = R.aligned_empty(len(rows), R.NODE_REC)
    vals[:] = nodes[rows]
    if cordon:
        vals["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
    else:
        vals["flags"] |= np.uint16(R.NODE_SCHEDULABLE)
    return (R.TABLE_NODES, rows, vals)


def extra_reqs(specs):
    """Extra request rows from (ns, size, priority rank) triples."""
    x = R.aligned_empty(len(specs), R.PLACE_REQ)
    for i, (ns, size, prio) in enumerate(specs):
        x[i] = _req(ns, size, prio, group=100 + i)
    return x


def pods_for(occ):
    """Identity and state rows whose scheduled pods give ``occ`` per node (the resident tables count them)."""
    node = np.repeat(np.arange(len(occ), dtype=np.uint64), np.asarray(occ).astype(np.int64))
    pid = R.pod_ident_table(np.arange(len(node), dtype=np.uint64), np.zeros(len(node), np.uint32),
                            (R.PODID_SCHEDULED | (node << np.uint64(R.PODID_NODE_SHIFT))).astype(np.uint32))
    pst = R.aligned_empty(len(node), R.POD_STATE)
    pst[:] = 0
    return pst, pid


def fuzz_world(seed, n_nodes=400, n_domains=40, n_ns=5, n_reqs=600):
    """Random nodes (some cordoned, unlabelled or beyond the domains, occupancy up to above capacity) and requests
    (pinned on random nodes, missing ones included, sizes −1 .. 12, some namespaces beyond n_ns)."""
    rng = np.random.default_rng(seed)
    nodes = R.aligned_empty(n_nodes, R.NODE_REC)
    nodes["topo_value_hash"] = 0
    nodes["domain_id"] = rng.integers(0, n_domains + 2, n_nodes)
    nodes["capacity"] = rng.integers(0, 8, n_nodes)
    f = np.full(n_nodes, R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE)
    f[rng.random(n_nodes) < 0.1] &= ~R.NODE_SCHEDULABLE
    f[rng.random(n_nodes) < 0.05] &= ~R.NODE_HAS_TOPOLOGY
    nodes["flags"] = f
    occ = rng.integers(0, 9, n_nodes).astype(np.uint32)
    reqs = R.aligned_empty(n_reqs, R.PLACE_REQ)
    reqs["priority"] = rng.integers(0, 1 << 40, n_reqs, dtype=np.uint64)
    reqs["priority"][rng.random(n_reqs) < 0.2] = np.uint64(5) << np.uint64(25)  # key ties broken by the row
    reqs["group_key"] = rng.integers(0, 1 << 63, n_reqs, dtype=np.uint64)
    reqs["group"] = np.arange(n_reqs)
    reqs["ns"] = np.where(rng.random(n_reqs) < 0.03, n_ns + 1, rng.integers(0, n_ns, n_reqs))
    reqs["size"] = rng.integers(-1, 13, n_reqs)
    lead = rng.integers(0, n_nodes + 3, n_reqs).astype(np.uint32)
    lead[lead >= n_nodes] = R.NODE_NOT_FOUND
    reqs["leader_node"] = np.where(rng.random(n_reqs) < 0.3, lead, R.NONE)
    return types.SimpleNamespace(nodes=nodes, occ=occ, n_domains=n_domains, reqs=reqs, n_ns=n_ns)
