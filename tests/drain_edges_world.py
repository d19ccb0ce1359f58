"""Tables built to land on the edges of the drain kernels (``lws_b200/csrc/lwse_drain_kernels.cu``).

The drain cost and both passes of the per-key drain budget walk a group's pods 32 at a time (one warp,
``__match_any_sync`` per batch) and remember the group's distinct restart keys — the node, or its domain —
in a per-warp list of ``kCostList`` entries.  A batch whose fresh keys would not fit turns the list off for
the rest of the group, and from then on every batch re-reads all earlier batches instead ("slower, still
exact").  A batch adds at most 32 keys, so the earliest batch that can overflow the list is the third.
The set-form budget kernel strides over an LWS row's group range 32 groups at a time; the (LWS, key) table
of the per-key budget is open-addressed with linear probing from ``table_slot``; every kernel's grid is
capped at a multiple of the SM count and strides beyond it.

Every builder here lands exactly on its label, and the constants the labels depend on are restated
below (``tests/test_drain_edges.py`` reads them back from the sources).  Every table is small enough for
the spec oracle except the grid worlds, which are sized from the SM count of the device under test.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from lws_b200 import records as R

# the drain kernels' constants (lwse_drain_kernels.cu)
K_COST_THREADS = 256      # threads per CTA of drain_cost_kernel and drain_budget_walk_kernel
K_COST_LIST = 64          # distinct restart keys one warp remembers per group
WARP = 32
GRID_CAP = {              # CTAs per SM at most, per kernel (launch_drain_*)
    "drain_mark_kernel": 16, "drain_diff_kernel": 4, "drain_domain_mask_kernel": 4,
    "drain_cost_kernel": 8, "drain_budget_walk_kernel": 8, "drain_budget_kernel": 8,
}
GRID_THREADS = 256        # threads per CTA of the mark, diff, domain mask and budget kernels
# the (LWS, key) table (lwse_engine.cu): 256 slots, or the next power of two >= 2 x pairs
TABLE_MIN_SLOTS = 256
TABLE_PAIRS_FACTOR = 2
MIXER = 0xFF51AFD7ED558CCD  # table_slot's multiplier
H100_SMS = 132

I32_MAX = (1 << 31) - 1
M64 = (1 << 64) - 1
NONE = -1
REV = 0x5EED_0000_0000_0001
ON, AFTER, OFF = R.RESTART_ON_POD_RESTART, R.RESTART_AFTER_START, R.RESTART_NONE
GOOD_GROUP = (R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH | R.GRP_POD_RUNNING | R.GRP_POD_READY
              | R.GRP_WSTS_LABEL_NAME_MATCH | R.GRP_WSTS_FOUND | R.GRP_WSTS_REV_SETTLED | R.GRP_WSTS_OWNER_IS_POD
              | R.GRP_WSTS_OWNER_NAME_MATCH | R.GRP_REVISION_EXISTS)
# pods that fail the restart verdict (key NONE): not scheduled, scheduled on node n_nodes or on the largest
# node number the identity row holds, a name that does not parse, a worker of another StatefulSet
FAILS = ("unsched", "n_nodes", "node_max", "name", "foreign")


# --------------------------------------------------------------------------- #
# the table's slot and table size, restated
# --------------------------------------------------------------------------- #
def table_slot(key: int, mask: int) -> int:
    k = key & M64
    k ^= k >> 33
    k = (k * MIXER) & M64
    k ^= k >> 33
    return k & 0xFFFFFFFF & mask


def table_slots(pairs: int) -> int:
    slots = TABLE_MIN_SLOTS
    while slots < TABLE_PAIRS_FACTOR * pairs:
        slots <<= 1
    return slots


def probe_layout(entries, mask: int) -> dict:
    """Linear probing of ``entries`` (LWS << 32 | key) in insertion order → {entry: (home, slot)}; the
    kernel inserts in an unspecified order, so only what holds for every order is checked against this."""
    taken, out = {}, {}
    for e in entries:
        h = table_slot(e, mask)
        s = h
        while s in taken:
            s = (s + 1) & mask
        taken[s] = e
        out[e] = (h, s)
    return out


# --------------------------------------------------------------------------- #
# the warp walk, restated
# --------------------------------------------------------------------------- #
@dataclass
class Walk:
    fresh: list          # the keys the walk adds a pair for, in walk order
    overflow: int | None  # the batch whose fresh keys overflowed the list, None = the list held them all
    listed: int          # entries in the list at the end (or when it was turned off)


def warp_walk(keys) -> Walk:
    """One group's walk over its per-pod keys (NONE for a pod that fails the verdict): batch, match_any
    (the lowest lane of a key is its representative), the list, and after an overflow the re-read of every
    earlier batch."""
    keys = list(keys)
    lst, listed, overflow, fresh_all = [], True, None, []
    for b0 in range(0, len(keys), WARP):
        batch = keys[b0:b0 + WARP]
        fresh = [k != NONE and batch.index(k) == i for i, k in enumerate(batch)]
        if listed:
            fresh = [f and k not in lst for f, k in zip(fresh, batch)]
            add = [k for f, k in zip(fresh, batch) if f]
            if len(lst) + len(add) <= K_COST_LIST:
                lst += add
            else:
                listed, overflow = False, b0 // WARP
        if not listed:
            earlier = set(keys[:b0])
            fresh = [f and k not in earlier for f, k in zip(fresh, batch)]
        fresh_all += [k for f, k in zip(fresh, batch) if f]
    return Walk(fresh_all, overflow, len(lst))


# --------------------------------------------------------------------------- #
# a table builder
# --------------------------------------------------------------------------- #
@dataclass
class EdgeWorld:
    label: str
    lws: np.ndarray
    groups: np.ndarray
    pod_state: np.ndarray
    pod_ident: np.ndarray
    nodes: np.ndarray
    n_domains: int
    flags: int = 0
    notes: dict = field(default_factory=dict)  # label -> group rows / LWS rows / keys the label names


class Builder:
    """Objects, their groups and the groups' pods.  A group's first pod is its leader; a worker is a node
    row (it passes the verdict and is scheduled there) or one of FAILS; ``pending`` names pod positions
    whose phase is Pending.  Objects own consecutive group ranges in the order they are created."""

    def __init__(self, nodes: np.ndarray, n_domains: int):
        self.nodes, self.n_domains = nodes, n_domains
        self.objs, self.grps, self.pods = [], [], []

    def obj(self, policy=ON, size=None, annot=False, replicas=None, mu=0, pct=False) -> int:
        self.objs.append(dict(policy=policy, size=size, annot=annot, replicas=replicas, mu=mu, pct=pct, groups=[]))
        return len(self.objs) - 1

    def group(self, o: int, workers, leader=0, pending=(), ready=True, rev=REV) -> int:
        gi = len(self.grps)
        base = len(self.pods)
        luid, wuid = 0x1000_0000 + gi, 0x2000_0000 + gi
        run, pend = R.POD_PHASE_RUNNING, R.POD_PHASE_PENDING
        sts = R.POD_OWNER_STS << R.POD_OWNER_SHIFT
        self.pods.append([run | R.POD_IS_LEADER | sts, rev, 9, self._place(leader)])
        for w in workers:
            st = run | sts | R.POD_OWNER_NAME_MATCH
            if isinstance(w, str):
                place = {"unsched": R.PODID_NAME_OK, "n_nodes": self._place(len(self.nodes)),
                         "node_max": self._place(R.POD_NODE_MAX), "name": self._place(0) & ~R.PODID_NAME_OK,
                         "foreign": self._place(0)}[w]
                self.pods.append([st, rev, wuid ^ 0xFF if w == "foreign" else wuid, place])
            else:
                self.pods.append([st, rev, wuid, self._place(int(w))])
        for p in pending:
            self.pods[base + p][0] = (self.pods[base + p][0] & ~R.POD_PHASE_MASK) | pend
        n = len(self.pods) - base
        self.grps.append(dict(o=o, base=base, count=n, luid=luid, wuid=wuid, leader=leader, rev=rev,
                              flags=GOOD_GROUP if ready else GOOD_GROUP & ~R.GRP_POD_READY, workers=n - 1))
        self.objs[o]["groups"].append(gi)
        return gi

    @staticmethod
    def _place(node) -> int:
        return R.PODID_NAME_OK | R.PODID_SCHEDULED | (int(node) << R.PODID_NODE_SHIFT)

    def tables(self, label: str, flags: int = 0) -> EdgeWorld:
        L, G, P = len(self.objs), len(self.grps), len(self.pods)
        lws = R.aligned_empty(L, R.LWS_REC)
        gb = 0
        for i, o in enumerate(self.objs):
            gs = o["groups"]
            assert gs == list(range(gb, gb + len(gs))), "an object's groups are created together"
            gc = len(gs)
            size = o["size"] if o["size"] is not None else (self.grps[gs[0]]["count"] if gs else 1)
            reps = o["replicas"] if o["replicas"] is not None else gc
            lws[i]["rev_hash"] = REV
            lws[i]["size"] = size
            lws[i]["flags"] = (R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID | (o["policy"] << R.LWS_RESTART_SHIFT)
                               | (R.LWS_RECREATE_AFTER_START_ANNOT if o["annot"] else 0)
                               | (R.LWS_UNAVAIL_IS_PERCENT if o["pct"] else 0))
            lws[i]["replicas"] = reps
            lws[i]["max_unavailable"] = o["mu"]
            lws[i]["sts_replicas"] = lws[i]["sts_replicas_annotation"] = reps
            lws[i]["uid_hash"] = 0x7000 + i
            lws[i]["group_base"], lws[i]["group_count"] = gb, gc
            gb += gc
        g = R.aligned_empty(G, R.GROUP_REC)
        for i, d in enumerate(self.grps):
            g[i]["leader_rev_hash"] = g[i]["wsts_rev_hash"] = d["rev"]
            g[i]["wsts_spec_replicas"] = g[i]["wsts_avail_replicas"] = d["workers"]
            g[i]["leader_uid_hash"], g[i]["wsts_uid_hash"] = d["luid"], d["wuid"]
            g[i]["wsts_owner_uid_hash"] = d["luid"]
            g[i]["leader_node"] = d["leader"]
            g[i]["pod_base"], g[i]["pod_count"], g[i]["lws_index"] = d["base"], d["count"], d["o"]
            g[i]["flags"] = d["flags"]
        pst = R.aligned_empty(P, R.POD_STATE)
        pst[:] = [p[0] for p in self.pods]
        pid = R.pod_ident_table(np.array([p[1] for p in self.pods], np.uint64),
                                np.array([p[2] for p in self.pods], np.uint32),
                                np.array([p[3] for p in self.pods], np.uint32))
        return EdgeWorld(label, lws, g, pst, pid, self.nodes, self.n_domains, flags)


def node_table(n_nodes: int, per_domain: int, no_domain=(), beyond=()) -> tuple[np.ndarray, int]:
    """Nodes in domains of ``per_domain``; ``no_domain`` rows get LWSE_NONE, ``beyond`` rows an id past the
    last domain.  → (nodes, n_domains)."""
    nodes = R.aligned_empty(n_nodes, R.NODE_REC)
    dom = np.arange(n_nodes, dtype=np.int64) // per_domain
    special = np.zeros(n_nodes, bool)
    special[list(no_domain) + list(beyond)] = True
    n_domains = int(dom[~special].max()) + 1 if (~special).any() else 0
    dom[list(no_domain)] = R.NONE
    dom[list(beyond)] = n_domains + 3
    nodes["domain_id"] = dom.astype(np.uint32)
    nodes["topo_value_hash"] = (dom.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(1)
    nodes["capacity"] = 64
    nodes["flags"] = R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE
    return nodes, n_domains


# --------------------------------------------------------------------------- #
# 1. walk edges
# --------------------------------------------------------------------------- #
WALK_NODES, WALK_PER_DOMAIN = 4096, 4
WALK_NO_DOMAIN = tuple(range(4088, 4092))   # domain_id LWSE_NONE
WALK_BEYOND = tuple(range(4092, 4096))      # domain_id >= n_domains
WALK_POD_COUNTS = (1, 31, 32, 33, 63, 64, 65, 96, 97, 5003)
PENDING_AT = (0, 31, 32, 33, 64)            # positions of the only pending pod in a 65-pod group


def walk_world(seed: int = 7) -> EdgeWorld:
    rng = np.random.Generator(np.random.PCG64(seed))
    nodes, n_domains = node_table(WALK_NODES, WALK_PER_DOMAIN, WALK_NO_DOMAIN, WALK_BEYOND)
    b = Builder(nodes, n_domains)
    notes: dict = {}
    pool = np.arange(4088)

    def spread(n, k):
        """n workers over k distinct nodes (each used at least once, order shuffled)."""
        ns = rng.choice(pool, size=k, replace=False)
        w = np.concatenate([ns, rng.choice(ns, size=max(n - k, 0))])[:n]
        rng.shuffle(w)
        return [int(x) for x in w]

    # pod counts: workers on few nodes (duplicates in every batch), a failing pod every 7th position
    o = b.obj(ON)
    notes["counts"] = []
    for c in WALK_POD_COUNTS:
        w = spread(c - 1, min(24, max(c - 1, 1)) if c < 5000 else 4000)
        for i in range(5, len(w), 7):
            w[i] = FAILS[(i // 7) % len(FAILS)]
        notes["counts"].append(b.group(o, w, leader=int(rng.integers(0, 4088))))
    # distinct restart nodes 63 / 64 / 65 through the list's edge; overflow in the third batch (the
    # earliest possible) and in the seventh
    fresh_nodes = iter(rng.permutation(pool).tolist())
    take = lambda k: [next(fresh_nodes) for _ in range(k)]
    o = b.obj(ON)
    a = take(63)  # leader + 62 workers in two batches, then repeats
    notes["distinct_63"] = b.group(o, a[1:] + a[:33], leader=a[0])
    a = take(64)
    notes["distinct_64"] = b.group(o, a[1:] + a[5:38], leader=a[0])
    a = take(65)
    # batch 0: 32 new, batch 1: 32 new, batch 2: list keys with one new key (the 65th) twice, then a
    # fourth batch repeating keys of the list and of the overflowing batch
    b2 = [a[3], a[40], a[64], a[3], "unsched", a[64], a[10]] + a[11:36]
    notes["distinct_65_early"] = b.group(o, a[1:64] + b2 + [a[64], a[40], "name", a[64], a[2]], leader=a[0])
    # overflow in batch 6: batches 0-5 add 10 keys each (60), batch 6 adds 5 beside list keys; batch 7 brings
    # keys never seen, batches 8-9 repeat keys of the list, of batch 6 and of batch 7
    a = take(72)
    pods = []
    for k in range(6):
        new = a[10 * k: 10 * k + 10]
        batch = new + [new[j % 10] for j in range(11)] + [a[(7 * j) % (10 * k + 10)] for j in range(11)]
        pods += batch
    b6 = a[60:65] + [a[j] for j in range(0, 54, 2)]
    b7 = a[65:72] + [a[61], a[62]] + [a[j] for j in range(3, 26)]
    b8 = [a[66], a[60], a[1], a[70], "foreign", a[64], a[71]] + [a[j] for j in range(30, 55)]
    pods += b6 + b7 + b8 + [a[65], a[63], a[2], "n_nodes", a[69]]
    notes["distinct_late"] = b.group(o, pods[1:], leader=pods[0])
    # duplicates inside one batch, split across lanes by pods of every failing kind
    x, y = take(2)
    w = [x, "unsched", y, "n_nodes", x, "node_max", y, "name", x, "foreign"] * 3
    notes["dup_in_batch"] = b.group(o, w + [y], leader=x)
    # DOMAINS scope: 64 and 65 distinct domains through two nodes each, nodes of no domain in between
    doms = rng.permutation(n_domains)[:129].tolist()
    for name, k in (("domains_64", 64), ("domains_65", 65)):
        ds = doms[:k] if k == 64 else doms[64:129]
        w = []
        for i, d in enumerate(ds):
            w += [d * WALK_PER_DOMAIN + 1, WALK_NO_DOMAIN[i % 4], d * WALK_PER_DOMAIN + 2, WALK_BEYOND[i % 4]]
        w += [ds[0] * WALK_PER_DOMAIN + 3, ds[-1] * WALK_PER_DOMAIN]
        notes[name] = b.group(o, w, leader=ds[0] * WALK_PER_DOMAIN)
    # the pending gate: the only pending pod at a chunk edge, for AfterStart and for the annotation, with
    # size == pod_count (the scan decides) and size != pod_count (pending without a scan); and controls
    notes["pending"] = {}
    for policy, annot in ((AFTER, False), (ON, True)):
        for size in (65, 66):
            o = b.obj(policy, size=size, annot=annot)
            for at in (None,) + PENDING_AT:
                g = b.group(o, spread(64, 40), leader=int(rng.integers(0, 4088)),
                            pending=() if at is None else (at,))
                notes["pending"][(policy, annot, size, at)] = g
    # groups whose pod ranges overlap: appended below by editing the rows (same identity: the shared pods
    # count for both groups; another identity: they count for the first only)
    o = b.obj(ON)
    shared = [b.group(o, spread(47, 30), leader=int(rng.integers(0, 4088))) for _ in range(4)]
    w = b.tables("walk")
    g = w.groups
    # group shared[1] takes over shared[0]'s identity and starts in its range; shared[3] starts in shared[2]'s
    for dst, src, shift in ((shared[1], shared[0], 20), (shared[3], shared[2], 33)):
        g[dst]["pod_base"] = g[src]["pod_base"] + shift
        g[dst]["pod_count"] = 48
    for f in ("leader_rev_hash", "wsts_rev_hash", "leader_uid_hash", "wsts_uid_hash", "wsts_owner_uid_hash"):
        g[shared[1]][f] = g[shared[0]][f]
    notes["overlap_same"], notes["overlap_other"] = (shared[0], shared[1]), (shared[2], shared[3])
    w.notes = notes
    return w


# --------------------------------------------------------------------------- #
# 2. budget edges
# --------------------------------------------------------------------------- #
BUDGET_ROW_GROUPS = (31, 32, 33, 64, 65, 1000)
# (replicas, maxUnavailable, percent) rows whose floor sits at an int32 edge
INT32_FLOORS = ((I32_MAX, 0, False), (I32_MAX, 100, True), (5, -3, False), (40, -50, True),
                (1 << 30, 300, True), ((1 << 30) + 7, 250, True), (I32_MAX, 101, True), (3, I32_MAX, False))
BUDGET_NODES = 96


def budget_edges_world(seed: int = 11) -> EdgeWorld:
    rng = np.random.Generator(np.random.PCG64(seed))
    nodes, n_domains = node_table(BUDGET_NODES, 4)
    b = Builder(nodes, n_domains)
    notes: dict = {"rows": {}}
    node = lambda: int(rng.integers(0, BUDGET_NODES))

    def groups(o, n, ready_p=0.9):
        return [b.group(o, [node() for _ in range(int(rng.integers(0, 3)))], leader=node(),
                        ready=bool(rng.random() < ready_p)) for _ in range(n)]

    for n in BUDGET_ROW_GROUPS:
        o = b.obj(ON, size=None, mu=int(rng.integers(0, 4)))
        gs = groups(o, n)
        notes["rows"][n] = o
    # surge groups: replicas = group_count - 3; the last group below replicas on node 0 alone, the first surge
    # group on node 1 alone
    o = b.obj(ON, size=1, mu=1, replicas=9)
    gs = [b.group(o, [], leader=i if i in (0, 1) else int(rng.integers(2, BUDGET_NODES))) for i in
          (2, 2, 2, 2, 2, 2, 2, 2, 0, 1, 2, 2)]
    notes["surge"] = (o, gs[8], gs[9])
    # replicas 0 and negative
    for reps in (0, -4):
        o = b.obj(ON, replicas=reps, mu=1)
        groups(o, 3)
        notes["rows"][f"replicas_{reps}"] = o
    # floors at the int32 edges
    notes["int32"] = []
    for reps, mu, pct in INT32_FLOORS:
        o = b.obj(ON, replicas=reps, mu=mu, pct=pct)
        groups(o, 3, ready_p=1.0)
        notes["int32"].append(o)
    # rows for the range edits below
    o_host, o_other, o_a, o_b, o_past = (b.obj(ON, mu=1) for _ in range(5))
    for o_, n in ((o_host, 8), (o_other, 4), (o_a, 10), (o_b, 10), (o_past, 6)):
        groups(o_, n)
    # a policy-off object and an AfterStart object with a pending group
    groups(b.obj(OFF), 4)
    o = b.obj(AFTER)
    groups(o, 3)
    b.group(o, [node()], leader=node(), pending=(1,))
    w = b.tables("budget_edges")
    lws, g = w.lws, w.groups
    # a row inside o_host's range names o_other; o_a and o_b overlap by 5 groups; o_past runs past the table
    hb = int(lws[o_host]["group_base"])
    g[hb + 3]["lws_index"] = o_other
    lws[o_b]["group_base"] = int(lws[o_b]["group_base"]) - 5
    lws[o_past]["group_count"] = len(g) - int(lws[o_past]["group_base"]) + 1
    notes.update(host=(o_host, hb + 3, o_other), overlap=(o_a, o_b), past=o_past)
    w.notes = notes
    return w


# --------------------------------------------------------------------------- #
# 3. table edges
# --------------------------------------------------------------------------- #
TABLE_NODES = 2048


def pairs_world(pairs: int, seed: int = 3) -> EdgeWorld:
    """Exactly ``pairs`` member (group, node) restart pairs: single-pod groups, one domain per node (so the
    DOMAINS scope has the same pairs), and a policy-off object whose groups add no pair."""
    rng = np.random.Generator(np.random.PCG64(seed))
    nodes, n_domains = node_table(TABLE_NODES, 1)
    b = Builder(nodes, n_domains)
    for n in (pairs // 3, pairs // 3, pairs - 2 * (pairs // 3)):
        o = b.obj(ON)
        for _ in range(n):
            b.group(o, [], leader=int(rng.integers(0, TABLE_NODES)))
    o = b.obj(OFF)
    for _ in range(5):
        b.group(o, [], leader=int(rng.integers(0, TABLE_NODES)))
    w = b.tables(f"pairs_{pairs}")
    w.notes = {"pairs": pairs}
    return w


def wrap_world(chain: int = 12) -> EdgeWorld:
    """(LWS, key) entries chosen with the mixer: ``chain`` of them have the last slot of a 256-slot table as
    home, four more the first slot, so that their probes run past the end and wrap to slot 0; 64 pairs in
    all (the table keeps 256 slots)."""
    nodes, n_domains = node_table(TABLE_NODES, 1)
    b = Builder(nodes, n_domains)
    mask = TABLE_MIN_SLOTS - 1
    objs = [b.obj(ON) for _ in range(4)]
    want = {mask: chain, 0: 4}
    picked = []
    for L in objs:
        for n in range(TABLE_NODES):
            h = table_slot(L << 32 | n, mask)
            if want.get(h, 0) > 0 and len([p for p in picked if p[0] == L]) < 6:
                want[h] -= 1
                picked.append((L, n))
    assert not any(want.values()), want
    filler = iter(n for n in range(TABLE_NODES) if all(n != p[1] for p in picked))
    rows = []
    for L in objs:
        keys = [n for l_, n in picked if l_ == L]
        while len(keys) < 16:
            keys.append(next(filler))
        rows.append(keys)
    for L, keys in zip(objs, rows):
        for n in keys:
            b.group(L, [], leader=n)
    w = b.tables("wrap")
    w.notes = {"entries": [L << 32 | n for L, n in picked], "mask": mask}
    return w


# --------------------------------------------------------------------------- #
# 4. grid edges, sized from the SM count
# --------------------------------------------------------------------------- #
def grid_world(sms: int, what: str, seed: int = 5) -> EdgeWorld:
    """``nodes``: more nodes than the domain mask's grid has threads (4 x 256 x SMs), a few groups on them.
    ``groups``: more groups of 1-2 pods than the mark kernel's grid has threads (16 x 256 x SMs): the
    mark kernel's group loop, the diff's and the set-form budget's strides all run more than once."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if what == "nodes":
        n_nodes = GRID_CAP["drain_domain_mask_kernel"] * GRID_THREADS * sms + 4099
        n_groups = 4000
    else:
        n_nodes = 4096
        n_groups = GRID_CAP["drain_mark_kernel"] * GRID_THREADS * sms + 777
    nodes, n_domains = node_table(n_nodes, 4)
    per_obj = 2
    n_lws = -(-n_groups // per_obj)
    cnt = rng.integers(1, 3, size=n_groups).astype(np.int64)
    base = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    P = int(cnt.sum())
    lws = R.aligned_empty(n_lws, R.LWS_REC)
    gc = np.full(n_lws, per_obj, np.int64)
    gc[-1] = n_groups - per_obj * (n_lws - 1)
    policy = rng.choice([OFF, ON, AFTER], size=n_lws, p=[0.1, 0.7, 0.2]).astype(np.uint32)
    lws["rev_hash"] = REV
    lws["size"] = 2
    lws["flags"] = np.uint32(R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID) | (policy << np.uint32(R.LWS_RESTART_SHIFT))
    lws["replicas"] = lws["sts_replicas"] = lws["sts_replicas_annotation"] = gc
    lws["max_unavailable"] = rng.integers(0, 2, size=n_lws)
    lws["uid_hash"] = np.arange(n_lws, dtype=np.uint64) + np.uint64(0x7000)
    lws["group_base"] = np.arange(n_lws) * per_obj
    lws["group_count"] = gc
    g = R.aligned_empty(n_groups, R.GROUP_REC)
    gi = np.arange(n_groups, dtype=np.uint64)
    g["leader_rev_hash"] = g["wsts_rev_hash"] = REV
    g["wsts_spec_replicas"] = g["wsts_avail_replicas"] = cnt - 1
    g["leader_uid_hash"] = (gi + np.uint64(0x1000_0000)).astype(np.uint32)
    g["wsts_uid_hash"] = (gi + np.uint64(0x2000_0000)).astype(np.uint32)
    g["wsts_owner_uid_hash"] = g["leader_uid_hash"]
    pod_node = rng.integers(0, n_nodes, size=P).astype(np.uint32)
    g["leader_node"] = pod_node[base]
    g["pod_base"], g["pod_count"] = base, cnt
    g["lws_index"] = np.arange(n_groups) // per_obj
    g["flags"] = np.where(rng.random(n_groups) < 0.9, GOOD_GROUP, GOOD_GROUP & ~R.GRP_POD_READY).astype(np.uint32)
    lead = np.zeros(P, bool)
    lead[base] = True
    pst = R.aligned_empty(P, R.POD_STATE)
    sts = R.POD_OWNER_STS << R.POD_OWNER_SHIFT
    pst[:] = (R.POD_PHASE_RUNNING | sts | R.POD_OWNER_NAME_MATCH | np.where(lead, R.POD_IS_LEADER, 0)).astype(np.uint8)
    owner = np.repeat(g["wsts_uid_hash"], cnt)
    place = np.uint32(R.PODID_NAME_OK | R.PODID_SCHEDULED) | (pod_node << np.uint32(R.PODID_NODE_SHIFT))
    pid = R.pod_ident_table(np.full(P, REV, np.uint64), owner, place)
    return EdgeWorld(f"grid_{what}", lws, g, pst, pid, nodes, n_domains, 0, {"sms": sms})


# --------------------------------------------------------------------------- #
# 5. degenerate node tables
# --------------------------------------------------------------------------- #
def degenerate_world(kind: str) -> EdgeWorld:
    """The budget edges' objects on a node table with ``n_domains = 0`` (``no_domains``) or with more domain
    ids than nodes (``sparse_domains``: node n in domain 2n + 1 of 2 x n_nodes + 5)."""
    w = budget_edges_world(seed=13)
    nodes = w.nodes.copy()
    if kind == "no_domains":
        nodes["domain_id"] = R.NONE
        n_domains = 0
    else:
        nodes["domain_id"] = 2 * np.arange(len(nodes)) + 1
        n_domains = 2 * len(nodes) + 5
    return EdgeWorld(kind, w.lws, w.groups, w.pod_state, w.pod_ident, nodes, n_domains, 0, w.notes)


SMALL = ("budget_edges", "pairs_128", "pairs_129", "wrap", "no_domains", "sparse_domains")
BUILDERS = {
    "walk": walk_world,
    "budget_edges": budget_edges_world,
    "pairs_128": lambda: pairs_world(128),
    "pairs_129": lambda: pairs_world(129),
    "wrap": wrap_world,
    "no_domains": lambda: degenerate_world("no_domains"),
    "sparse_domains": lambda: degenerate_world("sparse_domains"),
}
_CACHE: dict = {}


def world(label: str) -> EdgeWorld:
    """The world of this label (built once per process; callers copy before they mutate)."""
    if label not in _CACHE:
        _CACHE[label] = BUILDERS[label]()
    return _CACHE[label]
