"""Tables built to land on the edges of the DS drain (``lwse_resident_ds_drain`` / ``lwse_resident_ds_drain_cost``).

The set form runs ``ds_drain_lost_kernel`` (one warp per LWS row over its group range, 32 groups a step), two linked
DS sweeps and ``ds_drain_diff_kernel`` (one thread per DS over its (V + 1) x n revision-role rows, the touched DS
appended with one atomic per warp).  The per-key form counts and fills a reverse link index with
``ds_drain_links_kernel`` behind ``place_index_scan_kernel`` (``first[n_lws]`` bounds the last LWS row's entries),
then runs ``ds_drain_pairs_kernel`` / ``ds_drain_insert_kernel`` over the drain budget's (LWS, key) table and
``ds_drain_finish_kernel`` over the (DS, key) table.  A fill entry carries the row's revision slot (``kDsDrainNewSlot``
for the new revision) and ``kDsDrainSpec``.  The engine refuses more than 2^30 index entries, (group, key) pairs or
(DS, key) pairs.  Every grid is capped at a multiple of the SM count and strides beyond it.

Each world here carries cases whose labels name the edge and the side they sit on; the constants the labels depend
on are restated below (``tests/test_ds_drain_edges.py`` reads them back from the sources).  Children are built with
``drain_edges_world.Builder``, DS rows with ``ds_limits_world``; the definitions are ``tests/ds_drain_ref.py``.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

import drain_edges_world as DW
import ds_limits_world as LW
from drain_budget_ref import key_of, owners
from drain_ref import restart_pairs
from ds_drain_ref import I32_MAX, I32_MIN, World, ds_ok, link_targets, ready_columns
from ds_link_world import none_links
from lws_b200 import records as R

# the DS drain's launch constants (lwse_ds_kernels.cu, lwse_drain_kernels.cu, lwse_place_ns_kernels.cu)
DS_THREADS = 128          # ds_grid: threads per CTA of the drain sweeps, the diff and both links passes
DS_CAP = 16               # ds_grid: CTAs per SM at most
LOST_THREADS = 256        # ds_drain_lost_kernel: 8 warps per CTA, one LWS row per warp
LOST_CAP = 8              # ... CTAs per SM at most
COST_THREADS = 256        # pairs / insert (per (LWS, key) slot) and finish (per (DS, key) slot)
COST_CAP = 8              # ... CTAs per SM at most
INDEX_SCAN_THREADS = 1024  # place_index_scan_kernel: one CTA, chunks of this many LWS rows
REFUSE_ABOVE = 1 << 30    # index entries, (group, key) pairs and (DS, key) pairs the engine accepts at most
NEW_SLOT, SPEC = 0xFF, 0x100  # kDsDrainNewSlot, kDsDrainSpec
H100_SMS = 132
WARP = 32
NONE = -1


def ds_grid(n_ds: int, sms: int) -> int:
    return min(-(-n_ds // DS_THREADS), DS_CAP * sms)


def grid_for(items: int, per_cta: int, cap: int) -> int:
    return min(max(-(-items // per_cta), 1), cap)


def ds_stride(sms: int) -> int:
    """DS rows one pass of a ds_grid kernel covers."""
    return DS_CAP * sms * DS_THREADS


def lost_stride(sms: int) -> int:
    """LWS rows one pass of ds_drain_lost_kernel covers (one per warp)."""
    return LOST_CAP * sms * (LOST_THREADS // WARP)


def cost_stride(sms: int) -> int:
    """Table slots one pass of the pairs, insert or finish kernel covers."""
    return COST_CAP * sms * COST_THREADS


# --------------------------------------------------------------------------- #
# builders
# --------------------------------------------------------------------------- #
class Kids:
    """Child LeaderWorkerSets of one-pod groups: ``child(nodes)`` makes a row with one group per entry, its leader
    on that node row.  ``node()`` hands out node rows no other child uses."""

    def __init__(self):
        self.specs, self.n_nodes = [], 0

    def node(self) -> int:
        self.n_nodes += 1
        return self.n_nodes - 1

    def child(self, nodes, ready=True, replicas=None) -> int:
        self.specs.append((list(nodes), ready, replicas))
        return len(self.specs) - 1

    def tables(self, label: str, per_domain: int = 4) -> DW.EdgeWorld:
        nodes, nd = DW.node_table(max(per_domain * -(-(self.n_nodes + 1) // per_domain), per_domain), per_domain)
        b = DW.Builder(nodes, nd)
        for ns, ready, reps in self.specs:
            o = b.obj(DW.ON, size=1, replicas=reps)
            for n in ns:
                b.group(o, [], leader=n, ready=ready)
        return b.tables(label)


@dataclass
class Case:
    label: str
    node: int                 # the node row whose drain the case is
    ds: int                   # the DS row it is about (-1: none is touched)
    row: int = -1             # the revision-role row it zeroes (-1: none)
    expect: dict = field(default_factory=dict)  # DS_DRAIN fields and verdict bits of the case's row


@dataclass
class DsEdgeWorld:
    label: str
    w: World
    cases: list = field(default_factory=list)
    notes: dict = field(default_factory=dict)


def world_of(e: DW.EdgeWorld, ds, roles, rr, targets) -> World:
    """A DS drain World over children ``e``: revision-role row r links to LWS row targets[r] (-1: not linked)."""
    import oracle

    base = oracle.sweep_lws(e.lws, e.groups, e.pod_state, e.pod_ident, e.nodes, e.flags & R.SWEEP_GANG)[:2]
    targets = np.asarray(targets, np.int64)
    links = none_links(len(rr))
    on = targets >= 0
    links["lws_row"][on] = targets[on]
    links["lws_uid_hash"][on] = e.lws["uid_hash"][targets[on]]
    links["reserved"] = 0
    return World(e.lws, e.groups, e.pod_state, e.pod_ident, e.nodes, e.n_domains, e.flags,
                 np.ascontiguousarray(ds), np.ascontiguousarray(roles), np.ascontiguousarray(rr), links, base)


def _ds(S, X, V, has_new=True, old_replicas=1, new_replicas=1) -> LW.DsRows:
    """A DS with every revision-role row present (ready 1 until a link says otherwise)."""
    x = LW._empty(S, X, V, has_new)
    x.roles["target_replicas"] = 1
    n = S + X
    for r in range(V + 1):
        for i in range(n):
            LW._put(x, r, i, old_replicas if r < V else new_replicas, ready=1, stamp=r + 1)
    return x


# --------------------------------------------------------------------------- #
# 1. limit DS through the drain
# --------------------------------------------------------------------------- #
LIMIT_V = (0, 1, 31, 32)
LIMIT_ROLES = ((1, 0), (2, 0), (10, 0), (9, 1))   # (spec roles, removed roles)
MATRIX = ((0, 0), (1, 1), (2, 1), (2, 2), (3, 1), (3, 2), (3, 3))  # (ready groups, of them on the drained node)


def limit_world() -> DsEdgeWorld:
    """One DS per V in LIMIT_V and role shape in LIMIT_ROLES, and DS with one special property each; every row has
    a child of its own (one ready group on a node of its own) unless a case says otherwise.  A case drains the node
    of one row's child, so that it touches that row alone."""
    k = Kids()
    items, tg, cases, notes = [], [], [], {}

    def add(x: LW.DsRows, label, child_of=None):
        n = len(x.roles)
        t = np.full(len(x.rr), NONE, np.int64)
        for j in range(len(x.rr)):
            if x.rr["flags"][j] & R.RR_EXISTS:
                c = child_of(j) if child_of else None
                t[j] = c if c is not None else k.child([k.node()])
        items.append(x)
        tg.append(t)
        notes[label] = len(items) - 1
        return len(items) - 1, n

    def case(label, d, r, i, **expect):
        cases.append((label, d, r, i, expect))

    for V in LIMIT_V:
        for S, X in LIMIT_ROLES:
            d, n = add(_ds(S, X, V), f"V{V}_S{S}_X{X}")
            i = n - 1
            spec = i < S
            tag = "spec" if spec else "removed"
            # the new revision's last role: a spec role serves (SERVICE_LOST; STALLS when the DS is rolling) and
            # sets its bit; a removed role counts in rows_zeroed and nothing else
            case(f"new_{tag}_role{i}_V{V}_S{S}_X{X}", d, V, i,
                 new_zeroed_roles=(1 << i) if spec else 0, old_zeroed_roles=0,
                 set=(R.DSD_SERVICE_LOST | (R.DSD_STALLS if V else 0)) if spec else 0,
                 clear=0 if spec else R.DSD_SERVICE_LOST | R.DSD_STALLS | R.DSD_OLD_SERVICE_LOST,
                 stable_before=V > 0, fell=0)
            if V:
                case(f"old{V - 1}_{tag}_role{i}_V{V}_S{S}_X{X}", d, V - 1, i,
                     new_zeroed_roles=0, old_zeroed_roles=(1 << i) if spec else 0,
                     set=R.DSD_OLD_SERVICE_LOST if spec else 0,
                     clear=R.DSD_SERVICE_LOST | R.DSD_STALLS | (0 if spec else R.DSD_OLD_SERVICE_LOST),
                     fell=(1 << (V - 1)) if spec else 0)
    # an old revision that does not serve before the drain (role 0 missing): zeroing its role 9 loses nothing
    x = _ds(10, 0, 31)
    x.rr["flags"][5 * 10 + 0] = 0
    d, _ = add(x, "old_not_ready")
    case("old5_spec_role9_not_ready_before", d, 5, 9, new_zeroed_roles=0, old_zeroed_roles=0, set=0,
         clear=R.DSD_OLD_SERVICE_LOST | R.DSD_SERVICE_LOST | R.DSD_STALLS, fell=0, ready_bit_clear_before=5)
    # a drained revision (nil replicas): its rows still serve while ready
    x = _ds(10, 0, 32)
    x.rr["replicas"][31 * 10: 32 * 10] = 0
    x.rr["flags"][31 * 10: 32 * 10] |= np.uint32(R.RR_REPLICAS_NIL)
    d, _ = add(x, "drained_rev")
    case("old31_spec_role9_drained_rev", d, 31, 9, new_zeroed_roles=0, old_zeroed_roles=1 << 9,
         set=R.DSD_OLD_SERVICE_LOST, clear=R.DSD_SERVICE_LOST | R.DSD_STALLS, fell=1 << 31, drained_bit=31)
    # not rolling (no old replicas), and INIT (rolling without a new revision): neither is stable, so none stalls
    d, _ = add(_ds(2, 0, 1, old_replicas=0), "not_rolling")
    case("new_spec_role1_not_rolling", d, 1, 1, new_zeroed_roles=2, old_zeroed_roles=0, set=R.DSD_SERVICE_LOST,
         clear=R.DSD_STALLS, stable_before=False, fell=0)
    d, _ = add(_ds(2, 0, 1, has_new=False), "init")
    case("new_spec_role1_init", d, 1, 1, new_zeroed_roles=2, old_zeroed_roles=0, set=R.DSD_SERVICE_LOST,
         clear=R.DSD_STALLS, stable_before=False, init=True, fell=0)
    # ready_before x lost: the new revision's role 1 linked to a child of `ready` ready groups, `lost` of them on
    # the drained node (ready 0: one group that is not ready, on that node); replicas = ready, so the DS is stable
    for ready, lost in MATRIX:
        x = _ds(2, 0, 1, new_replicas=1)
        x.rr["replicas"][1 * 2 + 1] = ready
        drained = k.node()

        def child_of(j, ready=ready, lost=lost, drained=drained):
            if j != 3:  # (row 3: the new revision's role 1)
                return None
            if ready == 0:
                return k.child([drained], ready=False)
            return k.child([drained] * lost + [k.node() for _ in range(ready - lost)])

        d, _ = add(x, f"matrix_{ready}_{lost}", child_of)
        zero = ready >= 1 and ready - lost < 1
        cases.append((f"ready{ready}_lost{lost}", d, 1, 1, dict(
            new_zeroed_roles=2 if zero else 0, old_zeroed_roles=0, rows_zeroed=int(zero), rows_touched=int(lost > 0),
            set=(R.DSD_SERVICE_LOST if zero else 0) | (R.DSD_STALLS if lost else 0),
            clear=0 if zero else R.DSD_SERVICE_LOST, fell=0, node=drained)))
    e = k.tables("limit")
    ds, roles, rr = LW.assemble(items)
    targets = np.full(len(rr), NONE, np.int64)
    vb = ds["rev_base"].astype(np.int64)
    for d, t in enumerate(tg):
        targets[vb[d]: vb[d] + len(t)] = t
    w = world_of(e, ds, roles, rr, targets)
    out = []
    for label, d, r, i, expect in cases:
        n = int(ds["n_roles"][d])
        row = int(vb[d]) + r * n + i
        node = expect.pop("node", None)
        if node is None:
            L = int(targets[row])
            node = int(e.groups["leader_node"][int(e.lws["group_base"][L])])
        expect.setdefault("rows_touched", 1)
        expect.setdefault("rows_zeroed", 1)
        out.append(Case(label, node, d, row, expect))
    return DsEdgeWorld("limit", w, out, notes)


# --------------------------------------------------------------------------- #
# 2. child LWS edges
# --------------------------------------------------------------------------- #
def child_edges_world() -> DsEdgeWorld:
    """The children of ``drain_edges_world.budget_edges_world``: rows of 31-1 000 groups, surge groups, replicas 0
    and -4, a group naming another LWS, overlapping ranges and a range past the table.  Each child gets a DS of one
    old revision and two spec roles whose four rows all link to it (new-revision replicas = its ready count, so the
    DS is stable before the drain); two DS of 32 old revisions link their rows to every child in turn."""
    import oracle

    e = DW.budget_edges_world()
    lws_out = oracle.sweep_lws(e.lws, e.groups, e.pod_state, e.pod_ident, e.nodes, e.flags & R.SWEEP_GANG)[0]
    items, tg, per = [], [], {}
    for L in range(len(e.lws)):
        x = _ds(2, 0, 1, new_replicas=max(int(lws_out["ready_replicas"][L]), 0))
        items.append(x)
        tg.append(np.full(4, L))
        per[L] = len(items) - 1
    for off in (0, 7):
        x = _ds(1, 1, 32)
        items.append(x)
        tg.append((np.arange(len(x.rr)) + off) % len(e.lws))
    ds, roles, rr = LW.assemble(items)
    w = world_of(e, ds, roles, rr, np.concatenate(tg))
    n = e.notes
    named = {f"rows_{g}": n["rows"][g] for g in DW.BUDGET_ROW_GROUPS}
    named.update(replicas_0=n["rows"]["replicas_0"], replicas_m4=n["rows"]["replicas_-4"], surge=n["surge"][0],
                 host=n["host"][0], other=n["host"][2], overlap_a=n["overlap"][0], overlap_b=n["overlap"][1],
                 past=n["past"])
    return DsEdgeWorld("child_edges", w, [], dict(named=named, ds_of=per, host_group=n["host"][1],
                                                   surge_groups=n["surge"][1:]))


# --------------------------------------------------------------------------- #
# 3. fan-out and the index scan
# --------------------------------------------------------------------------- #
FAN_ROWS = 100_000
SCAN_N_LWS = (2049, 1025, 1024, 1023)  # (the GPU test runs them in this order on one engine)


def fan_world(rows: int) -> DsEdgeWorld:
    """Every row of every DS linked to child 0 (one ready group on node 0): a V = 32, n = 10 DS (330 rows), then
    DS of 4 old revisions and 2 spec roles (10 rows each) up to ``rows`` rows.  Draining node 0 zeroes them all."""
    k = Kids()
    c = k.child([k.node()])
    k.child([k.node()])  # (a child no row links to)
    items = [_ds(10, 0, 32)]
    total = 330
    while total < rows:
        items.append(_ds(2, 0, 4))
        total += 10
    ds, roles, rr = LW.assemble(items)
    w = world_of(k.tables(f"fan_{rows}"), ds, roles, rr, np.full(len(rr), c))
    return DsEdgeWorld(f"fan_{rows}", w, [Case(f"one_child_{total}_rows", 0, -1)], dict(child=c, rows=total))


def scan_world(n_lws: int) -> DsEdgeWorld:
    """``n_lws`` children of one ready group; only the last is linked (from a DS of one old revision and two spec
    roles) and only its group is on node 0.  Its index entries start at first[n_lws - 1] and end at first[n_lws]."""
    k = Kids()
    drained, other = k.node(), k.node()
    for _ in range(n_lws - 1):
        k.child([other])
    last = k.child([drained])
    ds, roles, rr = LW.assemble([_ds(2, 0, 1)])
    w = world_of(k.tables(f"scan_{n_lws}"), ds, roles, rr, np.full(len(rr), last))
    return DsEdgeWorld(f"scan_{n_lws}", w, [Case(f"last_of_{n_lws}_lws_rows", drained, 0)], dict(last=last))


# --------------------------------------------------------------------------- #
# 4. grids, sized from the SM count
# --------------------------------------------------------------------------- #
def _one_role_ds(n_ds: int):
    """n_ds DS of one spec role and no old revision, with contiguous rows (DS i: role row i, revision-role row i)."""
    ds = R.aligned_empty(n_ds, R.DS_REC)
    ds["uid_hash"] = np.arange(n_ds, dtype=np.uint64) + np.uint64(1)
    ds["role_base"] = ds["rev_base"] = np.arange(n_ds)
    ds["n_roles"] = ds["n_spec_roles"] = 1
    ds["n_old_revs"] = 0
    ds["flags"] = R.DS_HAS_NEW_REVISION
    roles = R.aligned_empty(n_ds, R.DS_ROLE_REC)
    roles[:] = (1, 0, 0, R.ROLE_IN_SPEC)
    rr = R.aligned_empty(n_ds, R.DS_REVROLE_REC)
    rr[:] = (1, -1, 1, R.RR_EXISTS | (1 << R.RR_TS_SHIFT))
    return ds, roles, rr


def grid_ds_world(sms: int) -> DsEdgeWorld:
    """16 x 128 x SMs + 37 one-role DS: the drain sweeps, the diff and both links passes stride once.  DS in the
    last stride are linked on both sides of its first warp boundary (G + 31 and G + 32 share a child, as do G + 30
    and G + 33), with G + 0, G + 36 and the last DS of the first stride on a third; the first 40 DS on other
    children; every other row is not linked."""
    G = ds_stride(sms)
    n_ds = G + 37
    k = Kids()
    kids = [k.child([k.node()]) for _ in range(64)]
    ds, roles, rr = _one_role_ds(n_ds)
    t = np.full(n_ds, NONE, np.int64)
    t[[G + 31, G + 32]] = kids[0]
    t[[G + 30, G + 33]] = kids[1]
    t[[G - 1, G, G + 36]] = kids[2]
    t[:40] = [kids[3 + i % 61] for i in range(40)]
    w = world_of(k.tables(f"grid_ds_{sms}"), ds, roles, rr, t)
    cases = [Case("last_stride_warp_31_32", kids[0], G + 31), Case("last_stride_warp_30_33", kids[1], G + 30),
             Case("stride_edges_G-1_G_G+36", kids[2], G), Case("first_stride", kids[3], 0)]
    return DsEdgeWorld(f"grid_ds_{sms}", w, cases, dict(sms=sms, G=G, n_ds=n_ds))


def grid_links_world(sms: int) -> DsEdgeWorld:
    """One one-role DS per child of ``drain_edges_world.grid_world(sms, "groups")`` (16 x 256 x SMs + 777 groups of
    1-2 pods, two per LWS row): more LWS rows than the lost kernel's grid has warps, an (LWS, key) table past the
    pairs and insert grids, and more (DS, key) pairs than the finish grid has threads.  The cases drain the node of
    the highest LWS row that loses a group (in the lost kernel's last stride) and of the lowest."""
    e = DW.grid_world(sms, "groups")
    n = len(e.lws)
    ds, roles, rr = _one_role_ds(n)
    w = world_of(e, ds, roles, rr, np.arange(n))
    pl, pk, _ = lost_pair_arrays(w, False)
    cases = [Case("lost_last_stride", int(pk[-1]), int(pl[-1])), Case("lost_first_stride", int(pk[0]), int(pl[0]))]
    return DsEdgeWorld(f"grid_links_{sms}", w, cases, dict(sms=sms, n_lws=n))


# --------------------------------------------------------------------------- #
# 5. refusals: DS over one shared range of V = 32, n = 10 rows
# --------------------------------------------------------------------------- #
PAIRS_REFUSED, PAIRS_ACCEPTED = 3178, 3177        # DS over a child of 1 024 groups on 1 024 nodes
ENTRIES_REFUSED, ENTRIES_ACCEPTED = 3_253_764, 3_253_763  # DS over 330 children
SHARED_ROWS = 330
PAIRS_CHILD_GROUPS = 1024


def _shared_ds(n_ds: int):
    x = _ds(10, 0, 32)
    ds = R.aligned_empty(n_ds, R.DS_REC)
    ds["uid_hash"] = np.arange(n_ds, dtype=np.uint64) + np.uint64(1)
    ds["role_base"], ds["n_roles"], ds["n_spec_roles"] = 0, 10, 10
    ds["rev_base"], ds["n_old_revs"], ds["flags"] = 0, 32, R.DS_HAS_NEW_REVISION
    roles = R.aligned_empty(10, R.DS_ROLE_REC)
    roles[:] = x.roles
    rr = R.aligned_empty(SHARED_ROWS, R.DS_REVROLE_REC)
    rr[:] = x.rr
    return ds, roles, rr


def refuse_pairs_world(n_ds: int = PAIRS_REFUSED) -> DsEdgeWorld:
    """``n_ds`` DS sharing one 330-row range, every row linked to one child of 1 024 ready groups on 1 024 distinct
    nodes: a node's drain gives n_ds x 330 (row, key) pairs of (DS, key) pairs, 1 024 nodes in all."""
    k = Kids()
    c = k.child([k.node() for _ in range(PAIRS_CHILD_GROUPS)])
    ds, roles, rr = _shared_ds(n_ds)
    w = world_of(k.tables("refuse_pairs"), ds, roles, rr, np.full(SHARED_ROWS, c))
    return DsEdgeWorld(f"refuse_pairs_{n_ds}", w, [], dict(ds_pairs=n_ds * SHARED_ROWS * PAIRS_CHILD_GROUPS,
                                                          entries=n_ds * SHARED_ROWS))


def refuse_entries_world(n_ds: int = ENTRIES_REFUSED) -> DsEdgeWorld:
    """``n_ds`` DS sharing one 330-row range whose row k links to child k (one ready group on node k): n_ds x 330
    reverse-index entries, spread over 330 counters."""
    k = Kids()
    kids = [k.child([k.node()]) for _ in range(SHARED_ROWS)]
    ds, roles, rr = _shared_ds(n_ds)
    w = world_of(k.tables("refuse_entries"), ds, roles, rr, np.array(kids))
    return DsEdgeWorld(f"refuse_entries_{n_ds}", w, [], dict(entries=n_ds * SHARED_ROWS))


# --------------------------------------------------------------------------- #
# the per-key form, vectorised
# --------------------------------------------------------------------------- #
def entries_of(w: World):
    """Every (DS, revision-role row) the sweep reads, once per DS whose range holds the row: (DS, row, slot, spec),
    slot = V for the new revision."""
    ok = np.flatnonzero(ds_ok(w.ds, len(w.roles), len(w.revroles)))
    n = w.ds["n_roles"][ok].astype(np.int64)
    V = w.ds["n_old_revs"][ok].astype(np.int64)
    cnt = (V + 1) * n
    d = np.repeat(ok, cnt)
    k = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    nn = np.repeat(n, cnt)
    row = w.ds["rev_base"][d].astype(np.int64) + k
    spec = (k % nn) < w.ds["n_spec_roles"][d].astype(np.int64)
    return d, row, k // nn, spec


def lost_pair_arrays(w: World, by_domain: bool):
    """(L, key, lost) arrays of lost(L, key) > 0, sorted by (L, key)."""
    key = key_of(w.nodes, w.n_domains, by_domain)
    g, nd = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), w.base[1])
    kk = key[nd]
    g, kk = g[kk >= 0], kk[kk >= 0]
    gk = np.unique(g.astype(np.int64) << 32 | kk)
    g, kk = gk >> 32, gk & 0xFFFFFFFF
    own = owners(w.lws, w.groups)
    m = (own[g] >= 0) & ((w.base[1]["flags"][g] & R.GOUT_COND_READY) != 0)
    lk, lost = np.unique(own[g][m] << 32 | kk[m], return_counts=True)
    return lk >> 32, lk & 0xFFFFFFFF, lost.astype(np.int64)


def ds_drain_cost_vec(w: World, by_domain=False, before_ds_out=None) -> np.ndarray:
    """``ds_drain_ref.ds_drain_cost_ref`` restated with array operations: every (row, key) fact, ORed per (DS, key),
    gated by the DS's flags in the before sweep."""
    import oracle

    n_keys = w.n_domains if by_domain else len(w.nodes)
    out = np.zeros(n_keys, R.DS_DRAIN_COST)
    L, rb, _ = ready_columns(w, np.zeros(len(w.lws), np.int64))
    d, row, slot, spec = entries_of(w)
    Le = L[row]
    take = Le >= 0
    d, row, slot, spec, Le = d[take], row[take], slot[take], spec[take], Le[take]
    o = np.argsort(Le, kind="stable")
    d, row, slot, spec, Le = d[o], row[o], slot[o], spec[o], Le[o]
    pl, pk, plost = lost_pair_arrays(w, by_domain)
    lo, hi = np.searchsorted(Le, pl, "left"), np.searchsorted(Le, pl, "right")
    cnt = hi - lo
    p = np.repeat(np.arange(len(pl)), cnt)
    j = np.repeat(lo, cnt) + np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    key = pk[p]
    b = rb[row[j]]
    a = np.clip(b - plost[p], I32_MIN, I32_MAX)
    zero = (b >= 1) & (a < 1)
    out["rows_touched"] = np.bincount(key, minlength=n_keys)[:n_keys]
    out["rows_zeroed"] = np.bincount(key[zero], minlength=n_keys)[:n_keys]
    dd = d[j]
    V = w.ds["n_old_revs"][dd].astype(np.int64)
    new = spec[j] & (slot[j] == V)
    nz, nc = new & zero, new & (a != b)
    om = np.where(spec[j] & (slot[j] < V) & zero, np.left_shift(1, np.minimum(slot[j], 31)), 0).astype(np.int64)
    dk, inv = np.unique(dd << 32 | key, return_inverse=True)
    NZ = np.zeros(len(dk), bool)
    NC = np.zeros(len(dk), bool)
    OM = np.zeros(len(dk), np.int64)
    np.logical_or.at(NZ, inv, nz)
    np.logical_or.at(NC, inv, nc)
    np.bitwise_or.at(OM, inv, om)
    if before_ds_out is None:
        rr = w.revroles.copy()
        rr["ready_replicas"] = rb
        before_ds_out = oracle.sweep_ds(w.ds, w.roles, rr)[0]
    D, K = dk >> 32, dk & 0xFFFFFFFF
    f, rrv = before_ds_out["flags"][D].astype(np.int64), before_ds_out["ready_revs"][D].astype(np.int64)
    out["ds_touched"] = np.bincount(K, minlength=n_keys)[:n_keys]
    out["ds_service_lost"] = np.bincount(K[NZ & ((f & R.DOUT_NEW_READY) != 0)], minlength=n_keys)[:n_keys]
    out["ds_old_service_lost"] = np.bincount(K[(OM & rrv) != 0], minlength=n_keys)[:n_keys]
    out["ds_stalled"] = np.bincount(K[NC & ((f & R.DOUT_STABLE) != 0)], minlength=n_keys)[:n_keys]
    return out


def ds_pairs_of(w: World, by_domain: bool) -> int:
    """(row, key) pairs of the per-key form: the pairs kernel's count that sizes the (DS, key) table."""
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    d, row, _, _ = entries_of(w)
    per_L = np.bincount(L[row][L[row] >= 0], minlength=len(w.lws))
    pl, _, _ = lost_pair_arrays(w, by_domain)
    return int(per_L[pl].sum())


SMALL = ("limit", "child_edges", "fan_330", "scan_2049", "scan_1025", "scan_1024", "scan_1023")
BUILDERS = {
    "limit": limit_world,
    "child_edges": child_edges_world,
    "fan_330": lambda: fan_world(330),
    "fan_100k": lambda: fan_world(FAN_ROWS),
    **{f"scan_{n}": (lambda n=n: scan_world(n)) for n in SCAN_N_LWS},
}
_CACHE: dict = {}


def world(label: str) -> DsEdgeWorld:
    """The world of this label (built once per process)."""
    if label not in _CACHE:
        if label.startswith("grid_ds_"):
            _CACHE[label] = grid_ds_world(int(label.rsplit("_", 1)[1]))
        elif label.startswith("grid_links_"):
            _CACHE[label] = grid_links_world(int(label.rsplit("_", 1)[1]))
        else:
            _CACHE[label] = BUILDERS[label]()
    return _CACHE[label]
