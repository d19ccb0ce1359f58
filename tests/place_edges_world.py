"""Placement tables built to land on each launch path of the round, at that path's thresholds.

Two launchers pick the code a placement call runs (``lws_b200/csrc/lwse_place_kernels.cu`` and
``lwse_place_ns_kernels.cu``):

* ``launch_place`` runs the general form as ONE thread-block cluster (128 warps in either cluster
  shape) when there are few requests — or few predicted unpinned ones — and the node and holder tables
  are small, else as a cooperative grid of ``clamp(ceil(n_reqs / 16), 16, sm_count)`` CTAs of 16 warps.
  A warp keeps its first ``kCacheQ`` requests in shared memory; the rest live in their result rows.
  The prediction is the previous call's unpinned count for the same geometry (none after a change).
* ``launch_place_ns`` runs the namespace form, one CTA per namespace on ``min(n_namespaces, 2 x
  sm_count)`` CTAs, when its shared memory fits (``place_ns_supported``).  A namespace keeps the state of
  its first ``kNsCache`` unpinned requests in shared memory and the first ``kNsKeep`` requests of each
  thread in registers; the scan form stages the node-word table when it fits in 100 KB.

Every builder here sets the counts with numpy so that its case lands exactly where its label says, and
the constants the labels depend on are restated below (``tests/test_place_edges.py`` reads them back
from the kernel sources).  Every node table also carries the row-level edges of the spec: capacities
15, 16 and 65 535 (the 4-bit free-slot nibble saturates, the domain sum does not), occupancy above
capacity, domains without a usable node and domains whose nodes are all full, unschedulable,
unlabelled and out-of-range-label nodes; the request tables carry sizes 0, negative and larger than
any domain, priorities equal above bit 25, pinned leaders on each kind of node and on a missing node,
and rows of a namespace that does not exist.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from lws_b200 import records as R

# the general launcher's constants (lwse_place_kernels.cu)
K_PLACE_THREADS = 512   # threads per CTA of place_kernel (the 16-CTA cluster shape halves it: same warps)
K_CLUSTER_CTAS = 8      # CTAs of the cluster at 512 threads
K_CACHE_Q = 4           # requests per warp whose state lives in shared memory
FEW_PER_WARP = 8        # few_reqs: n_reqs <= kClusterCtas * kPlaceWarps * 8
PREDICTED_PER_WARP = 2  # or predicted unpinned <= kClusterCtas * kPlaceWarps * 2 ...
MAX_CLUSTER_REQS = 1 << 14   # ... with n_reqs <= 1 << 14
MAX_CLUSTER_NODES = 1 << 16  # and n_nodes <= 1 << 16
MAX_CLUSTER_HOLD = 1 << 16   # and n_namespaces * hold_stride <= 1 << 16
HISTORY_ABOVE = 1024         # the engine records a call's unpinned count only beyond this many requests
K_PLACE_WARPS = K_PLACE_THREADS // 32
CLUSTER_WARPS = K_CLUSTER_CTAS * K_PLACE_WARPS
GRID_MIN_CTAS = 16

# the namespace launcher's constants (lwse_place_ns_kernels.cu)
K_NS_THREADS = 512       # two-level form
K_NS_SCAN_THREADS = 256  # scan form
K_NS_KEEP = 2            # requests per thread kept in registers
K_NS_CACHE = 256         # unpinned requests per namespace whose state lives in shared memory
NS_SMEM_LIMIT = 200 * 1024     # place_ns_supported
STAGE_SMEM_LIMIT = 100 * 1024  # the scan form stages the word table at or below this

H100_SXM_SMS = 132
USABLE = R.NODE_HAS_TOPOLOGY | R.NODE_SCHEDULABLE
TOO_BIG = 0x7FFFFFFF  # a request size beyond any domain's free capacity
EDGE_LIVE = 1         # live unpinned rows among Requests.edges (the TOO_BIG one)


# --------------------------------------------------------------------------- #
# the launchers' choices, restated
# --------------------------------------------------------------------------- #
def hold_stride(n_domains: int) -> int:
    return (n_domains + 1) & ~1


def ns_smem_bytes(word_rows: int, n_domains: int, scan: bool, stage: bool) -> int:
    free_bytes = (n_domains * 4 + 15) & ~15
    base = free_bytes + (((n_domains + 1) * 4 + 15) & ~15) + n_domains * 8 + 256 * 32 + 16 + 128
    if scan:
        return base + (word_rows * 2048 if stage else 0)
    return base + n_domains * 16 + free_bytes


def word_rows(n_nodes: int) -> int:
    return max(1, (n_nodes + 255) // 256)


def place_ns_supported(n_nodes: int, n_domains: int) -> bool:
    return (ns_smem_bytes(word_rows(n_nodes), n_domains, False, False) <= NS_SMEM_LIMIT
            and n_domains < (1 << 28) and n_nodes < (1 << 28))


def stage_words(n_nodes: int, n_domains: int) -> bool:
    return ns_smem_bytes(word_rows(n_nodes), n_domains, True, True) <= STAGE_SMEM_LIMIT


def few_reqs(n_reqs: int) -> bool:
    return n_reqs <= CLUSTER_WARPS * FEW_PER_WARP


def general_path(n_reqs, n_nodes, n_domains, n_namespaces, expect_unpinned) -> str:
    small = ((few_reqs(n_reqs) or (expect_unpinned <= CLUSTER_WARPS * PREDICTED_PER_WARP and n_reqs <= MAX_CLUSTER_REQS))
             and n_nodes <= MAX_CLUSTER_NODES and n_namespaces * hold_stride(n_domains) <= MAX_CLUSTER_HOLD)
    return "cluster" if small else "grid"


def grid_ctas(n_reqs: int, sm_count: int) -> int:
    return max(GRID_MIN_CTAS, min(-(-n_reqs // K_PLACE_WARPS), sm_count))


def general_warps(path: str, n_reqs: int, sm_count: int) -> int:
    return CLUSTER_WARPS if path == "cluster" else grid_ctas(n_reqs, sm_count) * K_PLACE_WARPS


def grouped(reqs) -> bool:
    return bool(np.all(np.diff(reqs["ns"].astype(np.int64)) >= 0))


def host_form(reqs, n_nodes, n_domains) -> str:
    """What ``lwse_place_host`` runs: the namespace form for a grouped table it can fit, else the general one."""
    return "namespace" if len(reqs) and grouped(reqs) and place_ns_supported(n_nodes, n_domains) else "general"


def live_unpinned(reqs, n_namespaces) -> np.ndarray:
    return (reqs["leader_node"] == R.NONE) & (reqs["size"] >= 1) & (reqs["ns"] < n_namespaces)


def general_calls(case: "Case", sm_count: int) -> list[dict]:
    """The path, warps and per-warp requests of each call of ``case.calls`` in order, through one entry
    point right after the node table was uploaded (no history)."""
    out, history = [], None
    n_nodes = len(case.nodes)
    for reqs in case.calls:
        n = len(reqs)
        expect = n if history is None else history
        path = general_path(n, n_nodes, case.n_domains, case.n_namespaces, expect)
        unp = int(live_unpinned(reqs, case.n_namespaces).sum())
        gw = general_warps(path, n, sm_count)
        out.append({"path": path, "expect_unpinned": expect, "live_unpinned": unp, "warps": gw,
                    "ctas": None if path == "cluster" else grid_ctas(n, sm_count),
                    "per_warp": -(-unp // gw), "n_reqs": n, "n_nodes": n_nodes,
                    "hold": case.n_namespaces * hold_stride(case.n_domains)})
        if n > HISTORY_ABOVE:
            history = unp
    return out


def ns_view(case: "Case", sm_count: int) -> dict:
    """The namespace launcher's view of a (grouped) case."""
    reqs, n_ns = case.calls[0], case.n_namespaces
    ns = reqs["ns"].astype(np.int64)
    inr = ns < n_ns
    rows = np.bincount(ns[inr], minlength=n_ns)
    unp = np.bincount(ns[live_unpinned(reqs, n_ns)], minlength=n_ns)
    pinned = np.bincount(ns[inr & (reqs["leader_node"] != R.NONE)], minlength=n_ns)
    n_nodes = len(case.nodes)
    grid = max(1, min(n_ns, 2 * sm_count))
    return {"supported": place_ns_supported(n_nodes, case.n_domains), "stage_words": stage_words(n_nodes, case.n_domains),
            "smem": ns_smem_bytes(word_rows(n_nodes), case.n_domains, False, False),
            "scan_smem": ns_smem_bytes(word_rows(n_nodes), case.n_domains, True, True),
            "rows": rows, "unpinned": unp, "pinned": pinned, "grid": grid, "n_nodes": n_nodes}


# --------------------------------------------------------------------------- #
# builders
# --------------------------------------------------------------------------- #
class Nodes:
    """Node rows listed domain by domain; ``build`` shuffles them, so no domain is a run of rows."""

    def __init__(self, n_domains: int):
        self.n_domains = n_domains
        self.cols = {"domain": [], "capacity": [], "occ": [], "flags": []}
        self.regular: list[int] = []  # domains with free capacity >= 3

    def add(self, domains, per_domain: int, capacity: int, occ: int = 0, flags: int = USABLE):
        d = np.repeat(np.asarray(domains, dtype=np.int64), per_domain)
        for k, v in (("domain", d), ("capacity", np.full(len(d), capacity)), ("occ", np.full(len(d), occ)),
                     ("flags", np.full(len(d), flags))):
            self.cols[k].append(v)
        return self

    def regular_domains(self, domains, per_domain: int, capacity: int = 6, occ: int = 2):
        assert capacity - occ >= 3
        self.regular.extend(int(d) for d in domains)
        return self.add(domains, per_domain, capacity, occ)

    def with_edges(self, dead_empty, dead_unusable, dead_full):
        """The row-level edges: saturating capacities inside regular domains, and three kinds of dead domain
        (``dead_empty`` gets no node rows at all)."""
        reg = self.regular
        self.add(reg[0:1], 1, 15)            # free 15: the nibble's largest value
        self.add(reg[1:2], 1, 16)            # free 16: the nibble saturates, the domain sum counts 16
        self.add(reg[2:3], 1, 65535)         # free 65 535
        self.add(reg[3:4], 1, 65535, 65534)  # free 1 beside free nodes
        self.add(reg[4:5], 1, 4, 9)          # occupancy above capacity: free 0
        self.add(reg[5:6], 1, 8, 0, R.NODE_HAS_TOPOLOGY)   # labelled, not schedulable: leaders claim through it
        self.add(reg[6:7], 1, 8, 0, R.NODE_SCHEDULABLE)    # schedulable, no topology label
        self.add([self.n_domains + 3], 1, 8)               # labelled with a domain that does not exist
        self.add(dead_unusable, 2, 8, 0, R.NODE_HAS_TOPOLOGY)
        self.add(dead_full, 1, 3, 3)
        self.add(dead_full, 1, 2, 7)
        return self

    def build(self, seed: int):
        cols = {k: np.concatenate(v) for k, v in self.cols.items()}
        perm = np.random.default_rng(seed).permutation(len(cols["domain"]))
        nodes = R.aligned_empty(len(perm), R.NODE_REC)
        nodes["domain_id"] = cols["domain"][perm]
        nodes["capacity"] = cols["capacity"][perm]
        nodes["flags"] = cols["flags"][perm]
        nodes["topo_value_hash"] = nodes["domain_id"].astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        return nodes, cols["occ"][perm].astype(np.uint32)


class Requests:
    """Request rows namespace by namespace; ``build`` keeps that order (grouped) or interleaves the rows."""

    def __init__(self, nodes: np.ndarray, n_domains: int, seed: int):
        self.rng = np.random.default_rng(seed)
        self.parts: list[np.ndarray] = []
        dom = nodes["domain_id"].astype(np.int64)
        fl = nodes["flags"]
        labelled = (fl & R.NODE_HAS_TOPOLOGY) != 0
        self.claims = {}  # node rows whose leaders claim their domain, by domain
        for n in np.flatnonzero(labelled & (dom < n_domains)):
            self.claims.setdefault(int(dom[n]), []).append(int(n))
        self.n_nodes = len(nodes)
        self.unusable_leader = np.flatnonzero(labelled & ((fl & R.NODE_SCHEDULABLE) == 0) & (dom < n_domains))
        self.unlabelled_leader = np.flatnonzero(~labelled)
        self.out_of_range_leader = np.flatnonzero(labelled & (dom >= n_domains))

    def _rows(self, ns, n):
        t = R.aligned_empty(n, R.PLACE_REQ)
        t["ns"] = ns
        t["priority"] = self.rng.integers(0, 1 << 63, size=n, dtype=np.uint64)
        t["group_key"] = self.rng.integers(0, 1 << 63, size=n, dtype=np.uint64)
        t["group"] = self.rng.integers(0, 1 << 31, size=n)
        t["size"] = self.rng.integers(1, 4, size=n)
        t["leader_node"] = R.NONE
        return t

    def unpinned(self, ns, n, ties: int = 0):
        """``n`` live unpinned requests of sizes 1-3; ``ties`` of them share their priority above bit 25."""
        t = self._rows(ns, n)
        if ties:
            at = self.rng.choice(n, size=ties, replace=False)
            t["priority"][at] = (np.uint64(0x1234567) << np.uint64(25)) | self.rng.integers(0, 1 << 25, size=ties, dtype=np.uint64)
        self.parts.append(t)
        return self

    def pinned(self, ns, domains, per_domain: int = 1):
        """Requests whose leaders sit on nodes of ``domains``: more than one per domain is a conflict."""
        nodes = [self.claims[int(d)][k % len(self.claims[int(d)])] for d in domains for k in range(per_domain)]
        t = self._rows(ns, len(nodes))
        t["leader_node"] = np.asarray(nodes, dtype=np.uint32)
        self.parts.append(t)
        return self

    def edges(self, ns):
        """Dead sizes, a size no domain holds (a live unpinned request: ``EDGE_LIVE``), and leaders on each
        kind of node that is not a plain usable one."""
        t = self._rows(ns, 7)
        t["size"][:3] = [0, -3, TOO_BIG]
        t["leader_node"][3] = self.unusable_leader[0]           # claims: labelled, not schedulable
        t["leader_node"][4] = self.unlabelled_leader[0]         # no claim
        t["leader_node"][5] = self.out_of_range_leader[0]       # no claim: no such domain
        t["leader_node"][6] = self.n_nodes + 5                  # no claim: no such node
        self.parts.append(t)
        return self

    def build(self, interleave: bool = False) -> np.ndarray:
        t = np.concatenate(self.parts)
        if interleave:
            t = t[self.rng.permutation(len(t))]
        out = R.aligned_empty(len(t), R.PLACE_REQ)
        out[:] = t
        return out


@dataclass
class Case:
    label: str
    doc: str
    nodes: np.ndarray
    occ: np.ndarray
    n_domains: int
    n_namespaces: int
    calls: list            # request tables, in call order (one geometry)
    entry: str             # "general" | "grouped" | "tick"
    edges: list = field(default_factory=list)  # (quantity, limit, "under" | "over"[, call index])
    contention: bool = False
    paths: list = field(default_factory=list)  # declared general paths, per call


def _regular(n_domains, dead=6):
    """Domains 0 .. n_domains - dead - 1 regular, the last ``dead`` split over the three dead kinds."""
    reg = list(range(n_domains - dead))
    d = list(range(n_domains - dead, n_domains))
    k = max(1, dead // 3)
    return reg, d[:k], d[k:2 * k], d[2 * k:]


def _node_table(n_domains, per_domain, seed, dead=6, capacity=6, occ=2):
    reg, empty, unusable, full = _regular(n_domains, dead)
    b = Nodes(n_domains).regular_domains(reg, per_domain, capacity, occ)
    return b.with_edges(empty, unusable, full).build(seed), reg


def _pad(b: Nodes, target: int):
    """Regular-domain rows until the table has exactly ``target`` rows."""
    have = sum(len(v) for v in b.cols["domain"])
    assert have <= target
    if target > have:
        extra = np.asarray(b.regular, dtype=np.int64)[np.arange(target - have) % len(b.regular)]
        b.cols["domain"].append(extra)
        for k, v in (("capacity", 6), ("occ", 2), ("flags", USABLE)):
            b.cols[k].append(np.full(len(extra), v))
    return b


def _sized_nodes(n_domains, n_nodes, seed, dead=6):
    reg, empty, unusable, full = _regular(n_domains, dead)
    b = Nodes(n_domains).regular_domains(reg, 1).with_edges(empty, unusable, full)
    return _pad(b, n_nodes).build(seed)


# --------------------------------------------------------------------------- #
# general form
# --------------------------------------------------------------------------- #
def g1_cluster_1024(sm_count):
    (nodes, occ), reg = _node_table(150, 3, seed=1)
    q = Requests(nodes, 150, seed=11)
    for v in range(4):
        q.unpinned(v, 256, ties=8)
    return Case("G1_cluster_1024", "1 024 live unpinned requests on the cluster: 8 per warp, 4 of them spilled",
                nodes, occ, 150, 4, [q.build(interleave=True)], "general",
                [("n_reqs", CLUSTER_WARPS * FEW_PER_WARP, "under"), ("per_warp", K_CACHE_Q, "over")],
                contention=True, paths=["cluster"])


def g1_grid_1025(sm_count):
    (nodes, occ), reg = _node_table(150, 3, seed=1)
    q = Requests(nodes, 150, seed=12)
    for v, n in enumerate((256, 256, 256, 257)):
        q.unpinned(v, n, ties=8)
    return Case("G1_grid_1025", "1 025 requests and no history: the grid", nodes, occ, 150, 4,
                [q.build(interleave=True)], "general",
                [("n_reqs", CLUSTER_WARPS * FEW_PER_WARP, "over"), ("expect_unpinned", CLUSTER_WARPS * PREDICTED_PER_WARP, "over")],
                contention=True, paths=["grid"])


def g2_misprediction(sm_count):
    """One geometry of 16 384 rows; only the pinned / unpinned mix changes between the calls."""
    n, n_dom, n_ns = 16384, 64, 8
    (nodes, occ), reg = _node_table(n_dom, 4, seed=2)
    quiet = Requests(nodes, n_dom, seed=21)
    per_ns = n // n_ns
    for v in range(n_ns):
        k_unp = 25
        quiet.unpinned(v, k_unp, ties=4).edges(v)
        rest = per_ns - k_unp - 7
        quiet.pinned(v, [reg[(v * 7 + i) % len(reg)] for i in range(rest)])
    burst = Requests(nodes, n_dom, seed=22)
    for v in range(n_ns):
        burst.unpinned(v, per_ns, ties=16)
    a, b = quiet.build(interleave=True), burst.build(interleave=True)
    return Case("G2_misprediction", "a quiet call, then a burst the quiet history sends to the cluster (128 per "
                "warp), then the same burst on the grid the burst's history picks", nodes, occ, n_dom, n_ns,
                [a, b, b], "general",
                [("expect_unpinned", CLUSTER_WARPS * PREDICTED_PER_WARP, "over", 0),
                 ("expect_unpinned", CLUSTER_WARPS * PREDICTED_PER_WARP, "under", 1),
                 ("n_reqs", MAX_CLUSTER_REQS, "under", 1), ("per_warp", K_CACHE_Q, "over", 1),
                 ("expect_unpinned", CLUSTER_WARPS * PREDICTED_PER_WARP, "over", 2)],
                contention=True, paths=["grid", "cluster", "grid"])


def g3_grid_overflow(sm_count):
    gw = sm_count * K_PLACE_WARPS
    n_unp = 5 * gw + 1
    n = max(MAX_CLUSTER_REQS + 16, n_unp + 4000)
    n_dom, n_ns = 256, 8
    (nodes, occ), reg = _node_table(n_dom, 2, seed=3)
    q = Requests(nodes, n_dom, seed=31)
    for v in range(n_ns):
        q.unpinned(v, n_unp // n_ns + (1 if v < n_unp % n_ns else 0), ties=8).edges(v)
    rest = n - n_unp - 7 * n_ns
    for v in range(n_ns):
        k = rest // n_ns + (1 if v < rest % n_ns else 0)
        q.pinned(v, [reg[(v * 13 + i) % 40] for i in range(k)])  # 40 claimed domains, the rest contested
    return Case("G3_grid_overflow", "more than 4 x GW live unpinned requests on the grid: 6 per warp",
                nodes, occ, n_dom, n_ns, [q.build(interleave=True)], "general",
                [("n_reqs", MAX_CLUSTER_REQS, "over"), ("per_warp", K_CACHE_Q, "over")],
                contention=True, paths=["grid"])


def _g4_nodes(n_nodes, seed):
    n_dom = 64
    nodes, occ = _sized_nodes(n_dom, n_nodes, seed)
    q = Requests(nodes, n_dom, seed=seed + 100)
    reg = list(range(n_dom - 6))
    for v in range(2):
        q.unpinned(v, 36, ties=4).edges(v).pinned(v, reg[v:v + 3], per_domain=2)
    return nodes, occ, n_dom, q.build(interleave=True)


def g4_nodes_65536(sm_count):
    nodes, occ, n_dom, reqs = _g4_nodes(65536, 41)
    return Case("G4_nodes_65536", "65 536 nodes: still the cluster", nodes, occ, n_dom, 2, [reqs], "general",
                [("n_nodes", MAX_CLUSTER_NODES, "under")], paths=["cluster"])


def g4_nodes_65537(sm_count):
    nodes, occ, n_dom, reqs = _g4_nodes(65537, 42)
    assert len(reqs) <= 100
    return Case("G4_nodes_65537", "65 537 nodes: the grid, at its 16-CTA floor for 100 requests", nodes, occ, n_dom, 2,
                [reqs], "general", [("n_nodes", MAX_CLUSTER_NODES, "over"), ("ctas", GRID_MIN_CTAS, "under")],
                paths=["grid"])


def _g4_hold(n_dom, seed):
    n_ns = 8
    reg, empty, unusable, full = _regular(n_dom, 30)
    b = Nodes(n_dom).regular_domains(reg[0::2], 2)  # every other domain has no node at all
    nodes, occ = b.with_edges(reg[1::2] + empty, unusable, full).build(seed)
    q = Requests(nodes, n_dom, seed=seed + 100)
    for v in range(n_ns):
        q.unpinned(v, 40, ties=4).edges(v).pinned(v, [reg[2 * (v + i)] for i in range(4)] + [unusable[v]], per_domain=2)
    return nodes, occ, q.build(interleave=True)


def g4_hold_65536(sm_count):
    nodes, occ, reqs = _g4_hold(8192, 43)
    return Case("G4_hold_65536", "8 namespaces x 8 192 domains: a holder table of exactly 65 536 keys, the cluster",
                nodes, occ, 8192, 8, [reqs], "general", [("hold", MAX_CLUSTER_HOLD, "under")], paths=["cluster"])


def g4_hold_65552(sm_count):
    nodes, occ, reqs = _g4_hold(8193, 44)
    return Case("G4_hold_65552", "8 namespaces x 8 193 domains (odd: the paired loads read the padded tail): "
                "65 552 holder keys, the grid", nodes, occ, 8193, 8, [reqs], "general",
                [("hold", MAX_CLUSTER_HOLD, "over")], paths=["grid"])


# --------------------------------------------------------------------------- #
# namespace form
# --------------------------------------------------------------------------- #
def n1_cache(sm_count):
    n_dom = 96
    (nodes, occ), reg = _node_table(n_dom, 2, seed=5)
    q = Requests(nodes, n_dom, seed=51)
    # namespace v: exactly this many live unpinned requests, competing for ~80 domains
    for v, n in enumerate((256, 257, 640)):
        q.pinned(v, reg[v * 5:v * 5 + 6], per_domain=2).unpinned(v, n - EDGE_LIVE, ties=12).edges(v)
    q.pinned(3, reg[:4]).edges(3)  # a namespace without live unpinned work
    t = q.build()
    t["ns"][-5:] = 6  # rows of a namespace that does not exist, at the end of the grouped table
    return Case("N1_cache", "namespaces of exactly 256, 257 and 640 live unpinned requests under tight capacity",
                nodes, occ, n_dom, 4, [t], "grouped", [("unpinned[0]", K_NS_CACHE, "under"), ("unpinned[1]", K_NS_CACHE, "over"),
                                                       ("unpinned[2]", K_NS_CACHE, "over")], contention=True)


KEEP_SCAN = K_NS_KEEP * K_NS_SCAN_THREADS  # positions of a namespace the scan form keeps in registers
KEEP_TWO_LEVEL = K_NS_KEEP * K_NS_THREADS
N2_ROWS = (KEEP_SCAN, KEEP_SCAN + 1, KEEP_TWO_LEVEL, KEEP_TWO_LEVEL + 1, KEEP_TWO_LEVEL + 300)


def n2_unkept(sm_count):
    """Rows 0 and 1 of a namespace claim domains a and b.  Past the kept positions: row 512 claims a with
    priority 0 (it wins, row 0 conflicts), row 513 claims b against row 1's priority 0 (it conflicts), rows
    1024 and 1100 claim a and b and conflict, and rows 1200 / 1201 claim a third domain c, 1201 winning."""
    n_dom = 80
    (nodes, occ), reg = _node_table(n_dom, 2, seed=6)
    q = Requests(nodes, n_dom, seed=61)
    for v, n in enumerate(N2_ROWS):
        a, b, c = reg[v * 3:v * 3 + 3]
        t = q._rows(v, n)
        q.edges(v)
        t[2:9] = q.parts.pop()
        claims = {0: (a, None), 1: (b, 0), 512: (a, 0), 513: (b, None), 1024: (a, None), 1100: (b, None),
                  1200: (c, None), 1201: (c, 0)}
        for p, (d, prio) in claims.items():
            if p < n:
                t["leader_node"][p] = q.claims[d][p % len(q.claims[d])]
                if prio is not None:
                    t["priority"][p] = prio
        q.parts.append(t)
    t = q.build()
    return Case("N2_unkept", "namespaces of 512 / 513 (scan) and 1 024 / 1 025 / 1 324 (two-level) rows, with pinned "
                "claims past the kept positions on domains claimed before them", nodes, occ, n_dom, 5, [t], "grouped",
                [("rows[0]", KEEP_SCAN, "under"), ("rows[1]", KEEP_SCAN, "over"), ("rows[2]", KEEP_TWO_LEVEL, "under"),
                 ("rows[3]", KEEP_TWO_LEVEL, "over")], contention=True)


def _n4(n_nodes, n_dom, seed):
    nodes, occ = _sized_nodes(n_dom, n_nodes, seed)
    q = Requests(nodes, n_dom, seed=seed + 100)
    reg = list(range(n_dom - 6))
    for v in range(3):
        q.pinned(v, reg[v * 4:v * 4 + 3], per_domain=2).unpinned(v, 300, ties=6).edges(v)
    return nodes, occ, q.build()


def _n4_case(label, n_nodes, n_dom, seed, over):
    nodes, occ, t = _n4(n_nodes, n_dom, seed)
    return Case(label, f"{n_nodes} nodes, {n_dom} domains: the scan form's word table "
                f"{'not staged' if over else 'staged'}", nodes, occ, n_dom, 3, [t], "grouped",
                [("scan_smem", STAGE_SMEM_LIMIT, "over" if over else "under")], contention=True)


def n4_stage_11520(sm_count):
    return _n4_case("N4_stage_11520", 11520, 48, 71, False)


def n4_stage_11521(sm_count):
    return _n4_case("N4_stage_11521", 11521, 48, 72, True)


def n4_stage_9728(sm_count):
    return _n4_case("N4_stage_9728", 9728, 1000, 73, False)


def n4_stage_9729(sm_count):
    return _n4_case("N4_stage_9729", 9729, 1000, 74, True)


N5_EXTRA = 5


def n5_ctas(sm_count):
    """CTA b takes namespaces b, b + G, ... (G = 2 x sm_count).  CTAs 0-4 have an empty or pinned-only first
    namespace and their work in the second; of the others, every third has work and the rest only empty
    or pinned-only namespaces."""
    g = 2 * sm_count
    n_ns = g + N5_EXTRA
    n_dom = 32
    (nodes, occ), reg = _node_table(n_dom, 2, seed=8)
    q = Requests(nodes, n_dom, seed=81)
    kind = {}
    for v in range(n_ns):
        b = v % g
        if v >= g or (b >= N5_EXTRA and b % 3 == 0):
            kind[v] = "work"
        else:
            kind[v] = "empty" if v % 2 == 0 else "pinned"
    for v in range(n_ns):
        if kind[v] == "work":
            q.unpinned(v, 30, ties=2).pinned(v, reg[v % 20:v % 20 + 2], per_domain=2)
        elif kind[v] == "pinned":
            q.pinned(v, reg[v % 20:v % 20 + 3], per_domain=2).edges(v)
            q.parts[-1]["size"][:3] = 0  # no live unpinned row: the dead sizes only
    t = q.build()
    c = Case("N5_ctas", "2 x sm_count + 5 namespaces: CTAs whose work comes late, CTAs without any", nodes, occ, n_dom,
             n_ns, [t], "grouped", [("n_namespaces", 2 * sm_count, "over")], contention=True)
    c.kind = kind
    return c


# --------------------------------------------------------------------------- #
# resident tick
# --------------------------------------------------------------------------- #
NS_DOMAIN_LIMIT = 5456  # the most domains the namespace form fits (place_ns_supported)


def _n3(n_dom, seed):
    nodes, occ = _sized_nodes(n_dom, n_dom + 600, seed)
    q = Requests(nodes, n_dom, seed=seed + 100)
    reg = list(range(n_dom - 6))
    for v in range(3):
        q.pinned(v, reg[v * 9:v * 9 + 4], per_domain=2).unpinned(v, 150, ties=6).edges(v)
    return nodes, occ, q.build()


def n3_domains_5456(sm_count):
    nodes, occ, t = _n3(NS_DOMAIN_LIMIT, 91)
    return Case("N3_domains_5456", "5 456 domains: the namespace form still fits", nodes, occ, NS_DOMAIN_LIMIT, 3, [t],
                "tick", [("smem", NS_SMEM_LIMIT, "under")])


def n3_domains_5457(sm_count):
    nodes, occ, t = _n3(NS_DOMAIN_LIMIT + 1, 92)
    return Case("N3_domains_5457", "5 457 domains: the tick falls back to the general form", nodes, occ,
                NS_DOMAIN_LIMIT + 1, 3, [t], "tick", [("smem", NS_SMEM_LIMIT, "over")])


BUILDERS = {f.__name__: f for f in (g1_cluster_1024, g1_grid_1025, g2_misprediction, g3_grid_overflow, g4_nodes_65536,
                                    g4_nodes_65537, g4_hold_65536, g4_hold_65552, n1_cache, n2_unkept, n4_stage_11520,
                                    n4_stage_11521, n4_stage_9728, n4_stage_9729, n5_ctas, n3_domains_5456,
                                    n3_domains_5457)}
GENERAL = [k for k in BUILDERS if k.startswith("g")]
NAMESPACE = [k for k in BUILDERS if k.startswith(("n1", "n2", "n4", "n5"))]
TICK = [k for k in BUILDERS if k.startswith("n3")]


def quantities(case: Case, sm_count: int, call: int = 0) -> dict:
    """Every quantity an edge of ``case`` names, from the mirror."""
    if case.entry == "general":
        return general_calls(case, sm_count)[call]
    v = ns_view(case, sm_count)
    q = {"smem": v["smem"], "scan_smem": v["scan_smem"], "n_namespaces": case.n_namespaces}
    for k in ("rows", "unpinned"):
        for i, x in enumerate(v[k]):
            q[f"{k}[{i}]"] = int(x)
    return q


# --------------------------------------------------------------------------- #
# what the spec gives, counted without solving it
# --------------------------------------------------------------------------- #
def dom_free(nodes, occ, n_domains) -> np.ndarray:
    usable = ((nodes["flags"] & USABLE) == USABLE) & (nodes["domain_id"] < n_domains)
    cap = nodes["capacity"].astype(np.int64)
    free = np.where(usable, np.maximum(cap - occ.astype(np.int64), 0), 0)
    return np.bincount(nodes["domain_id"][usable].astype(np.int64), weights=free[usable], minlength=n_domains).astype(np.int64)


def pinned_domain(nodes, n_domains, leader) -> int:
    if leader >= len(nodes):
        return -1
    nd = nodes[leader]
    return int(nd["domain_id"]) if (nd["flags"] & R.NODE_HAS_TOPOLOGY) and nd["domain_id"] < n_domains else -1


def expected_counts(nodes, occ, n_domains, n_namespaces, reqs) -> dict:
    """PLACED / CONFLICT / UNSCHEDULABLE rows of the spec, counted: a namespace's live unpinned requests of
    sizes every free domain holds share one feasible set, so min(requests, free unclaimed domains) of them
    hold a domain; pinned claims hold one domain each and the rest of a domain's claims conflict."""
    df = dom_free(nodes, occ, n_domains)
    biggest = int(df.max())
    smallest = int(df[df > 0].min())
    placed = conflict = unsched = 0
    for v in range(n_namespaces):
        rows = reqs[reqs["ns"] == v]
        pin = rows[rows["leader_node"] != R.NONE]
        claims = [pinned_domain(nodes, n_domains, int(x)) for x in pin["leader_node"]]
        claims = [d for d in claims if d >= 0]
        held = set(claims)
        placed += len(held)
        conflict += len(claims) - len(held)
        unp = rows[rows["leader_node"] == R.NONE]
        size = unp["size"].astype(np.int64)
        dead = (size < 1) | (size > biggest)
        fit = size[~dead]
        assert fit.size == 0 or fit.max() <= smallest, "the counting rule needs one feasible set per namespace"
        avail = int(((df > 0) & ~np.isin(np.arange(n_domains), list(held))).sum())
        won = min(len(fit), avail)
        placed += won
        unsched += int(dead.sum()) + len(fit) - won
    unsched += int((reqs["ns"] >= n_namespaces).sum())
    return {"placed": placed, "conflict": conflict, "unschedulable": unsched}


def flag_counts(out) -> dict:
    f = out["flags"]
    return {"placed": int(((f & R.PLACE_PLACED) != 0).sum()), "conflict": int(((f & R.PLACE_CONFLICT) != 0).sum()),
            "unschedulable": int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum())}


def _mix32(x):
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16)
    x = (x * np.uint32(0x85EBCA6B)).astype(np.uint32)
    x ^= x >> np.uint32(13)
    x = (x * np.uint32(0xC2B2AE35)).astype(np.uint32)
    x ^= x >> np.uint32(16)
    return x


def deferred_acceptance(nodes, occ, n_domains, n_namespaces, reqs) -> tuple[dict, np.ndarray]:
    """The domain level of the round as the kernels run it, every proposal of a round against the holders
    at its start: → (displacement rounds per namespace — rounds in which a claim met a holder — and the
    domain every live unpinned request ends on, -1 for none)."""
    df = dom_free(nodes, occ, n_domains)
    d_all = np.arange(n_domains, dtype=np.uint32)
    final = np.full(len(reqs), -1, np.int64)
    rounds = {}
    with np.errstate(over="ignore"):
        for v in range(n_namespaces):
            rows = np.flatnonzero(reqs["ns"] == v)
            held = {pinned_domain(nodes, n_domains, int(reqs["leader_node"][r])) for r in rows
                    if reqs["leader_node"][r] != R.NONE}
            live = rows[(reqs["leader_node"][rows] == R.NONE) & (reqs["size"][rows] >= 1)]
            if not len(live):
                continue
            keys = ((reqs["priority"][live] >> np.uint64(25)) << np.uint64(24)) | live.astype(np.uint64)
            size = reqs["size"][live].astype(np.int64)
            ok = (df[None, :] >= size[:, None]) & ~np.isin(np.arange(n_domains), list(held))[None, :]
            key_lo = (reqs["group_key"][live] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            h = _mix32(key_lo[:, None] ^ (d_all[None, :] * np.uint32(0x9E3779B1)).astype(np.uint32)) | np.uint32(1)
            h = np.where(ok, h, 0).astype(np.int64)
            INF = np.iinfo(np.uint64).max
            holder = np.full(n_domains, INF, np.uint64)
            holder_of = np.full(n_domains, -1, np.int64)
            own = np.full(len(live), -1, np.int64)
            dead = np.zeros(len(live), bool)
            disp = 0
            while True:
                act = np.flatnonzero((own < 0) & ~dead)
                if not len(act):
                    break
                score = np.where(holder[None, :] >= keys[act, None], h[act], 0)
                best = score.argmax(1)
                none = score.max(1) == 0
                dead[act[none]] = True
                act, best = act[~none], best[~none]
                if not len(act):
                    break
                met = False
                for i, d in zip(act, best):
                    if holder[d] != INF:
                        met = True
                    if keys[i] < holder[d]:
                        if holder_of[d] >= 0:
                            own[holder_of[d]] = -1
                        holder[d], holder_of[d], own[i] = keys[i], i, d
                disp += met
            rounds[v] = disp
            final[live] = own
    return rounds, final
