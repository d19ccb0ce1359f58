"""Drain placement (lwse_resident_drain_place_cost) without a GPU: the locality rule of DESIGN.md §3.5 — solving
only the namespaces of rules (a) and (b) — against the definition that solves every namespace, on seeded informer
worlds and on a built world of the rule's edges; the definition against the informer's own three-step composition
(``drain_place_query`` → ``whatif_ref``), which pins U_k's statement through the ``group`` field; the informer's
report; the record layout against lwse.h."""
import copy
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from drain_place_ref import composition_ref, drain_place_ref
from drain_ref import special_tables
from lws_b200 import informer
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def built_world():
    """special_tables' objects (one group per restart-verdict case) on 8 nodes of 3 usable domains, with request
    rows at the locality rule's edges: holders on every node, two pinned rows on one domain (the CONFLICT row is
    promoted when the holder's leader drains), restarted groups whose leader is elsewhere, dead rows, rows of no
    namespace, nodes in no domain or beyond n_domains, a cordoned node and a full one (capacity = its pods, so
    the engine sees it full too).  Free slots [4, 3, 2, 0, 2, 8, 6, 6]: domain 0 (nodes 0 and 1) has 7, the
    others 2, so one unpinned row of each size 3 .. 7, alone in its namespace, lands in domain 0 with
    dom_free - free[n] for the node it did not choose (4 or 3) just at, one below, or further below its size:
    the capacity clause of rule (b).  → (lws, groups, pst, pid, nodes, n_domains, occ, reqs, n_ns)."""
    lws, groups, pst, pid, nodes = special_tables()
    nodes = nodes.copy()
    n_domains = 4  # domain 3 has no node
    occ = R.occupancy_of(pid, len(nodes)).astype(np.uint32)
    nodes["domain_id"] = [0, 0, 1, 1, 2, 2, R.NONE, 9]
    nodes["capacity"] = occ + np.array([4, 3, 2, 0, 2, 8, 6, 6], np.uint32)  # node 3: full
    nodes["flags"] |= np.uint16(R.NODE_SCHEDULABLE | R.NODE_HAS_TOPOLOGY)
    nodes["flags"][5] &= ~np.uint16(R.NODE_SCHEDULABLE)  # cordoned already
    rng = np.random.default_rng(3)
    rows = []

    def req(ns, size, leader=R.NONE, group=R.NONE):
        rows.append((int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 62)), group, ns, size, leader))

    for n in range(8):
        req(0, 2, leader=n, group=n % len(groups))  # a holder on every node (nodes 6 and 7: no domain)
    req(0, 1, leader=0)                             # a second pinned row on domain 0: CONFLICT until 0's drain
    for size in (1, 2, 3, 4, 5, 6, 7, 9):           # unpinned rows around the domains' free slots
        req(1, size)
        req(2, size)
    req(1, 0, leader=2)                             # dead pinned row
    req(2, -1)                                      # dead unpinned row
    for g in range(len(groups)):                    # restarted groups whose leader sits on another key
        req(2, 1, leader=(g + 3) % 8, group=g)
    for size in (3, 4, 5, 6, 7):                    # the capacity clause, one row per namespace
        req(size, size)
    req(8, 2, leader=4)                             # a row of no namespace, pinned on a drained key
    reqs = R.aligned_empty(len(rows), R.PLACE_REQ)
    for i, r in enumerate(rows):
        reqs[i] = r
    return lws, groups, pst, pid, nodes, n_domains, occ, reqs, 8


def big_namespace_world():
    """The built world plus two large namespaces: 257 rows pinned on node 0 (kNsCache + 1 unpinned by its drain)
    among 1 025 rows (kNsKeep x 512 + 1), and 256 pinned on node 1 among 1 024."""
    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = built_world()
    rng = np.random.default_rng(9)
    extra = []
    for ns, n_rows, n_pinned, node in ((n_ns, 1025, 257, 0), (n_ns + 1, 1024, 256, 1)):
        x = R.aligned_empty(n_rows, R.PLACE_REQ)
        x["priority"] = rng.integers(0, 1 << 62, size=n_rows, dtype=np.uint64)
        x["group_key"] = rng.integers(0, 1 << 62, size=n_rows, dtype=np.uint64)
        x["group"] = R.NONE
        x["ns"] = ns
        x["size"] = rng.integers(1, 3, size=n_rows)
        x["leader_node"] = R.NONE
        x["leader_node"][:n_pinned] = node
        extra.append(x)
    reqs = reqs.copy()
    reqs["ns"][reqs["ns"] >= n_ns] = n_ns + 2  # (the row of no namespace stays outside)
    all_reqs = R.aligned_empty(len(reqs) + sum(len(x) for x in extra), R.PLACE_REQ)
    all_reqs[: len(reqs)] = reqs
    all_reqs[len(reqs):] = np.concatenate(extra)
    return lws, groups, pst, pid, nodes, nd, occ, all_reqs, n_ns + 2


@functools.lru_cache(maxsize=None)
def _enc(seed):
    from informer_world import make_world

    items, cluster = make_world(seed, n_lws=14, n_nodes=28)
    return informer.IncrementalEncoder(items, cluster, "zone")


def _enc_world(seed):
    enc = _enc(seed)
    lws, groups, pst, pid, reqs = enc.full_tables()
    return lws, groups, pst, pid, enc.node_rec, enc.n_domains, R.occupancy_of(pid, len(enc.node_rec)), reqs, enc.n_namespaces


WORLDS = {"built": built_world, "big_namespaces": big_namespace_world, "seed3": lambda: _enc_world(3),
          "seed11": lambda: _enc_world(11)}


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", list(WORLDS))
def test_pruned_equals_the_definition(name, by_domain):
    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = WORLDS[name]()
    full = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, by_domain)
    pruned = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, by_domain, pruned=True)
    fields = [f for f in R.DRAIN_PLACE_COST.names if f not in ("namespaces_solved", "reserved")]
    for f in fields:
        assert np.array_equal(full[f], pruned[f]), (name, f)
    assert (pruned["namespaces_solved"] <= n_ns).all()
    if name == "built":  # the edges happen: restarts, unpinning, changed rows
        assert full["groups_restarted"].any() and full["unpinned"].any() and full["n_changed"].any()
    if name == "big_namespaces":
        if by_domain:
            assert full["unpinned"][0] >= 513
        else:
            assert full["unpinned"][0] >= 257 and full["unpinned"][1] >= 256


def test_capacity_clause_is_needed_and_exact():
    """Rule (b)'s node clause dom_free[d] - free[n] < size at its edge: the built world has holders in domain 0
    with dom_free - free[n] at their size ("just at": not solved, and draining n leaves them), one below it and
    further below (solved, and draining n moves them).  Without the clause, or with it one tighter, the pruned
    answer is wrong for some node key; with it, exact."""
    import oracle

    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = built_world()
    base = oracle.place(nodes, occ, nd, n_ns, reqs, threads=4)
    free = nodes["capacity"].astype(np.int64) - occ
    free[5] = 0  # (cordoned)
    gaps = set()
    for r in np.flatnonzero((reqs["ns"] >= 3) & (reqs["ns"] < n_ns)):
        assert base["domain_id"][r] == 0 and base["flags"][r] & R.PLACE_PLACED
        other = 1 - int(base["leader_node"][r])
        gaps.add(int(free[0] + free[1] - free[other]) - int(reqs["size"][r]))
    assert {0, -1, -2} <= gaps  # just at, one below, two below
    full = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns)
    exact = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, pruned=True)
    fields = [f for f in R.DRAIN_PLACE_COST.names if f not in ("namespaces_solved", "reserved")]
    assert all(np.array_equal(full[f], exact[f]) for f in fields)
    for clause in ("dropped", "tight"):
        wrong = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, pruned=True, capacity_clause=clause)
        assert any(not np.array_equal(full[f], wrong[f]) for f in ("n_changed", "n_lost", "n_moved", "stranded")), clause


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("seed", [3, 11])
def test_definition_equals_the_informer_composition(seed, by_domain):
    enc = _enc(seed)
    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = _enc_world(seed)
    ref = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, by_domain)
    comp = composition_ref(enc, by_domain)
    names = {row for row in enc.node_index.values()}
    for k in range(len(ref)):
        nk = [k] if not by_domain else np.flatnonzero(nodes["domain_id"] == k).tolist()
        if not any(n in names for n in nk):
            continue
        assert ref[k].tobytes() == comp[k].tobytes(), (seed, by_domain, k)


def test_report_names_the_keys():
    enc = _enc(3)
    before = copy.deepcopy(vars(enc))
    rows = np.zeros(len(enc.node_rec), R.DRAIN_PLACE_COST)
    rows["stranded"][2] = 4
    rep = enc.drain_place_report(rows, "nodes")
    names = {row: name for name, row in enc.node_index.items()}
    assert rep[2]["node"] == names.get(2) and rep[2]["stranded"] == 4 and "reserved" not in rep[2]
    drows = np.zeros(enc.n_domains, R.DRAIN_PLACE_COST)
    rep = enc.drain_place_report(drows, "domains")
    assert {r["topology"] for r in rep} <= set(enc.domain_values) | {None}
    with pytest.raises(ValueError):
        enc.drain_place_report(drows, "racks")
    assert list(before) == list(vars(enc))


def test_record_matches_header():
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("size %zu\\n", sizeof(lwse_drain_place_cost));']
    for f in R.DRAIN_PLACE_COST.names:
        lines.append(f'printf("{f} %zu\\n", offsetof(lwse_drain_place_cost, {f}));')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {l.split(" ")[0]: int(l.split(" ")[1]) for l in out.strip().splitlines()}
    assert got["size"] == R.DRAIN_PLACE_COST.itemsize == 64
    for f in R.DRAIN_PLACE_COST.names:
        assert got[f] == R.DRAIN_PLACE_COST.fields[f][1], f
