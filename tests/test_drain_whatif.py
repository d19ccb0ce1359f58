"""Drain what-if and drain cost (lwse_resident_drain_*) without a GPU: the one-pass cost restated in numpy
(tests/drain_ref.py) against the definition — the spec oracle's sweep with the drained nodes' pods deleting,
diffed against its sweep of the tables as they are — node by node and for sets of nodes; the informer's
helpers; the record layouts against lwse.h."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from drain_ref import (COST_OF, RESTART, TOTALS, drain_cost_ref, drain_whatif_ref, restart_pairs, set_totals_ref,
                       special_tables)
from lws_b200 import informer
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _node_world():
    from informer_world import make_world
    from node_world import NodeWorld

    items, cluster = make_world(21, n_lws=14, n_nodes=24)
    world = NodeWorld(items, cluster, 22, p_node=0.2)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=1.0, node_spare=6)
    for _ in range(25):
        world.step(enc)
    enc.flush()
    return enc


def _lifecycle_world():
    from informer_world import make_world
    from lifecycle_world import LifecycleWorld

    items, cluster = make_world(31, n_lws=16, n_nodes=20)
    world = LifecycleWorld(items, cluster, 32)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=1.0)
    for _ in range(25):
        world.step(enc)
    enc.flush()
    return enc


def _tables(name):
    if name == "special":
        return special_tables()
    enc = _node_world() if name == "node" else _lifecycle_world()
    lws, groups, pst, pid, _ = enc.full_tables()
    return lws, groups, pst, pid, enc.node_rec


WORLDS = ["special", "node", "lifecycle"]


@pytest.fixture(scope="module", params=WORLDS)
def world(request):
    lws, groups, pst, pid, nodes = _tables(request.param)
    base = oracle.sweep_lws(lws, groups, pst, pid, nodes)[:2]
    return request.param, (lws, groups, pst, pid, nodes), base


def test_cost_equals_the_whatif_of_each_node(world):
    """drain_cost_ref row n == the totals of the oracle what-if with D = {n}, for every node; the LWS rows never
    change."""
    _, (lws, groups, pst, pid, nodes), base = world
    cost = drain_cost_ref(lws, groups, pst, pid, len(nodes), base[1])
    assert np.array_equal(cost["pods"], R.occupancy_of(pid, len(nodes)))
    restarted_any = 0
    for n in range(len(nodes)):
        ref = drain_whatif_ref(lws, groups, pst, pid, nodes, [n], base=base)
        assert ref["lws_out"].tobytes() == base[0].tobytes()
        for k in TOTALS:
            assert int(cost[COST_OF[k]][n]) == ref[k], (n, k)
        restarted_any += ref["n_groups_restarted"]
    assert restarted_any > 0


def test_node_sets(world):
    """Multi-node sets D: the restart totals of the pairs against the oracle what-if, duplicates allowed."""
    name, (lws, groups, pst, pid, nodes), base = world
    rng = np.random.default_rng(5)
    n = len(nodes)
    sets = [[], list(range(n)), [0, 0, 1], list(rng.choice(n, size=max(2, n // 4), replace=False))]
    sets += [list(rng.choice(n, size=3)) for _ in range(4)]
    for d in sets:
        ref = drain_whatif_ref(lws, groups, pst, pid, nodes, d, base=base)
        got = set_totals_ref(lws, groups, pst, pid, n, base[1], d)
        for k, v in got.items():
            assert ref[k] == v, (name, d, k)
        if not d:
            assert ref["n_changed"] == 0 and ref["n_pods_evicted"] == 0


def test_special_table_reaches_every_case():
    """The purpose-built table: which groups each node restarts."""
    lws, groups, pst, pid, nodes = special_tables()
    base = oracle.sweep_lws(lws, groups, pst, pid, nodes)[:2]
    bf = base[1]["flags"]
    g, n = restart_pairs(lws, groups, pst, pid, len(nodes), base[1])
    by_group = {}
    for gi, ni in zip(g.tolist(), n.tolist()):
        by_group.setdefault(gi, set()).add(ni)
    assert by_group[0] == {0, 1, 2}        # spread over three nodes
    assert by_group[1] == {3, 4}           # two pods on one node count once
    assert by_group[2] == {5}
    assert by_group[3] == {6}              # the leader alone
    assert 4 not in by_group               # policy None
    assert by_group[5] == {0, 1, 2}        # AfterStart, open
    assert 6 not in by_group and 7 not in by_group  # pending gate closed
    assert by_group[8] == {0, 1, 2}        # annotation, open
    assert by_group[9] == {0, 1, 2}        # size != pods: pending, but OnPodRestart is not gated
    assert by_group[10] == {0, 7}          # the worker outside the range does not count
    assert bf[11] & RESTART and 11 not in by_group  # already restarting
    assert by_group[12] == {3, 2}          # the unparsable worker: RESTART_ERROR, not a restart
    assert by_group[13] == {3}             # stale chain: only the leader
    assert by_group[14] == {3, 2}          # the foreign worker does not belong
    assert by_group[15] == {1, 2} and by_group[16] == {1, 2}  # leader pod unscheduled: its workers still restart
    assert by_group[17] == {2}             # leader not found by name: only the leader pod itself
    assert by_group[18] == {6}
    assert (bf[-2:] & R.GOUT_BAD_TABLE).all() and len(groups) - 2 not in by_group and len(groups) - 1 not in by_group
    ref = drain_whatif_ref(lws, groups, pst, pid, nodes, [1], base=base)
    assert ref["n_leaders_evicted"] == 2   # the two BAD_TABLE rows name node 1
    assert not ((ref["after_all"]["flags"][[15, 16]] & RESTART) == 0).any()
    f12 = int(ref["after_all"]["flags"][12])  # its unparsable worker is on node 1, its restart nodes are not
    assert f12 & R.GOUT_RESTART_ERROR and not f12 & RESTART


def test_informer_helpers():
    enc = _node_world()
    names = sorted(enc.node_index)[:3]
    rows = enc.whatif_drain(names + names[:1])
    assert rows.dtype == np.uint32 and rows.tolist() == sorted({enc.node_index[n] for n in names})
    lws, groups, pst, pid, _ = enc.full_tables()
    base = oracle.sweep_lws(lws, groups, pst, pid, enc.node_rec)[:2]
    ref = drain_whatif_ref(lws, groups, pst, pid, enc.node_rec, rows, base=base)
    segs = enc.drain_place_query(ref, names)
    (t0, nrows, nvals), (t1, rrows, rvals) = segs
    assert t0 == R.TABLE_NODES and sorted(nrows.tolist()) == rows.tolist()
    assert not (nvals["flags"] & R.NODE_SCHEDULABLE).any()
    assert t1 == R.TABLE_PLACE_REQS and rvals.dtype == R.PLACE_REQ and (rvals["leader_node"] == R.NONE).all()
    hit = ((ref["before"]["flags"] & RESTART) == 0) & ((ref["after"]["flags"] & RESTART) != 0)
    owned = np.flatnonzero(enc._group_lws[: len(groups)] >= 0)
    want = set(ref["rows"][hit].tolist()) | set(owned[np.isin(groups["leader_node"][owned], rows)].tolist())
    assert rrows.tolist() == sorted(want)
    for f in R.PLACE_REQ.names:
        if f != "leader_node":
            assert np.array_equal(rvals[f], enc.reqs[rrows][f]), f


def test_records_match_header():
    """Sizes and offsets of lwse_drain_cost and lwse_drain_whatif, via a gcc-compiled probe."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("lwse_drain_cost %zu\\n", sizeof(lwse_drain_cost));',
             'printf("lwse_drain_whatif %zu\\n", sizeof(lwse_drain_whatif));']
    for f in R.DRAIN_COST.names:
        lines.append(f'printf("lwse_drain_cost.{f} %zu\\n", offsetof(lwse_drain_cost, {f}));')
    for f, _ in R.DrainWhatIf._fields_:
        lines.append(f'printf("lwse_drain_whatif.{f} %zu\\n", offsetof(lwse_drain_whatif, {f}));')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = dict(l.split() for l in out.strip().splitlines())
    assert int(got["lwse_drain_cost"]) == R.DRAIN_COST.itemsize == 32
    for f in R.DRAIN_COST.names:
        assert int(got[f"lwse_drain_cost.{f}"]) == R.DRAIN_COST.fields[f][1], f
    assert int(got["lwse_drain_whatif"]) == C.sizeof(R.DrainWhatIf)
    for f, _ in R.DrainWhatIf._fields_:
        assert int(got[f"lwse_drain_whatif.{f}"]) == getattr(R.DrainWhatIf, f).offset, f
