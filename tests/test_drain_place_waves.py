"""Drain placement waves (lwse_resident_drain_place_waves) without a GPU: the set locality rule against the literal
plan that solves every namespace for every probe, on the drain placement's worlds, both scopes, several key orders,
caps and constraint masks; LWS floor alone is the drain waves plan; the records against lwse.h."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from drain_place_waves_ref import EDGE_WORLDS, plan, probe
from drain_waves_ref import plan_literal as waves_literal
from lws_b200 import records as R
from test_drain_place_cost import WORLDS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASKS = {"floor": R.DPW_LWS_FLOOR, "stranded": R.DPW_STRANDED, "bumped": R.DPW_BUMPED,
         "default": R.DPW_LWS_FLOOR | R.DPW_STRANDED, "all": R.DPW_ALL}
CPU_WORLDS = ("built", "seed3")


def ids_of(world, by_domain, order):
    nodes, nd = world[4], world[5]
    ids = np.arange(nd if by_domain else len(nodes))
    if order == "reversed":
        ids = ids[::-1].copy()
    elif order == "random":
        ids = np.random.default_rng(7).permutation(ids)
    elif order == "by_cost":  # fewest groups restarted first, then by id
        from drain_budget_ref import drain_budget_cost_ref
        import oracle

        lws, groups, pst, pid, nodes, nd = world[:6]
        base = oracle.sweep_lws(lws, groups, pst, pid, nodes, 0)[:2]
        c = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, nd, base[1], by_domain)[ids]
        ids = ids[np.lexsort((ids, c["groups_restarted"]))]
    return ids


def same(a, b, skip=("namespaces_solved",)):
    ka, wa, ta = a
    kb, wb, tb = b
    if ta != tb or not np.array_equal(ka, kb):
        return False
    return all(np.array_equal(wa[f], wb[f]) for f in R.DRAIN_PLACE_WAVE.names if f not in skip)


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("order", ["given", "reversed", "random", "by_cost"])
@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", CPU_WORLDS)
def test_locality_equals_the_literal_plan(name, by_domain, order, mask):
    world = WORLDS[name]()
    ids = ids_of(world, by_domain, order)
    for cap in (1, 2, 64):
        lit = plan(world, ids, by_domain, cap, MASKS[mask], clause=None)
        fast = plan(world, ids, by_domain, cap, MASKS[mask], clause="exact")
        assert same(lit, fast), (name, by_domain, order, mask, cap)


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("name", list(EDGE_WORLDS))
def test_edge_worlds_locality_equals_the_literal_plan(name, mask):
    world, ids, _ = EDGE_WORLDS[name]()
    by_domain = name == "strand"
    for order in (ids, ids[::-1]):
        for cap in (1, 2, 64):
            assert same(plan(world, order, by_domain, cap, MASKS[mask], clause=None),
                        plan(world, order, by_domain, cap, MASKS[mask], clause="exact")), (name, mask, cap)


def test_sum_world_edges():
    """Nodes 0 and 1 drained together leave B (size 5) dom_free - sum - size = -1: bumped, not stranded, and the
    second key opens a wave under BUMPED; A (size 4) sits at exactly 0 and keeps its row."""
    world, ids, notes = EDGE_WORLDS["sum"]()
    reqs = world[7]
    keys, waves, tot = plan(world, ids, False, 64, R.DPW_BUMPED, clause=None)
    assert keys["wave"][0] == 0 and keys["wave"][1] == 1  # each alone fine, together B is bumped
    assert keys["alone"][0] == 0 and keys["alone"][1] == 0
    import oracle

    lws, groups, pst, pid, nodes, nd, occ, _, n_ns = world
    bg = oracle.sweep_lws(lws, groups, pst, pid, nodes, 0)[:2]
    bp = oracle.place(nodes, occ, nd, n_ns, reqs, threads=4)
    assert int(bp["leader_node"][notes["A"]]) == 2 and int(bp["leader_node"][notes["B"]]) == 2
    pl, _, _ = probe(world, bg, bp, [0, 1], False, None)
    assert pl["bumped"] == 1 and pl["stranded"] == 0  # B alone loses its domain; A (gap 0) keeps it
    assert keys["alone"][5] & R.DPW_STRANDED  # the pinned row of no namespace on node 5
    assert keys["unpinned"][0] == 1  # the pinned row on node 0, of no group


def test_sum_clause_mutations_give_wrong_plans():
    world, ids, _ = EDGE_WORLDS["sum"]()
    for mask in (R.DPW_BUMPED, R.DPW_ALL):
        lit = plan(world, ids, False, 64, mask, clause=None)
        assert same(lit, plan(world, ids, False, 64, mask, clause="exact"))
        for clause in ("per_node", "key_only"):
            assert not same(lit, plan(world, ids, False, 64, mask, clause=clause)), (mask, clause)


def test_strand_world_edges():
    """Domains 1 and 2 strand together (the second opens a wave); domain 5 strands alone but not with the wave
    holding domain 6, and lands on BREACHES_ALONE."""
    import oracle

    world, ids, _ = EDGE_WORLDS["strand"]()
    keys, waves, tot = plan(world, ids, True, 64, R.DPW_STRANDED, clause=None)
    assert keys["wave"].tolist()[:3] == [0, 1, 0]
    assert keys["status"][3] == R.DRAINW_BREACHES_ALONE and keys["alone"][3] == R.DPW_STRANDED
    lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns = world
    bg = oracle.sweep_lws(lws, groups, pst, pid, nodes, 0)[:2]
    bp = oracle.place(nodes, occ, nd, n_ns, reqs, threads=4)
    assert probe(world, bg, bp, [1, 6, 5], True, None)[0]["stranded"] == 0  # wave 0 with 5 added: no strand
    assert (waves["stranded"] == 0).all()


def test_cap_world_fills_every_wave():
    world, ids, _ = EDGE_WORLDS["cap"]()
    keys, waves, tot = plan(world, ids, False, 64, R.DPW_LWS_FLOOR | R.DPW_STRANDED, clause=None)
    assert tot["n_waves"] == 64 and keys["wave"][:64].tolist() == list(range(64))
    assert keys["status"][64] == R.DRAINW_NO_WAVE


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", CPU_WORLDS)
def test_floor_alone_is_the_drain_waves_plan(name, by_domain):
    world = WORLDS[name]()
    lws, groups, pst, pid, nodes, nd = world[:6]
    ids = ids_of(world, by_domain, "given")
    keys, waves, tot = plan(world, ids, by_domain, 64, R.DPW_LWS_FLOOR)
    wk, ww, wt = waves_literal(lws, groups, pst, pid, nodes, nd, ids, by_domain, 64)
    assert tot == wt
    for f in ("id", "wave", "status", "groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(keys[f], wk[f]), f
    for f in R.DRAIN_WAVE.names:
        if f != "reserved":
            assert np.array_equal(waves[f], ww[f]), f
    assert (waves["lws_breached"] == 0).all()


def test_records_match_header():
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("key %zu\\n", sizeof(lwse_drain_place_wave_key));',
             'printf("wave %zu\\n", sizeof(lwse_drain_place_wave));',
             'printf("query %zu\\n", sizeof(lwse_drain_place_waves_query));']
    for dt, c in ((R.DRAIN_PLACE_WAVE_KEY, "lwse_drain_place_wave_key"), (R.DRAIN_PLACE_WAVE, "lwse_drain_place_wave")):
        for f in dt.names:
            lines.append(f'printf("{c}.{f} %zu\\n", offsetof({c}, {f}));')
    lines += [f'printf("bits %u %u %u\\n", LWSE_DPW_LWS_FLOOR, LWSE_DPW_STRANDED, LWSE_DPW_BUMPED);', "return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {l.split(" ")[0]: l.split(" ")[1:] for l in out.strip().splitlines()}
    assert int(got["key"][0]) == R.DRAIN_PLACE_WAVE_KEY.itemsize == 48
    assert int(got["wave"][0]) == R.DRAIN_PLACE_WAVE.itemsize == 96
    assert int(got["query"][0]) == 64
    assert [int(x) for x in got["bits"]] == [R.DPW_LWS_FLOOR, R.DPW_STRANDED, R.DPW_BUMPED]
    for dt, c in ((R.DRAIN_PLACE_WAVE_KEY, "lwse_drain_place_wave_key"), (R.DRAIN_PLACE_WAVE, "lwse_drain_place_wave")):
        for f in dt.names:
            assert int(got[f"{c}.{f}"][0]) == dt.fields[f][1], (c, f)


def test_report_names_keys_and_verdicts():
    import copy

    from test_drain_place_cost import _enc

    enc = _enc(3)
    before = copy.deepcopy(vars(enc))
    names = {row: name for name, row in enc.node_index.items()}
    rows = sorted(names)[:3]
    keys = np.zeros(3, R.DRAIN_PLACE_WAVE_KEY)
    keys["id"] = rows
    keys["wave"] = [0, R.NONE, R.NONE]
    keys["status"] = [R.DRAINW_PLANNED, R.DRAINW_BREACHES_ALONE, R.DRAINW_NO_WAVE]
    keys["alone"] = [0, R.DPW_STRANDED | R.DPW_BUMPED, 0]
    rep = enc.drain_place_waves_report({"keys": keys, "waves": np.zeros(1, R.DRAIN_PLACE_WAVE)}, "nodes")
    assert rep["waves"] == [[names[rows[0]]]]
    assert rep["unplanned"] == [(names[rows[1]], "breaches_alone", ["stranded", "bumped"]),
                                (names[rows[2]], "no_wave", [])]
    assert list(before) == list(vars(enc))
