"""Drain waves (lwse_resident_drain_waves) without a GPU: the fast reference (restart pairs and per-(LWS, wave)
counters, tests/drain_waves_ref.py) against the literal one (first-fit where every probe is the set-form drain
budget) on seeded worlds, both scopes, four key orders and three wave caps; the edges world case by case; every
wave row against the set form over its ids; the record layouts against lwse.h."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from drain_budget_ref import domain_nodes, drain_budget_cost_ref, drain_budget_ref
from drain_waves_ref import (orders, plan_fast, plan_literal, plan_threads, wave_row_of_set, waves_edges_world,
                             waves_world)
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = R.NONE


@functools.lru_cache(maxsize=None)
def _world(name):
    """(lws, groups, pst, pid, nodes, n_domains, sweep flags, base)."""
    if name == "edges":
        w, _, _ = waves_edges_world()
        t = (w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, 0)
    else:
        seed = {"seed5": 5, "seed6": 6}[name]
        w = waves_world(n_lws=120 if seed == 5 else 160, n_nodes=96 if seed == 5 else 64, seed=seed)
        t = (w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, w.flags & R.SWEEP_GANG)
    return t + (oracle.sweep_lws(*t[:5], t[6])[:2],)


def _plans(name, by_domain, ids, max_waves):
    lws, groups, pst, pid, nodes, nd, fl, base = _world(name)
    fast = plan_fast(lws, base[0], groups, pst, pid, nodes, nd, base[1], ids, by_domain, max_waves)
    lit = plan_literal(lws, groups, pst, pid, nodes, nd, ids, by_domain, max_waves, flags=fl, base=base)
    return fast, lit


def check_waves(name, by_domain, ids, plan):
    """Every wave row equals the set form over its ids, with nothing breached; the alone columns equal the
    per-key drain budget."""
    lws, groups, pst, pid, nodes, nd, fl, base = _world(name)
    keys, waves, totals = plan
    cost = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, nd, base[1], by_domain)
    for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(keys[f], cost[f][np.asarray(ids, dtype=np.int64)]), f
    assert totals["n_waves"] == len(waves) and sum(totals[k] for k in ("n_planned", "n_breaches_alone", "n_no_wave")) == len(ids)
    for w in range(len(waves)):
        ws = keys["id"][keys["wave"] == w].astype(np.int64)
        d = domain_nodes(nodes, nd, ws) if by_domain else ws
        rows, tot = drain_budget_ref(lws, groups, pst, pid, nodes, d, fl, base=base)
        assert tot["n_breached"] == 0
        assert waves[w].tobytes() == wave_row_of_set(rows, tot, len(ws)).tobytes(), w
    assert ((keys["wave"] == NONE) == (keys["status"] != R.DRAINW_PLANNED)).all()


@pytest.mark.parametrize("max_waves", [1, 2, 64])
@pytest.mark.parametrize("order", ["given", "reversed", "by_cost", "random"])
@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", ["seed5", "seed6"])
def test_references_agree(name, by_domain, order, max_waves):
    lws, groups, pst, pid, nodes, nd, fl, base = _world(name)
    cost = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, nd, base[1], by_domain)
    ids = orders(np.arange(len(cost)), cost)[order]
    fast, lit = _plans(name, by_domain, ids, max_waves)
    for a, b in zip(fast[:2], lit[:2]):
        assert a.tobytes() == b.tobytes()
    assert fast[2] == lit[2]
    check_waves(name, by_domain, ids, fast)


def test_worlds_cover_every_outcome():
    """Across the seeded worlds at cap 2: planned keys, keys breaching alone, keys without a wave, shared waves."""
    seen = {"planned": 0, "alone": 0, "no_wave": 0, "shared": 0, "waves": 0}
    for name in ("seed5", "seed6"):
        for by_domain in (False, True):
            nk = _world(name)[5] if by_domain else len(_world(name)[4])
            lws, groups, pst, pid, nodes, nd, fl, base = _world(name)
            keys, waves, tot = plan_fast(lws, base[0], groups, pst, pid, nodes, nd, base[1], np.arange(nk), by_domain, 2)
            seen["planned"] += tot["n_planned"]
            seen["alone"] += tot["n_breaches_alone"]
            seen["no_wave"] += tot["n_no_wave"]
            seen["shared"] += int((waves["n_keys"] > 1).sum())
            seen["waves"] += tot["n_waves"]
    assert all(v > 0 for v in seen.values()), seen


@functools.lru_cache(maxsize=None)
def _edges_plan(max_waves, by_domain=False):
    _, ids, notes = waves_edges_world()
    fast, lit = _plans("edges", by_domain, ids, max_waves)
    return ids, notes, fast, lit


@pytest.mark.parametrize("max_waves", [1, 2, 64])
@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
def test_edges_references_agree(max_waves, by_domain):
    ids, _, fast, lit = _edges_plan(max_waves, by_domain)
    assert fast[0].tobytes() == lit[0].tobytes() and fast[1].tobytes() == lit[1].tobytes() and fast[2] == lit[2]
    check_waves("edges", by_domain, ids, fast)


def _outcome(max_waves=64):
    ids, notes, (keys, waves, tot), _ = _edges_plan(max_waves)
    pos = {k: i for i, k in enumerate(ids)}
    return {lab: [keys[pos[k]] for k in ks] for lab, ks in notes.items()}, waves, tot


def test_edges_pairs_per_pass():
    """A key with exactly as many (pair, column) items as the plan kernel takes per pass fits its slack; one more
    pair, in a second pass, breaches alone."""
    o, _, _ = _outcome()
    T = plan_threads()
    (ex,), (ov,) = o["pair_exact"], o["pair_over"]
    assert ex["groups_restarted"] == T and ex["status"] == R.DRAINW_PLANNED and ex["wave"] == 0
    assert ov["groups_restarted"] == T + 1 and ov["status"] == R.DRAINW_BREACHES_ALONE and ov["lws_breached"] == 1


def test_edges_below_floor():
    """A row already below its floor: its ready group's key breaches alone, its not-ready group's key plans."""
    o, _, _ = _outcome()
    ready, not_ready = o["below"]
    assert ready["status"] == R.DRAINW_BREACHES_ALONE and ready["wave"] == NONE and ready["ready_restarted"] == 1
    assert not_ready["status"] == R.DRAINW_PLANNED and not_ready["ready_restarted"] == 0 and not_ready["lws_touched"] == 1


def test_edges_shared_group():
    """Two keys restarting the same single group of an object with slack 1 share a wave; a third key restarting
    another group of it does not."""
    o, waves, _ = _outcome()
    a, b = o["shared"]
    (c,) = o["third"]
    assert a["wave"] == b["wave"] != NONE and c["wave"] not in (NONE, a["wave"])
    assert a["lws_breached"] == b["lws_breached"] == c["lws_breached"] == 0


def test_edges_never_a_constraint():
    """A non-member group and a NOT_EVALUATED row of slack 0 constrain nothing; the non-member counts in the totals;
    a percentage maxUnavailable above 100 at replicas 2^30 gives floor 0 (mu in 64 bits); a key without pods plans."""
    o, waves, _ = _outcome()
    for lab in ("foreign", "unevaluated", "pct", "empty"):
        (k,) = o[lab]
        assert k["status"] == R.DRAINW_PLANNED and k["lws_breached"] == 0, lab
    (f,) = o["foreign"]
    assert f["groups_restarted"] == 1 and f["lws_touched"] == 0
    (u,) = o["unevaluated"]
    assert u["lws_touched"] == 1 and u["ready_restarted"] == 1
    (e,) = o["empty"]
    assert e["groups_restarted"] == 0 and e["wave"] == 0


@pytest.mark.parametrize("max_waves", [2, 64])
def test_edges_wave_cap(max_waves):
    """65 keys on 65 ready groups of one object with slack 1: key i opens wave i up to the cap, the rest are NO_WAVE
    (the top bit of a 64-bit wave mask at cap 64), while the breaching keys stay BREACHES_ALONE."""
    o, waves, tot = _outcome(max_waves)
    cap = o["cap"]
    for i, k in enumerate(cap):
        if i < max_waves:
            assert k["status"] == R.DRAINW_PLANNED and k["wave"] == i, i
        else:
            assert k["status"] == R.DRAINW_NO_WAVE and k["wave"] == NONE, i
    assert tot["n_waves"] == max_waves and len(waves) == max_waves
    assert o["pair_over"][0]["status"] == o["below"][0]["status"] == R.DRAINW_BREACHES_ALONE


def test_records_match_header():
    """Sizes and offsets of lwse_drain_wave_key, lwse_drain_wave and lwse_drain_waves_query, and the constants, via
    a gcc-compiled probe."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){"]
    for s, names in (("lwse_drain_wave_key", R.DRAIN_WAVE_KEY.names), ("lwse_drain_wave", R.DRAIN_WAVE.names),
                     ("lwse_drain_waves_query", [f for f, _ in R.DrainWavesQuery._fields_])):
        lines.append(f'printf("{s} %zu\\n", sizeof({s}));')
        for f in names:
            lines.append(f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));')
    lines.append('printf("consts %u %u %u %u\\n", LWSE_DRAIN_WAVES_MAX, LWSE_DRAINW_PLANNED, LWSE_DRAINW_BREACHES_ALONE, '
                 'LWSE_DRAINW_NO_WAVE);')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {l.split(" ", 1)[0]: l.split(" ", 1)[1] for l in out.strip().splitlines()}
    assert int(got["lwse_drain_wave_key"]) == R.DRAIN_WAVE_KEY.itemsize == 32
    assert int(got["lwse_drain_wave"]) == R.DRAIN_WAVE.itemsize == 48
    for s, dt in (("lwse_drain_wave_key", R.DRAIN_WAVE_KEY), ("lwse_drain_wave", R.DRAIN_WAVE)):
        for f in dt.names:
            assert int(got[f"{s}.{f}"]) == dt.fields[f][1], f
    assert int(got["lwse_drain_waves_query"]) == C.sizeof(R.DrainWavesQuery)
    for f, _ in R.DrainWavesQuery._fields_:
        assert int(got[f"lwse_drain_waves_query.{f}"]) == getattr(R.DrainWavesQuery, f).offset, f
    assert got["consts"] == f"{R.DRAIN_WAVES_MAX} {R.DRAINW_PLANNED} {R.DRAINW_BREACHES_ALONE} {R.DRAINW_NO_WAVE}"


def test_informer_report():
    """drain_waves_report names each wave's nodes (topology values) in query order and lists the unplanned keys."""
    from test_drain_whatif import _node_world

    enc = _node_world()
    names = {row: name for name, row in enc.node_index.items()}
    rows = sorted(names)[:4]
    keys = np.zeros(4, R.DRAIN_WAVE_KEY)
    keys["id"] = rows
    keys["wave"] = [1, 0, NONE, 1]
    keys["status"] = [R.DRAINW_PLANNED, R.DRAINW_PLANNED, R.DRAINW_NO_WAVE, R.DRAINW_PLANNED]
    rep = enc.drain_waves_report({"keys": keys, "waves": np.zeros(2, R.DRAIN_WAVE)})
    assert rep["waves"] == [[names[rows[1]]], [names[rows[0]], names[rows[3]]]]
    assert rep["unplanned"] == [(names[rows[2]], "no_wave")]
    vals = {d: v for v, d in enc._domain_ids.items()}
    keys["id"] = [0, 1, 2, 3]
    keys["status"][2] = R.DRAINW_BREACHES_ALONE
    rep = enc.drain_waves_report({"keys": keys, "waves": np.zeros(2, R.DRAIN_WAVE)}, "domains")
    assert rep["waves"][0] == [vals.get(1)] and rep["unplanned"] == [(vals.get(2), "breaches_alone")]
    with pytest.raises(ValueError):
        enc.drain_waves_report({"keys": keys, "waves": []}, "racks")
