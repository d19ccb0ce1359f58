"""Rollout placement waves (lwse_resident_rollout_place_waves) without a GPU: the per-namespace plan against the
literal global first-fit on seeded fuzz worlds and on every edge world, in both query forms, four key orders, caps
1, 2 and 64 and every constraint mask; each edge on its side; three wrong statements caught; the per-namespace
numbering of argument (1); the records against lwse.h; the informer report and the argument checks."""
import os
import re

import numpy as np
import pytest

from lws_b200 import records as R
from rollout_place_ref import fuzz_world, proposals
from rollout_place_waves_ref import (ALL_MASKS, edge_queries, key_orders, rollout_place_waves_ref, same_plan, tie_world,
                                     waves_world)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS = (1, 2, 64)


def fuzz_query(w, seed, n=48):
    """Distinct exclusive objects (and a few that are not), in the namespace synth deals them to."""
    rng = np.random.default_rng(seed)
    excl = np.flatnonzero(w.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY)
    other = np.flatnonzero(~w.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY)
    rows = np.concatenate([rng.choice(excl, min(n, len(excl)), replace=False), rng.choice(other, 4, replace=False)])
    rows = rng.permutation(rows).astype(np.uint32)
    return rows, (rows.astype(np.int64) % w.n_ns).astype(np.uint32)


def _both(w, rows, ns, recs, cap, mask):
    a = rollout_place_waves_ref(w, rows, ns, recs, max_waves=cap, constraints=mask)
    b = rollout_place_waves_ref(w, rows, ns, recs, max_waves=cap, constraints=mask, mode="ns")
    assert same_plan(a, b), (cap, mask, a["keys"], b["keys"], a["waves"], b["waves"])
    return a


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ns_plan_equals_the_literal_plan_on_fuzz_worlds(seed):
    w = fuzz_world(seed)
    rows, ns = fuzz_query(w, seed)
    planned = 0
    for recs in (None, proposals(w.lws, rows, seed)[1]):
        surge = rollout_place_waves_ref(w, rows, ns, recs, mode="ns")["alone_rows"]["surge"]
        for name, o in key_orders(len(rows), surge, seed).items():
            for cap in CAPS:
                for mask in ALL_MASKS:
                    a = _both(w, rows[o], ns[o], None if recs is None else recs[o], cap, mask)
                    planned += a["n_planned"]
    assert planned > 0


@pytest.fixture(scope="module")
def edge():
    w, rows = waves_world()
    return w, rows, edge_queries(w, rows)


def test_ns_plan_equals_the_literal_plan_on_the_edge_worlds(edge):
    w, _, q = edge
    for label, (rows, ns, recs) in q.items():
        surge = rollout_place_waves_ref(w, rows, ns, recs, mode="ns")["alone_rows"]["surge"]
        for o in key_orders(len(rows), surge, 7).values():
            for cap in CAPS:
                for mask in ALL_MASKS:
                    _both(w, rows[o], ns[o], None if recs is None else recs[o], cap, mask)
    tw, rows, ns, recs = tie_world()
    for cap in CAPS:
        for mask in ALL_MASKS:
            _both(tw, rows, ns, recs, cap, mask)
            _both(tw, rows[::-1].copy(), ns, recs[::-1].copy(), cap, mask)


def _plan(w, q, label, cap=64, mask=R.RPW_STRANDED):
    rows, ns, recs = q[label]
    p = rollout_place_waves_ref(w, rows, ns, recs, max_waves=cap, constraints=mask)
    return [(int(k["wave"]) if k["wave"] != R.NONE else None, int(k["status"]), int(k["alone"])) for k in p["keys"]], p


def test_each_edge_lands_on_its_side(edge):
    w, rows, q = edge
    P, T, NW, NS = R.ROLLW_PLANNED, R.ROLLW_TRIGGERS_ALONE, R.ROLLW_NO_WAVE, R.ROLLW_NOT_SOLVED
    # two objects that each need the last 3 domains: clean alone, the second opens wave 1; in two namespaces they share
    keys, p = _plan(w, q, "pair_one_ns")
    assert keys == [(0, P, 0), (1, P, 0)] and p["n_waves"] == 2 and p["waves"]["surge"].tolist() == [3, 3]
    keys, p = _plan(w, q, "pair_two_ns")
    assert keys == [(0, P, 0), (0, P, 0)] and p["waves"]["namespaces"].tolist() == [2]
    # three of them under a cap of 2: the third gets no wave while another namespace still plans into wave 0
    keys, p = _plan(w, q, "cap", cap=2)
    assert keys == [(0, P, 0), (1, P, 0), (None, NW, 0), (0, P, 0)] and p["n_no_wave"] == 1
    # strands alone next to an open wave: TRIGGERS_ALONE; with stranding allowed it joins that wave
    keys, _ = _plan(w, q, "strands_alone")
    assert keys == [(0, P, 0), (None, T, R.RPW_STRANDED), (0, P, 0)]
    keys, _ = _plan(w, q, "strands_alone", mask=R.RPW_BUMPED)
    assert keys[1] == (0, P, R.RPW_STRANDED)
    # surge rows that bump other rows, or the object's own: only BUMPED refuses them
    for label in ("bumps", "own"):
        keys, p = _plan(w, q, label)
        assert keys[0] == (0, P, R.RPW_BUMPED)
        keys, _ = _plan(w, q, label, mask=R.RPW_BUMPED)
        assert keys[0] == (None, T, R.RPW_BUMPED)
    _, p = _plan(w, q, "own")
    assert (p["waves"][0]["own_lost"], p["waves"][0]["bumped"]) == (2, 1)
    _, p = _plan(w, q, "bumps")
    assert (p["waves"][0]["own_lost"], p["waves"][0]["bumped"]) == (0, 3)
    # no extra row goes to wave 0; NOT_EXCLUSIVE, NOT_FORECAST and NOT_MODELLED entries open nothing; UNFINISHED is
    # solved with the peak it replayed
    keys, p = _plan(w, q, "flags")
    assert keys[0] == (0, P, 0) and [k[1] for k in keys[1:5]] == [NS] * 4
    assert keys[5] == (None, T, R.RPW_STRANDED)
    uf = p["alone_rows"][5]
    assert uf["fc_flags"] & R.LWSF_UNFINISHED and uf["flags"] & R.RPL_SOLVED and uf["surge"] == 3
    keys, p = _plan(w, q, "flags", mask=R.RPW_BUMPED)
    assert keys[5] == (0, P, R.RPW_STRANDED) and p["waves"][0]["n_keys"] == 3


def test_the_tie_pins_query_order():
    """Argument (1): the extra rows of P and Q tie on priority, so their order in the namespace decides who takes
    Q's favourite domain.  In query order both place in one wave; reversed, P strands and opens wave 1."""
    w, rows, ns, recs = tie_world()
    a = rollout_place_waves_ref(w, rows, ns, recs)
    assert a["keys"]["wave"].tolist() == [0, 0] and a["waves"]["stranded"].tolist() == [0]
    b = rollout_place_waves_ref(w, rows[::-1].copy(), ns, recs[::-1].copy())
    assert b["keys"]["wave"].tolist() == [0, 1]


@pytest.mark.parametrize("variant", ["alone_only", "drop_earlier", "reverse_ns"])
def test_wrong_statements_give_wrong_plans(edge, variant):
    w, _, q = edge
    cases = [q["pair_one_ns"], q["cap"]] if variant != "reverse_ns" else [tie_world()[1:]]
    wt = w if variant != "reverse_ns" else tie_world()[0]
    wrong = 0
    for rows, ns, recs in cases:
        a = rollout_place_waves_ref(wt, rows, ns, recs, max_waves=2)
        b = rollout_place_waves_ref(wt, rows, ns, recs, max_waves=2, variant=variant)
        wrong += 0 if same_plan(a, b) else 1
    assert wrong > 0


def test_renumbering_per_namespace_gives_the_same_plans(edge):
    w, _, q = edge
    tw, trows, tns, trecs = tie_world()
    fw = fuzz_world(2)
    frows, fns = fuzz_query(fw, 2)
    for wt, (rows, ns, recs) in [(w, v) for v in q.values()] + [(tw, (trows, tns, trecs)), (fw, (frows, fns, None))]:
        for mask in ALL_MASKS:
            a = rollout_place_waves_ref(wt, rows, ns, recs, constraints=mask)
            b = rollout_place_waves_ref(wt, rows, ns, recs, constraints=mask, variant="by_ns")
            assert same_plan(a, b)


def test_records_match_header():
    h = open(os.path.join(ROOT, "include", "lwse.h")).read()
    for name, dt in (("lwse_rollout_wave_key", R.ROLLOUT_WAVE_KEY), ("lwse_rollout_wave", R.ROLLOUT_WAVE)):
        s = h[h.index(f"typedef struct {name} {{"):]
        s = s[: s.index(f"}} {name};")]
        fields = re.findall(r"^\s+u?int32_t (\w+)(?:\[\d+\])?;", s, re.M)
        assert tuple(fields) == dt.names
    for name, bit in re.findall(r"#define LWSE_RPW_(\w+) \(1u << (\d+)\)", h):
        assert getattr(R, "RPW_" + name) == 1 << int(bit)
    for name, v in re.findall(r"#define LWSE_ROLLW_(\w+) (\d+)u", h):
        assert getattr(R, "ROLLW_" + name) == int(v)
    s = h[h.index("typedef struct lwse_rollout_place_waves_query {"):]
    s = s[: s.index("} lwse_rollout_place_waves_query;")]
    names = re.findall(r"^\s+(?:const )?\w+\*? ?\*?(\w+);", s, re.M)
    assert tuple(names) == tuple(f[0] for f in R.RolloutPlaceWavesQuery._fields_)


def test_argument_checks():
    from lws_b200.engine import rollout_waves_args

    rows = np.array([1, 2, 3], np.uint32)
    ns = np.zeros(3, np.uint32)
    assert rollout_waves_args(rows, ns, None, 64, R.RPW_STRANDED)[0].tolist() == [1, 2, 3]
    for bad in (dict(rows=np.array([1, 2, 1], np.uint32)), dict(ns=np.zeros(2, np.uint32)), dict(max_waves=0),
                dict(max_waves=65), dict(constraints=0), dict(constraints=4), dict(recs=np.zeros(3, np.uint32))):
        kw = dict(rows=rows, ns=ns, recs=None, max_waves=64, constraints=R.RPW_STRANDED)
        kw.update(bad)
        with pytest.raises(ValueError):
            rollout_waves_args(**kw)


def test_informer_report():
    from informer_world import make_world

    from lws_b200 import informer

    items, cluster = make_world(3, n_lws=14, n_nodes=28)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    rows, ns = enc.rollout_place_query()
    keys = sorted(k for k, sl in enc.slots.items() if int(enc.lws["flags"][sl.lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY)
    n = len(rows)
    assert n >= 3
    kr = np.zeros(n, R.ROLLOUT_WAVE_KEY)
    kr["wave"] = R.NONE
    kr["status"] = R.ROLLW_PLANNED
    kr["wave"][0], kr["wave"][1] = 1, 0
    kr["status"][2:] = R.ROLLW_TRIGGERS_ALONE
    kr["alone"][2:] = R.RPW_STRANDED
    kr["wave"][2:] = R.NONE
    waves = np.zeros(2, R.ROLLOUT_WAVE)
    rep = enc.rollout_place_waves_report({"keys": kr, "waves": waves, "lws_rows": rows, "ns": ns})
    assert rep["waves"] == [[keys[1]], [keys[0]]]
    assert [(u["namespace"], u["name"]) for u in rep["unplanned"]] == keys[2:]
    assert all(u["status"] == "triggers_alone" and u["alone"] == ["stranded"] for u in rep["unplanned"])
