"""Drain placement waves on the device (lwse_resident_drain_place_waves): byte for byte against the locality
reference (tests/drain_place_waves_ref.py) on the drain placement's worlds, both scopes, caps and constraint masks;
the LWS-floor-only plan against lwse_resident_drain_waves; the alone columns against both per-key forms; the
errors."""
import ctypes as C

import numpy as np
import pytest

from drain_place_waves_ref import plan
from lws_b200 import records as R
from test_drain_place_cost import WORLDS

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6
MASKS = {"floor": R.DPW_LWS_FLOOR, "stranded": R.DPW_STRANDED, "bumped": R.DPW_BUMPED,
         "default": R.DPW_LWS_FLOOR | R.DPW_STRANDED, "all": R.DPW_ALL}


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def load(engine, world):
    lws, groups, pst, pid, nodes, nd, _, reqs, n_ns = world
    engine.upload_nodes(nodes, nd)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, n_ns)
    engine.resident_tick(engine.make_tick((), R.TICK_PLACE))


def call(engine, by_domain, ids, cap, mask):
    kw = {"domains": ids} if by_domain else {"nodes": ids}
    return engine.resident_drain_place_waves(max_waves=cap, constraints=mask, **kw)


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", ["built", "big_namespaces", "seed3", "seed11"])
def test_matches_the_reference(engine, name, by_domain, mask):
    world = WORLDS[name]()
    load(engine, world)
    occ = engine.resident_occupancy()
    world = world[:6] + (occ,) + world[7:]
    nodes, nd = world[4], world[5]
    ids = np.arange(nd if by_domain else len(nodes))
    rng = np.random.default_rng(7)
    for order in (ids, ids[::-1].copy(), rng.permutation(ids)):
        for cap in (1, 2, 64):
            got = call(engine, by_domain, order, cap, MASKS[mask])
            keys, waves, tot = plan(world, order, by_domain, cap, MASKS[mask], base_place=engine.resident_place_outputs())
            assert {k: got[k] for k in tot} == tot, (name, mask, cap)
            assert got["keys"].tobytes() == keys.tobytes(), (name, mask, cap, got["keys"], keys)
            assert got["waves"].tobytes() == waves.tobytes(), (name, mask, cap, got["waves"], waves)


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", ["built", "seed3"])
def test_floor_alone_is_drain_waves_and_alone_columns(engine, name, by_domain):
    world = WORLDS[name]()
    load(engine, world)
    nodes, nd = world[4], world[5]
    ids = np.arange(nd if by_domain else len(nodes))
    got = call(engine, by_domain, ids, 64, R.DPW_LWS_FLOOR)
    kw = {"domains": ids} if by_domain else {"nodes": ids}
    want = engine.resident_drain_waves(**kw)
    for f in ("id", "wave", "status", "groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(got["keys"][f], want["keys"][f]), f
    for f in R.DRAIN_WAVE.names:
        if f != "reserved":
            assert np.array_equal(got["waves"][f], want["waves"][f]), f
    scope = "domains" if by_domain else "nodes"
    pc = engine.resident_drain_place_cost(scope)[ids]
    bc = engine.resident_drain_budget_cost(scope)[ids]
    for f in ("unpinned", "stranded", "bumped"):
        assert np.array_equal(got["keys"][f], pc[f]), f
    for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(got["keys"][f], bc[f]), f


def test_errors(engine):
    from lws_b200.engine import lib

    world = WORLDS["built"]()
    load(engine, world)
    n = len(world[4])
    keys = R.aligned_empty(n, R.DRAIN_PLACE_WAVE_KEY)
    waves = R.aligned_empty(64, R.DRAIN_PLACE_WAVE)
    ids = np.arange(n, dtype=np.uint32)

    def q(**kw):
        x = R.DrainPlaceWavesQuery()
        x.ids, x.n_ids, x.scope, x.max_waves, x.constraints = R.ptr(ids), n, R.DRAIN_NODES, 64, R.DPW_STRANDED
        x.keys, x.waves = R.ptr(keys), R.ptr(waves)
        for k, v in kw.items():
            setattr(x, k, v)
        return lib().lwse_resident_drain_place_waves(engine._h, C.byref(x))

    assert q() == 0
    for bad in ({"constraints": 0}, {"constraints": 8}, {"max_waves": 0}, {"max_waves": 65}, {"reserved": 1},
                {"reserved1": 1}, {"waves": None}, {"keys": None}, {"ids": None}, {"scope": 7}):
        assert q(**bad) == ERR_INVALID_ARG, bad
    out_of_range = np.array([n], dtype=np.uint32)
    assert q(ids=R.ptr(out_of_range), n_ids=1) == ERR_INVALID_ARG
    dup = np.zeros(2, dtype=np.uint32)
    x = R.DrainPlaceWavesQuery()
    x.ids, x.n_ids, x.scope, x.max_waves, x.constraints = R.ptr(dup), 2, R.DRAIN_NODES, 64, R.DPW_STRANDED
    x.keys, x.waves = R.ptr(keys), R.ptr(waves)
    assert lib().lwse_resident_drain_place_waves(engine._h, C.byref(x)) == ERR_INVALID_ARG


@pytest.fixture(scope="module")
def c3():
    from lws_b200 import synth

    return synth.make("C3", 1.0, seed=synth.SEED)


class _T:
    def __init__(self, world):
        self.groups, self.nodes = world[1], world[4]


def check_waves(engine, t, reqs, got, by_domain, mask, ids):
    """Every wave against the engine's own set forms; the first-fit property against each earlier wave's prefix."""
    from test_gpu_drain_place_cost import composition

    d = t.nodes["domain_id"].astype(np.int64)
    nodes_of = (lambda ks: np.concatenate([np.flatnonzero(d == k) for k in ks])) if by_domain else (
        lambda ks: np.asarray(ks, dtype=np.int64))
    k = got["keys"]
    for w in range(got["n_waves"]):
        W = k["id"][k["wave"] == w].astype(np.int64)
        row = composition(engine, t, reqs, nodes_of(W))
        wr = got["waves"][w]
        assert row["stranded"] == wr["stranded"] and row["bumped"] == wr["bumped"], (w, row, wr)
        for f in ("unpinned", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict"):
            assert row[f] == wr[f], (w, f)
        if mask & R.DPW_STRANDED:
            assert wr["stranded"] == 0
        if mask & R.DPW_BUMPED:
            assert wr["bumped"] == 0
        br = engine.resident_drain_budget(nodes=nodes_of(W))["n_breached"]
        assert br == wr["lws_breached"] and (br == 0 or not mask & R.DPW_LWS_FLOOR)
    # first fit: a key planned at w fails against every earlier wave as it stood at that key
    for i in range(len(k)):
        if k["status"][i] != R.DRAINW_PLANNED:
            continue
        for v in range(int(k["wave"][i])):
            prefix = [int(x) for x in k["id"][:i][k["wave"][:i] == v]]
            if not prefix:
                continue
            S = nodes_of(prefix + [int(k["id"][i])])
            row = composition(engine, t, reqs, S)
            br = engine.resident_drain_budget(nodes=S)["n_breached"]
            assert ((mask & R.DPW_LWS_FLOOR and br) or (mask & R.DPW_STRANDED and row["stranded"])
                    or (mask & R.DPW_BUMPED and row["bumped"])), (i, v)


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("name", ["sum", "strand", "cap"])
def test_edge_worlds_match_the_reference_and_the_set_forms(engine, name, mask):
    from drain_place_waves_ref import EDGE_WORLDS

    world, ids, _ = EDGE_WORLDS[name]()
    by_domain = name == "strand"
    load(engine, world)
    occ = engine.resident_occupancy()
    world = world[:6] + (occ,) + world[7:]
    ids = np.asarray(ids)
    for order in (ids, ids[::-1].copy()):
        for cap in (1, 2, 64):
            got = call(engine, by_domain, order, cap, MASKS[mask])
            keys, waves, tot = plan(world, order, by_domain, cap, MASKS[mask], base_place=engine.resident_place_outputs())
            assert {k: got[k] for k in tot} == tot, (name, mask, cap)
            assert got["keys"].tobytes() == keys.tobytes(), (name, mask, cap, got["keys"], keys)
            assert got["waves"].tobytes() == waves.tobytes(), (name, mask, cap, got["waves"], waves)
    got = call(engine, by_domain, ids, 64, MASKS[mask])
    check_waves(engine, _T(world), world[7], got, by_domain, MASKS[mask], ids)


def test_spare_domains_default_equals_floor(engine):
    from drain_place_waves_ref import EDGE_WORLDS

    world, ids, _ = EDGE_WORLDS["cap"]()  # nothing a drain unpins: every request keeps its domain
    load(engine, world)
    a = call(engine, False, np.asarray(ids), 64, R.DPW_LWS_FLOOR | R.DPW_STRANDED)
    b = call(engine, False, np.asarray(ids), 64, R.DPW_LWS_FLOOR)
    assert a["keys"].tobytes() == b["keys"].tobytes() and a["waves"].tobytes() == b["waves"].tobytes()


@pytest.mark.parametrize("scope", ["domains", "nodes"])
def test_c3_waves_hold_against_the_set_forms(engine, c3, scope):
    t = c3
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    cost = engine.resident_drain_budget_cost(scope)
    ids = np.arange(len(cost))
    ids = ids[np.lexsort((ids, cost["groups_restarted"], -cost["min_margin"].astype(np.int64)))]
    if scope == "nodes":
        ids = ids[:2000]
    mask = R.DPW_LWS_FLOOR | R.DPW_STRANDED
    got = call(engine, scope == "domains", ids, 64, mask)
    assert got["n_planned"] + got["n_breaches_alone"] + got["n_no_wave"] == len(ids)
    k = got["keys"]
    pc = engine.resident_drain_place_cost(scope)[k["id"]]
    for f in ("unpinned", "stranded", "bumped"):
        assert np.array_equal(k[f], pc[f]), f
    assert np.array_equal(k["status"] == R.DRAINW_BREACHES_ALONE, (k["alone"] & mask) != 0)
    from test_gpu_drain_place_cost import composition

    d = t.nodes["domain_id"].astype(np.int64)
    for w in range(got["n_waves"]):
        W = k["id"][k["wave"] == w].astype(np.int64)
        S = np.concatenate([np.flatnonzero(d == x) for x in W]) if scope == "domains" else W
        row = composition(engine, t, reqs, S)
        assert row["stranded"] == 0 == got["waves"][w]["stranded"]
        for f in ("unpinned", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed"):
            assert row[f] == got["waves"][w][f], (w, f)
        assert engine.resident_drain_budget(nodes=S)["n_breached"] == 0


def test_isolation_from_a_tick_in_flight(engine, c3):
    t = c3
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    ids = np.arange(64)
    want = call(engine, True, ids, 8, R.DPW_ALL)
    rows = np.asarray([3, 7, 11], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = reqs[rows]
    vals["size"] += 1
    seg = (R.TABLE_PLACE_REQS, rows, vals)
    engine.resident_tick_submit(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    engine.resident_tick_wait()
    ref_out = engine.resident_place_outputs().copy()
    vals["size"] -= 1
    engine.resident_tick(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    vals["size"] += 1
    engine.resident_tick_submit(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    call(engine, True, ids, 8, R.DPW_ALL)
    engine.resident_tick_wait()
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    vals["size"] -= 1
    engine.resident_tick(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    again = call(engine, True, ids, 8, R.DPW_ALL)
    assert again["keys"].tobytes() == want["keys"].tobytes() and again["waves"].tobytes() == want["waves"].tobytes()


def test_not_ready_and_unsupported(c3):
    from lws_b200.engine import Engine, LwseError

    t = c3
    e = Engine(0)
    try:
        e.upload_nodes(t.nodes, t.n_domains)
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        e.resident_tick(e.make_tick((), t.flags))
        with pytest.raises(LwseError) as ei:  # no placement round yet
            e.resident_drain_place_waves(nodes=[0, 1])
        assert ei.value.status == ERR_NOT_READY
        reqs = t.place_requests()
        e.resident_place_load(reqs, t.n_namespaces)
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        e.resident_drain_place_waves(nodes=[0, 1])
        e.upload_nodes(t.nodes, 5457)  # the domains do not fit one CTA: the namespace form is not offered
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        with pytest.raises(LwseError) as ei:
            e.resident_drain_place_waves(domains=[0, 1])
        assert ei.value.status == -7
    finally:
        e.close()
