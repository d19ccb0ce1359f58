"""Drain waves on the device (lwse_resident_drain_waves): byte for byte against the fast reference
(tests/drain_waves_ref.py) on the seeded worlds, the edges world, the breach world at 20 000 objects and C3, for
both scopes; every wave against the engine's own set-form drain budget and the alone columns against its per-key
form; the first-fit property against the set form; isolation from ticks in flight; the error returns."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
from drain_budget_ref import budget_world, domain_nodes, min_margin_of
from drain_waves_ref import orders, plan_fast, waves_edges_world, waves_world
from lws_b200 import engine as E
from lws_b200 import synth
from lws_b200 import records as R
from test_gpu_node_events import Arena

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6
NONE = R.NONE


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


def load(engine, t):
    lws, groups, pst, pid, nodes, n_domains, flags = t
    engine.upload_nodes(nodes, n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick((), flags))


@functools.lru_cache(maxsize=None)
def world(name):
    if name == "edges":
        w, _, _ = waves_edges_world()
        return (w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, 0)
    if name == "C3":
        w = synth.make("C3", 1.0, seed=synth.SEED)
    elif name == "breach":
        w = budget_world(n_lws=20_000, n_nodes=2048, seed=17)
    elif name == "small_breach":
        w = budget_world(n_lws=160, n_nodes=48, seed=5)
    else:
        w = waves_world(n_lws=120 if name == "seed5" else 160, n_nodes=96 if name == "seed5" else 64,
                        seed=5 if name == "seed5" else 6)
    return (w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, w.flags)


def ids_of(engine, name, scope):
    if name == "edges":
        return np.asarray(waves_edges_world()[1], dtype=np.int64)
    cost = engine.resident_drain_budget_cost(scope)
    return orders(np.arange(len(cost)), cost)["by_cost"]


def check_against_engine(engine, got, scope, ids):
    """Every wave: the engine's set form over its ids breaches nothing and gives the wave's totals; the alone
    columns equal the engine's per-key form."""
    cost = engine.resident_drain_budget_cost(scope)
    keys = got["keys"]
    for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(keys[f], cost[f][ids]), f
    kw = "nodes" if scope == "nodes" else "domains"
    for w, row in enumerate(got["waves"]):
        ws = keys["id"][keys["wave"] == w]
        s = engine.resident_drain_budget(**{kw: ws})
        assert s["n_breached"] == 0, w
        assert row["n_keys"] == len(ws) and row["lws_touched"] == s["n_touched"]
        assert row["lws_loses_available"] == s["n_loses_available"]
        for f in ("n_pods_evicted", "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted", "n_pods_recreated"):
            assert row[f] == s[f], (w, f)
        assert int(row["min_margin"]) == min_margin_of(s["rows"]), w


@pytest.mark.parametrize("name", ["seed5", "seed6", "edges", "small_breach", "breach", "C3"])
def test_equals_the_reference(engine, name):
    t = world(name)
    load(engine, t)
    lws, groups, pst, pid, nodes, nd, flags = t
    base = engine.resident_outputs()
    assert base[1].tobytes() == oracle.sweep_lws(lws, groups, pst, pid, nodes, flags & R.SWEEP_GANG,
                                                 threads=16)[1].tobytes()
    for scope, by_domain in (("nodes", False), ("domains", True)):
        ids = ids_of(engine, name, scope)
        for mw in ((1, 2, 64) if name in ("seed5", "seed6", "edges") else (64,)):
            got = engine.resident_drain_waves(**{scope: ids}, max_waves=mw)
            keys, waves, tot = plan_fast(lws, base[0], groups, pst, pid, nodes, nd, base[1], ids, by_domain, mw)
            assert got["keys"].tobytes() == keys.tobytes(), (scope, mw)
            assert got["waves"].tobytes() == waves.tobytes(), (scope, mw)
            assert {k: got[k] for k in R.DRAIN_WAVES_TOTALS} == tot, (scope, mw)
            if mw == 64:
                check_against_engine(engine, got, scope, ids)
        if name == "C3":  # every floor is 0: one wave holds every key
            assert got["n_waves"] == 1 and got["n_planned"] == len(ids)


def test_first_fit_property(engine):
    """On a small world: each planned key breaches every earlier wave as it stood when the key was placed (the
    engine's set form), and fits the wave it was given."""
    t = world("seed5")
    load(engine, t)
    for scope in ("nodes", "domains"):
        ids = ids_of(engine, "seed5", scope)
        got = engine.resident_drain_waves(**{scope: ids})
        waves = [[] for _ in got["waves"]]
        checked = 0
        for k in got["keys"]:
            if k["status"] != R.DRAINW_PLANNED:
                continue
            w = int(k["wave"])
            for v in range(w):
                s = engine.resident_drain_budget(**{scope: waves[v] + [int(k["id"])]})
                assert s["n_breached"] > 0, (scope, int(k["id"]), v)
                checked += 1
            if waves[w]:
                assert engine.resident_drain_budget(**{scope: waves[w] + [int(k["id"])]})["n_breached"] == 0
            waves[w].append(int(k["id"]))
        assert checked > 0, scope


def test_isolation_from_ticks_in_flight(engine):
    """Plan calls between the submit and wait of ticks in flight: every tick's change lists, the final rows,
    occupancy, node and tick info equal a run without them."""
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(6):
        rows = np.sort(rng.choice(len(t.pod_state), size=2000, replace=False)).astype(np.uint32)
        sets.append([(R.TABLE_POD_STATE, rows, (t.pod_state[rows] ^ np.uint8(R.POD_ANY_RESTART)).astype(np.uint8))])

    def run(with_plan):
        engine.upload_nodes(t.nodes, t.n_domains)
        engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        engine.resident_place_load(reqs, t.n_namespaces)
        engine.resident_tick(engine.make_tick((), flags))
        arena = Arena(engine)
        out, infos, pending = [], [], 0

        def wait():
            r = engine.resident_tick_wait()
            out.append({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()})

        for k, segs in enumerate(sets):
            if pending == 2:
                wait()
                pending -= 1
            engine.resident_tick_submit(engine.make_tick(arena.put(segs, k & 1), flags))
            pending += 1
            info = (engine.resident_node_info(), engine.resident_tick_info())
            infos.append(info)
            if with_plan:
                assert engine.resident_drain_waves(nodes=[])["n_waves"] == 0
                engine.resident_drain_waves(domains=np.arange(t.n_domains))
                engine.resident_drain_waves(nodes=rng.permutation(len(t.nodes))[:500], max_waves=3)
                assert (engine.resident_node_info(), engine.resident_tick_info()) == info, k
        while pending:
            wait()
            pending -= 1
        return out, infos, engine.resident_place_outputs().copy(), engine.resident_occupancy().copy(), engine.resident_outputs()

    a_out, a_infos, a_rows, a_occ, a_res = run(True)
    b_out, b_infos, b_rows, b_occ, b_res = run(False)
    assert len(a_out) == len(b_out) == len(sets)
    for k, (x, y) in enumerate(zip(a_out, b_out)):
        for key in ("lws_rows", "group_rows", "place_rows"):
            ox, oy = np.argsort(x[key], kind="stable"), np.argsort(y[key], kind="stable")
            assert np.array_equal(x[key][ox], y[key][oy]), (k, key)
            out_key = key.replace("rows", "out")
            assert x[out_key][ox].tobytes() == y[out_key][oy].tobytes(), (k, out_key)
    assert a_infos == b_infos
    assert a_rows.tobytes() == b_rows.tobytes() and np.array_equal(a_occ, b_occ)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a_res, b_res))


def raw(e, ids=None, n_ids=0, scope=R.DRAIN_NODES, max_waves=64, reserved=0, keys=True, waves=True):
    kbuf = R.aligned_empty(max(n_ids, 1), R.DRAIN_WAVE_KEY)
    wbuf = R.aligned_empty(64, R.DRAIN_WAVE)
    kbuf.view(np.uint8)[:] = 0xAB
    wbuf.view(np.uint8)[:] = 0xAB
    q = R.DrainWavesQuery()
    q.ids, q.n_ids, q.scope, q.max_waves, q.reserved = ids, n_ids, scope, max_waves, reserved
    q.keys = R.ptr(kbuf) if keys else None
    q.waves = R.ptr(wbuf) if waves else None
    q.n_waves = q.n_planned = q.n_breaches_alone = q.n_no_wave = 0xABABABAB
    rc = E.lib().lwse_resident_drain_waves(e._h, C.byref(q))
    untouched = (kbuf.view(np.uint8) == 0xAB).all() and (wbuf.view(np.uint8) == 0xAB).all() and \
        (q.n_waves, q.n_planned, q.n_breaches_alone, q.n_no_wave) == (0xABABABAB,) * 4
    return rc, untouched


def test_errors():
    t = world("small_breach")
    lws, groups, pst, pid, nodes, nd, flags = t
    e = E.Engine(0)
    try:
        one = np.array([1], np.uint32)
        rc, clean = raw(e, R.ptr(one), 1)
        assert rc == ERR_NOT_READY and clean  # nothing loaded
        e.resident_load(lws, groups, pst, pid)
        e.resident_tick(e.make_tick((), flags))
        assert raw(e, R.ptr(one), 1) == (ERR_NOT_READY, True)  # no node table
        e.upload_nodes(nodes, nd)
        assert raw(e, R.ptr(one), 1)[0] == 0 and raw(e, R.ptr(one), 1, R.DRAIN_DOMAINS)[0] == 0
        assert raw(e, None, 0)[0] == 0 and raw(e, None, 0, keys=False)[0] == 0  # m = 0: no key buffer needed
        assert E.lib().lwse_resident_drain_waves(e._h, None) == ERR_INVALID_ARG
        two, past_n, past_d = np.array([1, 1], np.uint32), np.array([len(nodes)], np.uint32), np.array([nd], np.uint32)
        for kw in ({"ids": R.ptr(two), "n_ids": 2},                                         # a duplicate
                   {"ids": R.ptr(past_n), "n_ids": 1},            # a node out of range
                   {"ids": R.ptr(past_d), "n_ids": 1, "scope": R.DRAIN_DOMAINS},
                   {"ids": R.ptr(one), "n_ids": 1, "scope": 2},
                   {"ids": R.ptr(one), "n_ids": 1, "max_waves": 0},
                   {"ids": R.ptr(one), "n_ids": 1, "max_waves": 65},
                   {"ids": R.ptr(one), "n_ids": 1, "reserved": 1},
                   {"ids": None, "n_ids": 1},
                   {"ids": R.ptr(one), "n_ids": 1, "keys": False},
                   {"ids": R.ptr(one), "n_ids": 1, "waves": False}):
            assert raw(e, **kw) == (ERR_INVALID_ARG, True), kw
        # LWS or group rows patched without a sweep: not ready until the next sweep
        for table, vals in ((R.TABLE_LWS, lws[:1]), (R.TABLE_GROUPS, groups[:1])):
            e.resident_patch(table, [0], vals)
            assert raw(e, R.ptr(one), 1) == (ERR_NOT_READY, True)
            e.resident_tick(e.make_tick((), flags))
            assert raw(e, R.ptr(one), 1)[0] == 0
    finally:
        e.close()
