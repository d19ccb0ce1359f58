"""DS drain waves on the device (lwse_resident_ds_drain_waves): byte for byte against the fast reference
(tests/ds_drain_waves_ref.py) on the seeded worlds with slack and at the size of the DS drain's big world, for both
scopes and every constraint mask; every wave against the engine's own set forms and the alone columns against its
per-key forms; the first-fit property; the LWS-floor-only plan against lwse_resident_drain_waves; isolation from
ticks; the error returns."""
import ctypes as C
import functools

import numpy as np
import pytest

from drain_budget_ref import min_margin_of
from ds_drain_ref import overlap_worlds
from ds_drain_waves_ref import CONSTRAINTS, DEFAULT, ds_cost_per_ds, ds_waves_edges_world, orders, plan_fast, slack_world
from lws_b200 import engine as E
from lws_b200 import records as R

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6
WORLDS = {"mixed": dict(n_ds=30, n_nodes=96, seed=3), "pct100": dict(n_ds=30, n_nodes=96, seed=5, mu=(100, True)),
          "mu1": dict(n_ds=20, n_nodes=128, seed=7, mu=(1, False)), "mu2": dict(n_ds=24, n_nodes=96, seed=9, mu=(2, False)),
          "pct50": dict(n_ds=24, n_nodes=96, seed=13, mu=(50, True)),
          "big": dict(n_ds=3000, n_nodes=512, seed=7, mu=(100, True))}


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def world(name):
    return slack_world(**WORLDS[name])


def load(engine, w, link=True):
    engine.upload_nodes(w.nodes, w.n_domains)
    engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    engine.resident_tick(engine.make_tick((), w.flags))
    engine.ds_resident_load(w.ds, w.roles, w.revroles)
    return engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)] if link else [])


def by_cost(engine, scope):
    cost = engine.resident_drain_budget_cost(scope)
    return orders(np.arange(len(cost)), cost)


def check_against_engine(engine, got, scope, ids, constraints):
    """Every wave equals the engine's set forms over its ids, with the constrained counts 0; the alone columns equal
    the engine's per-key forms; BREACHES_ALONE iff alone & constraints."""
    bcost, dcost = engine.resident_drain_budget_cost(scope), engine.resident_ds_drain_cost(scope)
    keys = got["keys"]
    for f in ("groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
        assert np.array_equal(keys[f], bcost[f][ids]), f
    for f in ("ds_touched", "ds_service_lost", "ds_old_service_lost", "ds_stalled"):
        assert np.array_equal(keys[f], dcost[f][ids]), f
    assert np.array_equal(keys["status"] == R.DRAINW_BREACHES_ALONE, (keys["alone"] & constraints) != 0)
    for v, row in enumerate(got["waves"]):
        ws = keys["id"][keys["wave"] == v]
        b = engine.resident_drain_budget(**{scope: ws})
        d = engine.resident_ds_drain(**{scope: ws})
        assert row["n_keys"] == len(ws)
        for f, t in (("lws_touched", "n_touched"), ("lws_breached", "n_breached"), ("lws_loses_available", "n_loses_available"),
                     ("n_pods_evicted", "n_pods_evicted"), ("n_leaders_evicted", "n_leaders_evicted"),
                     ("n_groups_restarted", "n_groups_restarted"), ("n_ready_restarted", "n_ready_restarted"),
                     ("n_pods_recreated", "n_pods_recreated")):
            assert row[f] == b[t], (v, f)
        assert int(row["min_margin"]) == min_margin_of(b["rows"]), v
        for f, t in (("ds_touched", "n_touched"), ("ds_service_lost", "n_service_lost"),
                     ("ds_old_service_lost", "n_old_service_lost"), ("ds_stalled", "n_stalled"),
                     ("rows_touched", "rows_touched"), ("rows_zeroed", "rows_zeroed")):
            assert row[f] == d[t], (v, f)
        for bit, f in ((R.DSW_LWS_FLOOR, "lws_breached"), (R.DSW_DS_SERVICE, "ds_service_lost"),
                       (R.DSW_DS_OLD_SERVICE, "ds_old_service_lost"), (R.DSW_DS_STALL, "ds_stalled")):
            if constraints & bit:
                assert row[f] == 0, (v, f)


@pytest.mark.parametrize("name", ["mixed", "pct100", "mu1", "mu2", "pct50", "big"])
def test_equals_the_reference(engine, name):
    w = world(name)
    load(engine, w)
    res = engine.resident_outputs()
    assert res[0].tobytes() == w.base[0].tobytes() and res[1].tobytes() == w.base[1].tobytes()
    for scope, by_domain in (("nodes", False), ("domains", True)):
        ords = by_cost(engine, scope)
        for oname, ids in ords.items():
            if name == "big" and oname != "by_cost":
                continue
            for c in CONSTRAINTS:
                for mw in ((1, 2, 64) if name != "big" and oname == "by_cost" else (64,)):
                    got = engine.resident_ds_drain_waves(**{scope: ids}, max_waves=mw, constraints=c)
                    keys, waves, tot = plan_fast(w, ids, by_domain, mw, c)
                    assert got["keys"].tobytes() == keys.tobytes(), (scope, oname, c, mw)
                    assert got["waves"].tobytes() == waves.tobytes(), (scope, oname, c, mw)
                    assert {k: got[k] for k in R.DS_DRAIN_WAVES_TOTALS} == tot, (scope, oname, c, mw)
                    if mw == 64 and oname == "by_cost" and (name != "big" or c in (DEFAULT, R.DSW_ALL)):
                        check_against_engine(engine, got, scope, ids, c)


def test_lws_floor_only_equals_drain_waves(engine):
    for name in ("mixed", "pct100", "big"):
        w = world(name)
        load(engine, w)
        for scope in ("nodes", "domains"):
            ids = by_cost(engine, scope)["random"]
            for mw in (2, 64):
                got = engine.resident_ds_drain_waves(**{scope: ids}, max_waves=mw, constraints=R.DSW_LWS_FLOOR)
                ref = engine.resident_drain_waves(**{scope: ids}, max_waves=mw)
                assert {k: got[k] for k in R.DS_DRAIN_WAVES_TOTALS} == {k: ref[k] for k in R.DRAIN_WAVES_TOTALS}
                for f in ("id", "wave", "status", "groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
                    assert np.array_equal(got["keys"][f], ref["keys"][f]), (name, scope, f)
                for f in R.DRAIN_WAVE.names:
                    if f != "reserved":
                        assert np.array_equal(got["waves"][f], ref["waves"][f]), (name, scope, f)


def test_first_fit_property(engine):
    """Each planned key triggers a constrained verdict in every earlier wave as it stood when the key was placed
    (the engine's set forms), and fits the wave it was given."""
    def trig(scope, ids):
        b = engine.resident_drain_budget(**{scope: ids})
        d = engine.resident_ds_drain(**{scope: ids})
        return ((R.DSW_LWS_FLOOR if b["n_breached"] else 0) | (R.DSW_DS_SERVICE if d["n_service_lost"] else 0)
                | (R.DSW_DS_OLD_SERVICE if d["n_old_service_lost"] else 0) | (R.DSW_DS_STALL if d["n_stalled"] else 0))

    checked = 0
    for name, mask in (("mixed", R.DSW_DS_SERVICE), ("mu1", R.DSW_DS_SERVICE)):
        load(engine, world(name))
        for scope in ("nodes", "domains"):
            ids = by_cost(engine, scope)["given"]
            got = engine.resident_ds_drain_waves(**{scope: ids}, constraints=mask)
            waves = [[] for _ in got["waves"]]
            for k in got["keys"]:
                if k["status"] != R.DRAINW_PLANNED:
                    continue
                v = int(k["wave"])
                for u in range(v):
                    assert trig(scope, waves[u] + [int(k["id"])]) & mask, (name, scope, int(k["id"]), u)
                    checked += 1
                assert not trig(scope, waves[v] + [int(k["id"])]) & mask
                waves[v].append(int(k["id"]))
    assert checked > 0


def test_no_links_binds_no_ds_constraint(engine):
    """Before any link patch every row falls back: a DS-only plan puts every key in one wave."""
    w = world("pct100")
    load(engine, w, link=False)
    got = engine.resident_ds_drain_waves(nodes=np.arange(len(w.nodes)), constraints=R.DSW_ALL & ~R.DSW_LWS_FLOOR)
    assert got["n_waves"] == 1 and got["n_planned"] == len(w.nodes)
    assert not got["waves"]["ds_touched"].any() and not got["keys"]["alone"].any()


def test_isolation(engine):
    """Plan calls between the submit and wait of LWS ticks in flight, and before each DS tick: every LWS tick's
    change lists, the resident LWS rows, every DS tick's changed rows and full outputs and the DS tick info equal a
    run without them, and every resident table and the link table read back equal too."""
    from test_gpu_ds_drain import resident_tables
    from test_gpu_node_events import Arena

    w = world("big")
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(6):
        rows = np.sort(rng.choice(len(w.groups), size=200, replace=False)).astype(np.uint32)
        v = w.groups[rows].copy()
        v["flags"] ^= np.uint32(R.GRP_POD_READY)
        sets.append([(R.TABLE_GROUPS, rows, v)])

    def snap(r):
        return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()}

    def run(with_plan):
        first = snap(load(engine, w))
        first["info"] = engine.ds_resident_tick_info()
        arena = Arena(engine)
        lws_out, ds_out, answers = [], [first], []
        for k, segs in enumerate(sets):
            engine.resident_tick_submit(engine.make_tick(arena.put(segs, k & 1), w.flags))
            if with_plan:
                answers.append(engine.resident_ds_drain_waves(domains=np.arange(w.n_domains), constraints=R.DSW_ALL))
                engine.resident_ds_drain_waves(nodes=rng.permutation(len(w.nodes))[:200], max_waves=3)
            lws_out.append(snap(engine.resident_tick_wait()))
            if with_plan:
                engine.resident_ds_drain_waves(nodes=np.arange(len(w.nodes)))
            ds_out.append(snap(engine.ds_resident_tick([])))
            ds_out[-1]["info"] = engine.ds_resident_tick_info()
        return lws_out, ds_out, [x.copy() for x in engine.resident_outputs()], answers

    a = run(True)
    tables = resident_tables(engine, w)
    b = run(False)
    assert resident_tables(engine, w) == tables
    assert tables[4:] == [w.ds.tobytes(), w.roles.tobytes(), w.revroles.tobytes(), w.links.tobytes()]
    for k, (x, y) in enumerate(zip(a[0], b[0])):
        for key in ("lws_rows", "group_rows"):
            ox, oy = np.argsort(x[key], kind="stable"), np.argsort(y[key], kind="stable")
            assert np.array_equal(x[key][ox], y[key][oy]), (k, key)
            assert x[key.replace("rows", "out")][ox].tobytes() == y[key.replace("rows", "out")][oy].tobytes(), (k, key)
    for k, (x, y) in enumerate(zip(a[1], b[1])):
        assert np.array_equal(np.sort(x["rows"]), np.sort(y["rows"])), k
        for key in ("ds_out", "role_out", "revrole_out"):
            assert x[key].tobytes() == y[key].tobytes(), (k, key)
        ix = dict(x["info"], lws_ticks=x["info"]["lws_ticks"] - a[1][0]["info"]["lws_ticks"])
        iy = dict(y["info"], lws_ticks=y["info"]["lws_ticks"] - b[1][0]["info"]["lws_ticks"])
        assert ix == iy, k
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a[2], b[2]))
    assert all(ans["n_planned"] + ans["n_breaches_alone"] == w.n_domains for ans in a[3])


@functools.lru_cache(maxsize=None)
def edges():
    return ds_waves_edges_world()


def test_edges_world(engine):
    """The edges world byte for byte against the fast reference for both scopes, every mask and caps 2 and 64;
    its per-key rows against both per-key forms; and the evaluated-only binding refuted on the device's plan."""
    w, ids, notes = edges()
    load(engine, w)
    res = engine.resident_outputs()
    assert res[0].tobytes() == w.base[0].tobytes() and res[1].tobytes() == w.base[1].tobytes()
    for scope, by_domain in (("nodes", False), ("domains", True)):
        for c in CONSTRAINTS:
            for mw in (2, 64):
                got = engine.resident_ds_drain_waves(**{scope: ids}, max_waves=mw, constraints=c)
                keys, waves, tot = plan_fast(w, ids, by_domain, mw, c)
                assert got["keys"].tobytes() == keys.tobytes(), (scope, c, mw)
                assert got["waves"].tobytes() == waves.tobytes(), (scope, c, mw)
                assert {k: got[k] for k in R.DS_DRAIN_WAVES_TOTALS} == tot, (scope, c, mw)
                if mw == 64:
                    check_against_engine(engine, got, scope, np.asarray(ids), c)
    got = engine.resident_ds_drain_waves(nodes=ids, constraints=R.DSW_DS_SERVICE)
    k = got["keys"][list(ids).index(notes["unevaluated"][0])]
    assert k["status"] == R.DRAINW_BREACHES_ALONE and k["alone"] == R.DSW_DS_SERVICE
    wrong = plan_fast(w, ids, False, 64, R.DSW_DS_SERVICE, linked_bind=False)
    assert got["keys"].tobytes() != wrong[0].tobytes()
    st = [(int(x["status"]), int(x["wave"])) for x in
          engine.resident_ds_drain_waves(nodes=ids, constraints=R.DSW_ALL)["keys"][-65:]]
    assert st[:64] == [(R.DRAINW_PLANNED, v) for v in range(64)] and st[64] == (R.DRAINW_NO_WAVE, R.NONE)


def test_edges_overlapping_ranges(engine):
    """Two more DS over the range of the ``ready2`` DS: the device walks every DS over its own range, as the per-DS
    reference does, and plans as with disjoint copies of the rows."""
    w, ids, notes = edges()
    shared, copied = overlap_worlds(w, 2)
    answers = {}
    for name, x in (("shared", shared), ("copied", copied)):
        load(engine, x)
        assert engine.resident_ds_drain_cost("nodes").tobytes() == ds_cost_per_ds(x).tobytes(), name
        for c in (R.DSW_LWS_FLOOR, R.DSW_DS_SERVICE, R.DSW_ALL):
            got = engine.resident_ds_drain_waves(nodes=ids, constraints=c)
            keys, waves, _ = plan_fast(x, ids, False, 64, c)
            assert got["keys"].tobytes() == keys.tobytes() and got["waves"].tobytes() == waves.tobytes(), (name, c)
            answers[name, c] = (got["keys"].tobytes(), got["waves"].tobytes())
    for c in (R.DSW_LWS_FLOOR, R.DSW_DS_SERVICE, R.DSW_ALL):
        assert answers["shared", c] == answers["copied", c], c


def raw(e, ids=None, n_ids=0, scope=R.DRAIN_NODES, max_waves=64, constraints=DEFAULT, reserved=0, reserved1=0,
        keys=True, waves=True):
    kbuf = R.aligned_empty(max(n_ids, 1), R.DS_DRAIN_WAVE_KEY)
    wbuf = R.aligned_empty(64, R.DS_DRAIN_WAVE)
    kbuf.view(np.uint8)[:] = 0xAB
    wbuf.view(np.uint8)[:] = 0xAB
    q = R.DsDrainWavesQuery()
    q.ids, q.n_ids, q.scope, q.max_waves, q.constraints = ids, n_ids, scope, max_waves, constraints
    q.reserved, q.reserved1 = reserved, reserved1
    q.keys = R.ptr(kbuf) if keys else None
    q.waves = R.ptr(wbuf) if waves else None
    q.n_waves = q.n_planned = q.n_breaches_alone = q.n_no_wave = 0xABABABAB
    rc = E.lib().lwse_resident_ds_drain_waves(e._h, C.byref(q))
    untouched = (kbuf.view(np.uint8) == 0xAB).all() and (wbuf.view(np.uint8) == 0xAB).all() and \
        (q.n_waves, q.n_planned, q.n_breaches_alone, q.n_no_wave) == (0xABABABAB,) * 4
    return rc, untouched


def test_errors():
    w = world("mixed")
    e = E.Engine(0)
    try:
        one = np.array([1], np.uint32)
        assert raw(e, R.ptr(one), 1) == (ERR_NOT_READY, True)  # nothing loaded
        e.upload_nodes(w.nodes, w.n_domains)
        e.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        e.resident_tick(e.make_tick((), w.flags))
        assert raw(e, R.ptr(one), 1) == (ERR_NOT_READY, True)  # no DS tables
        e.ds_resident_load(w.ds, w.roles, w.revroles)
        e.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
        assert raw(e, R.ptr(one), 1)[0] == 0 and raw(e, R.ptr(one), 1, R.DRAIN_DOMAINS)[0] == 0
        assert raw(e, None, 0)[0] == 0 and raw(e, None, 0, keys=False)[0] == 0  # m = 0: no key buffer needed
        assert E.lib().lwse_resident_ds_drain_waves(e._h, None) == ERR_INVALID_ARG
        two, past_n = np.array([1, 1], np.uint32), np.array([len(w.nodes)], np.uint32)
        past_d = np.array([w.n_domains], np.uint32)
        for kw in ({"ids": R.ptr(two), "n_ids": 2},
                   {"ids": R.ptr(past_n), "n_ids": 1},
                   {"ids": R.ptr(past_d), "n_ids": 1, "scope": R.DRAIN_DOMAINS},
                   {"ids": R.ptr(one), "n_ids": 1, "scope": 2},
                   {"ids": R.ptr(one), "n_ids": 1, "max_waves": 0},
                   {"ids": R.ptr(one), "n_ids": 1, "max_waves": 65},
                   {"ids": R.ptr(one), "n_ids": 1, "constraints": 0},
                   {"ids": R.ptr(one), "n_ids": 1, "constraints": 16},
                   {"ids": R.ptr(one), "n_ids": 1, "reserved": 1},
                   {"ids": R.ptr(one), "n_ids": 1, "reserved1": 1},
                   {"ids": None, "n_ids": 1},
                   {"ids": R.ptr(one), "n_ids": 1, "keys": False},
                   {"ids": R.ptr(one), "n_ids": 1, "waves": False}):
            assert raw(e, **kw) == (ERR_INVALID_ARG, True), kw
        # LWS rows patched without a sweep: not ready until the next sweep
        e.resident_patch(R.TABLE_LWS, [0], w.lws[:1])
        assert raw(e, R.ptr(one), 1) == (ERR_NOT_READY, True)
        e.resident_tick(e.make_tick((), w.flags))
        assert raw(e, R.ptr(one), 1)[0] == 0
    finally:
        e.close()
