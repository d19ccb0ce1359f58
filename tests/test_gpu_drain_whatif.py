"""Drain what-if and drain cost on the device (lwse_resident_drain_*): bit for bit against the spec oracle's sweep
with the drained nodes' pods deleting (tests/drain_ref.py) on small tables and at C3, the same rows and change
lists as a real tick that sets the same bits, every node's cost against the what-if of that node and against
the numpy restatement, isolation from ticks in flight, the error returns, and the step to a placement what-if."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
from drain_ref import COST_OF, TOTALS, drain_cost_ref, drain_tables, drain_whatif_ref, special_tables
from lws_b200 import engine as E
from lws_b200 import informer, synth
from lws_b200 import records as R
from test_gpu_node_events import Arena
from test_place_whatif import whatif_ref

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def c3():
    return synth.make("C3", 1.0, seed=synth.SEED)


def load(engine, lws, groups, pst, pid, nodes, n_domains, flags=0):
    engine.upload_nodes(nodes, n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick((), flags))


def sorted_rows(res):
    o = np.argsort(res["rows"], kind="stable")
    return res["rows"][o], res["before"][o].tobytes(), res["after"][o].tobytes()


def check(got, ref, where):
    assert got["n_changed"] == ref["n_changed"], where
    r, b, a = sorted_rows(got)
    assert np.array_equal(r, ref["rows"]), where
    assert b == ref["before"].tobytes() and a == ref["after"].tobytes(), where
    for k in TOTALS:
        assert got[k] == ref[k], (where, k)


@functools.lru_cache(maxsize=1)
def small_worlds():
    from informer_world import make_world
    from lifecycle_world import LifecycleWorld
    from node_world import NodeWorld

    out = {"special": special_tables()}
    for name, cls, seed in (("node", NodeWorld, 21), ("lifecycle", LifecycleWorld, 31)):
        items, cluster = make_world(seed, n_lws=14, n_nodes=24)
        world = cls(items, cluster, seed + 1)
        enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=1.0, node_spare=4)
        for _ in range(25):
            world.step(enc)
        enc.flush()
        lws, groups, pst, pid, _ = enc.full_tables()
        out[name] = (lws, groups, pst, pid, enc.node_rec)
    return out


@pytest.mark.parametrize("name", ["special", "node", "lifecycle"])
@pytest.mark.parametrize("flags", [0, R.SWEEP_GANG])
def test_small_tables(engine, name, flags):
    lws, groups, pst, pid, nodes = small_worlds()[name]
    n_domains = int(nodes["domain_id"][nodes["domain_id"] != R.NONE].max(initial=0)) + 1
    load(engine, lws, groups, pst, pid, nodes, n_domains, flags)
    base = oracle.sweep_lws(lws, groups, pst, pid, nodes, flags)[:2]
    _, res = engine.resident_outputs()
    assert res.tobytes() == base[1].tobytes()
    cost = engine.resident_drain_cost()
    assert cost.tobytes() == drain_cost_ref(lws, groups, pst, pid, len(nodes), base[1]).tobytes()
    assert np.array_equal(cost["pods"], engine.resident_occupancy())
    for n in range(len(nodes)):
        got = engine.resident_drain_whatif([n])
        check(got, drain_whatif_ref(lws, groups, pst, pid, nodes, [n], flags, base=base), (name, n))
        for k in TOTALS:
            assert int(cost[COST_OF[k]][n]) == got[k], (name, n, k)
    rng = np.random.default_rng(3)
    for d in ([], list(range(len(nodes))), [1, 1, 2], list(rng.choice(len(nodes), 5))):
        check(engine.resident_drain_whatif(d), drain_whatif_ref(lws, groups, pst, pid, nodes, d, flags, base=base), (name, d))


def c3_sets(t):
    rng = np.random.default_rng(9)
    dom = int(rng.integers(0, t.n_domains))
    return {"one": [int(rng.integers(0, len(t.nodes)))], "domain": np.flatnonzero(t.nodes["domain_id"] == dom).tolist(),
            "percent": rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False).tolist()}


def test_c3_against_the_oracle_and_a_tick(engine, c3):
    """At C3: one node, one domain, 1 % of the nodes against the oracle; and a second engine that takes a tick
    whose patches set the same bits lists the same group rows, no LWS row, and holds the what-if's rows."""
    t = c3
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    fl = t.flags & R.SWEEP_GANG
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl, threads=16)[:2]
    other = E.Engine(0)
    try:
        for label, d in c3_sets(t).items():
            got = engine.resident_drain_whatif(d)
            ref = drain_whatif_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, d, fl, base=base)
            check(got, ref, label)
            assert got["n_pods_evicted"] > 0
            load(other, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
            g, pst, _, _ = drain_tables(t.groups, t.pod_state, t.pod_ident, d)
            prow = np.flatnonzero(pst != t.pod_state).astype(np.uint32)
            grow = np.flatnonzero(g["flags"] != t.groups["flags"]).astype(np.uint32)
            res = other.resident_tick(other.make_tick([(R.TABLE_POD_STATE, prow, pst[prow]), (R.TABLE_GROUPS, grow, g[grow])],
                                                      t.flags))
            assert res["n_lws"] == 0, label
            o = np.argsort(res["group_rows"], kind="stable")
            r, _, a = sorted_rows(got)
            assert np.array_equal(res["group_rows"][o], r) and res["group_out"][o].tobytes() == a, label
    finally:
        other.close()


def test_c3_cost(engine, c3):
    """drain_cost at C3: every node against the numpy restatement, 64 sampled nodes against the what-if."""
    t = c3
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    _, base_out = engine.resident_outputs()
    cost = engine.resident_drain_cost()
    ref = drain_cost_ref(t.lws, t.groups, t.pod_state, t.pod_ident, len(t.nodes), base_out)
    assert cost.tobytes() == ref.tobytes()
    assert np.array_equal(cost["pods"], engine.resident_occupancy())
    assert cost["groups_restarted"].sum() > 0
    for n in np.random.default_rng(4).choice(len(t.nodes), size=64, replace=False).tolist():
        got = engine.resident_drain_whatif([n], capacity=0)
        for k in TOTALS:
            assert int(cost[COST_OF[k]][n]) == got[k], (n, k)


def test_isolation_from_ticks_in_flight(engine, c3):
    """What-ifs and cost calls between the submit and wait of two ticks in flight, and between graph-replayed
    ticks: every tick's change lists, the final rows and occupancy equal a run without them; an empty what-if
    reports no change (its baseline is the newest submitted sweep)."""
    t = c3
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(10):
        rows = np.sort(rng.choice(len(t.pod_state), size=2000, replace=False)).astype(np.uint32)
        vals = (t.pod_state[rows] ^ np.uint8(R.POD_ANY_RESTART)).astype(np.uint8)
        sets.append([(R.TABLE_POD_STATE, rows, vals)])
    doms = rng.choice(t.n_domains, size=10, replace=False)

    def run(with_whatif):
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
            if with_whatif:
                assert engine.resident_drain_whatif([])["n_changed"] == 0, k
                engine.resident_drain_whatif(np.flatnonzero(t.nodes["domain_id"] == doms[k]))
                engine.resident_drain_cost()
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
    assert any(ti["graph"] for _, ti in a_infos)
    assert a_rows.tobytes() == b_rows.tobytes() and np.array_equal(a_occ, b_occ)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a_res, b_res))


def raw(e, nodes=None, n_nodes=0, capacity=0, rows=None, before=None, after=None):
    q = R.DrainWhatIf()
    q.nodes, q.n_nodes, q.capacity = nodes, n_nodes, capacity
    q.rows, q.before, q.after = rows, before, after
    return E.lib().lwse_resident_drain_whatif(e._h, C.byref(q))


def test_errors_capacity_and_empty_set(c3):
    lws, groups, pst, pid, nodes = special_tables()
    e = E.Engine(0)
    try:
        n = np.array([1], np.uint32)
        cost = R.aligned_empty(len(nodes), R.DRAIN_COST)
        assert raw(e, R.ptr(n), 1) == ERR_NOT_READY  # nothing loaded
        assert E.lib().lwse_resident_drain_cost(e._h, R.ptr(cost)) == ERR_NOT_READY
        e.resident_load(lws, groups, pst, pid)
        e.resident_tick(e.make_tick(()))
        assert raw(e, R.ptr(n), 1) == ERR_NOT_READY  # no node table
        e.upload_nodes(nodes, 4)
        assert raw(e, R.ptr(n), 1) == 0
        assert E.lib().lwse_resident_drain_whatif(e._h, None) == ERR_INVALID_ARG
        assert E.lib().lwse_resident_drain_cost(e._h, None) == ERR_INVALID_ARG
        assert raw(e, R.ptr(np.array([len(nodes)], np.uint32)), 1) == ERR_INVALID_ARG
        assert raw(e, None, 1) == ERR_INVALID_ARG
        assert raw(e, R.ptr(n), 1, capacity=4) == ERR_INVALID_ARG
        assert raw(e, None, 0) == 0  # an empty D
        # group or pod rows patched without a sweep: not ready until the next sweep
        for table, rows, vals in ((R.TABLE_POD_STATE, [0], pst[:1]), (R.TABLE_GROUPS, [0], groups[:1])):
            e.resident_patch(table, rows, vals)
            assert raw(e, R.ptr(n), 1) == ERR_NOT_READY
            e.resident_tick(e.make_tick(()))
            e.resident_tick(e.make_tick([(table, np.array(rows, np.uint32), vals)], R.TICK_NO_SWEEP))
            assert E.lib().lwse_resident_drain_cost(e._h, R.ptr(cost)) == ERR_NOT_READY
            e.resident_tick(e.make_tick(()))
            assert raw(e, R.ptr(n), 1) == 0
        base = oracle.sweep_lws(lws, groups, pst, pid, nodes)[:2]
        d = list(range(len(nodes)))
        ref = drain_whatif_ref(lws, groups, pst, pid, nodes, d, base=base)
        assert ref["n_changed"] > 3
        small = e.resident_drain_whatif(d, capacity=3)
        assert small["n_changed"] == ref["n_changed"] and len(small["rows"]) == 3
        for k in range(3):
            i = int(np.searchsorted(ref["rows"], small["rows"][k]))
            assert ref["rows"][i] == small["rows"][k]
            assert small["before"][k].tobytes() == ref["before"][i].tobytes()
            assert small["after"][k].tobytes() == ref["after"][i].tobytes()
        empty = e.resident_drain_whatif([])
        assert empty["n_changed"] == 0 and all(empty[k] == 0 for k in TOTALS)
    finally:
        e.close()


def test_drain_place_query(engine):
    """drain_place_query through lwse_resident_place_whatif against the placement spec over the patched rows."""
    from informer_world import make_world

    items, cluster = make_world(7, n_lws=18, n_nodes=40)
    enc = informer.IncrementalEncoder(items, cluster, "zone", spare=1.0, node_spare=8)
    lws, groups, pst, pid, reqs = enc.full_tables()
    engine.upload_nodes(enc.node_rec, enc.n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, enc.n_namespaces)
    engine.resident_tick(engine.make_tick((), R.TICK_PLACE))
    occ = engine.resident_occupancy()
    names = sorted(enc.node_index)[:6]
    res = engine.resident_drain_whatif(enc.whatif_drain(names))
    segs = enc.drain_place_query(res, names)
    assert len(segs[1][1]) > 0
    got = engine.resident_place_whatif(segs)
    ref = whatif_ref(enc.node_rec, occ, enc.n_domains, reqs, segs, n_ns=enc.n_namespaces)
    o = np.argsort(got["rows"], kind="stable")
    assert np.array_equal(got["rows"][o], ref["rows"])
    assert got["after"][o].tobytes() == ref["after"].tobytes()
