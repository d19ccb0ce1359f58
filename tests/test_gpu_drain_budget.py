"""Drain budget on the device (lwse_resident_drain_budget*): byte for byte against the definition
(tests/drain_budget_ref.py) on small tables, at C3 and on a world where floors bind, for both scopes; the NODES
rows against lwse_resident_drain_cost; isolation from ticks in flight; the error returns; a capacity below the
touched count; and an (LWS, key) table that grows well past C3's."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
from drain_budget_ref import budget_world, domain_nodes, drain_budget_cost_ref, drain_budget_ref, min_margin_of
from lws_b200 import engine as E
from lws_b200 import informer, synth
from lws_b200 import records as R
from test_gpu_node_events import Arena

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6
TOTALS = R.DRAIN_BUDGET_TOTALS


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def c3():
    return synth.make("C3", 1.0, seed=synth.SEED)


@pytest.fixture(scope="module")
def breach():
    return budget_world()


def load(engine, lws, groups, pst, pid, nodes, n_domains, flags=0):
    engine.upload_nodes(nodes, n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick((), flags))


def check_set(got, ref, where):
    rows, totals = ref
    for k in TOTALS:
        assert got[k] == totals[k], (where, k)
    o = np.argsort(got["rows"]["lws"], kind="stable")
    assert got["rows"][o].tobytes() == rows.tobytes(), where


def check_cost(engine, lws, groups, pst, pid, nodes, n_domains, base):
    """Both scopes against the reference; NODES rows start with the drain cost rows."""
    out = {}
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_drain_budget_cost(scope)
        ref = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, n_domains, base[1], by_domain)
        assert got.tobytes() == ref.tobytes(), scope
        out[scope] = got
    cost = engine.resident_drain_cost()
    head = out["nodes"].view(np.uint8).reshape(len(cost), 48)[:, :32]
    assert head.tobytes() == cost.tobytes()
    return out


@functools.lru_cache(maxsize=1)
def small_worlds():
    from test_gpu_drain_whatif import small_worlds as sw

    out = {}
    for name, (lws, groups, pst, pid, nodes) in sw().items():
        n_domains = int(nodes["domain_id"][nodes["domain_id"] != R.NONE].max(initial=0)) + 1
        if name == "special":
            nodes = nodes.copy()
            nodes["domain_id"][6], nodes["domain_id"][7], n_domains = R.NONE, 9, 4
        out[name] = (lws, groups, pst, pid, nodes, n_domains, 0)
    t = budget_world(n_lws=160, n_nodes=48, seed=5)
    out["breach"] = (t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    return out


@pytest.mark.parametrize("name", ["special", "node", "lifecycle", "breach"])
def test_small_tables(engine, name):
    lws, groups, pst, pid, nodes, n_domains, flags = small_worlds()[name]
    load(engine, lws, groups, pst, pid, nodes, n_domains, flags)
    fl = flags & R.SWEEP_GANG
    base = oracle.sweep_lws(lws, groups, pst, pid, nodes, fl)[:2]
    res = engine.resident_outputs()
    assert res[0].tobytes() == base[0].tobytes() and res[1].tobytes() == base[1].tobytes()
    cost = check_cost(engine, lws, groups, pst, pid, nodes, n_domains, base)
    for n in range(len(nodes)):
        got = engine.resident_drain_budget(nodes=[n])
        check_set(got, drain_budget_ref(lws, groups, pst, pid, nodes, [n], fl, base=base), (name, n))
        assert int(cost["nodes"]["min_margin"][n]) == min_margin_of(got["rows"])
    for d in range(n_domains):
        got = engine.resident_drain_budget(domains=[d])
        check_set(got, drain_budget_ref(lws, groups, pst, pid, nodes, domain_nodes(nodes, n_domains, [d]), fl, base=base),
                  (name, "domain", d))
        assert got["n_touched"] == cost["domains"]["lws_touched"][d]
    for ids in ([], list(range(n_domains)), [0, 0, 1]):
        got = engine.resident_drain_budget(domains=ids)
        check_set(got, drain_budget_ref(lws, groups, pst, pid, nodes, domain_nodes(nodes, n_domains, ids), fl, base=base),
                  (name, ids))


def test_c3(engine, c3):
    """At C3: both per-key forms against the reference, and the set form for one node, one domain and 1 % of
    the nodes against the spec oracle."""
    t = c3
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    fl = t.flags & R.SWEEP_GANG
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl, threads=16)[:2]
    res = engine.resident_outputs()
    assert res[0].tobytes() == base[0].tobytes() and res[1].tobytes() == base[1].tobytes()
    cost = check_cost(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, base)
    assert cost["nodes"]["lws_touched"].sum() > 0
    rng = np.random.default_rng(9)
    dom = int(rng.integers(0, t.n_domains))
    for label, kw, d in (("one", {"nodes": [3]}, [3]),
                         ("domain", {"domains": [dom]}, domain_nodes(t.nodes, t.n_domains, [dom])),
                         ("percent", None, rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False))):
        got = engine.resident_drain_budget(**(kw or {"nodes": d}))
        check_set(got, drain_budget_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, d, fl, base=base), label)
        assert got["n_touched"] > 0


def test_breach_world(engine, breach):
    """Floors that bind: breaches, LOSES_AVAILABLE and ALREADY_BELOW each several hundred times."""
    t = breach
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    fl = t.flags & R.SWEEP_GANG
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl)[:2]
    cost = check_cost(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, base)
    for scope in ("nodes", "domains"):
        assert cost[scope]["lws_breached"].sum() >= 300, scope
        assert cost[scope]["lws_loses_available"].sum() >= 300, scope
    seen = {"n_breached": 0, "n_loses_available": 0}
    rng = np.random.default_rng(2)
    for d in rng.choice(t.n_domains, size=8, replace=False).tolist():
        got = engine.resident_drain_budget(domains=[d])
        ref = drain_budget_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes,
                               domain_nodes(t.nodes, t.n_domains, [d]), fl, base=base)
        check_set(got, ref, d)
        for k in seen:
            seen[k] += got[k]
        assert got["n_already_below"] >= 300
        c = cost["domains"][d]
        assert (c["lws_touched"], c["lws_breached"], c["lws_loses_available"]) == \
               (got["n_touched"], got["n_breached"], got["n_loses_available"])
    assert all(v > 0 for v in seen.values()), seen
    nodes = rng.choice(len(t.nodes), size=len(t.nodes) // 10, replace=False)
    check_set(engine.resident_drain_budget(nodes=nodes),
              drain_budget_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, nodes, fl, base=base), "10 %")


def test_table_growth(engine):
    """A world with several times C3's (group, key) pairs, after a small one on the same engine: the table grows
    and every row stays exact."""
    lws, groups, pst, pid, nodes, n_domains, flags = small_worlds()["breach"]
    load(engine, lws, groups, pst, pid, nodes, n_domains, flags)
    engine.resident_drain_budget_cost("nodes")
    t = budget_world(n_lws=60_000, n_nodes=8192, seed=11)
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    base = engine.resident_outputs()
    got = engine.resident_drain_budget_cost("nodes")
    ref = drain_budget_cost_ref(t.lws, base[0], t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, base[1])
    assert got.tobytes() == ref.tobytes()
    assert int(got["groups_restarted"].sum()) > 3 * 412_029  # (C3's (group, node) pairs)


def test_isolation_from_ticks_in_flight(engine, c3):
    """Budget calls between the submit and wait of two ticks in flight: every tick's change lists, the final rows,
    occupancy, node and tick info equal a run without them."""
    t = c3
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(8):
        rows = np.sort(rng.choice(len(t.pod_state), size=2000, replace=False)).astype(np.uint32)
        sets.append([(R.TABLE_POD_STATE, rows, (t.pod_state[rows] ^ np.uint8(R.POD_ANY_RESTART)).astype(np.uint8))])
    doms = rng.choice(t.n_domains, size=8, replace=False)

    def run(with_budget):
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
            if with_budget:
                assert engine.resident_drain_budget(nodes=[])["n_touched"] == 0, k
                engine.resident_drain_budget(domains=[int(doms[k])])
                engine.resident_drain_budget_cost("domains")
                engine.resident_drain_budget_cost("nodes")
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


def raw(e, ids=None, n_ids=0, scope=R.DRAIN_NODES, capacity=0, rows=None):
    q = R.DrainBudgetQuery()
    q.ids, q.n_ids, q.scope, q.capacity, q.rows = ids, n_ids, scope, capacity, rows
    return E.lib().lwse_resident_drain_budget(e._h, C.byref(q))


def test_errors_and_capacity(breach):
    t = breach
    e = E.Engine(0)
    try:
        one = np.array([1], np.uint32)
        out = R.aligned_empty(len(t.nodes), R.DRAIN_BUDGET_COST)
        cost = E.lib().lwse_resident_drain_budget_cost
        assert raw(e, R.ptr(one), 1) == ERR_NOT_READY  # nothing loaded
        assert cost(e._h, R.DRAIN_NODES, R.ptr(out)) == ERR_NOT_READY
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        e.resident_tick(e.make_tick((), t.flags))
        assert raw(e, R.ptr(one), 1) == ERR_NOT_READY  # no node table
        e.upload_nodes(t.nodes, t.n_domains)
        assert raw(e, R.ptr(one), 1) == 0 and raw(e, R.ptr(one), 1, R.DRAIN_DOMAINS) == 0
        assert E.lib().lwse_resident_drain_budget(e._h, None) == ERR_INVALID_ARG
        assert cost(e._h, R.DRAIN_NODES, None) == ERR_INVALID_ARG
        assert cost(e._h, 2, R.ptr(out)) == ERR_INVALID_ARG
        assert raw(e, R.ptr(one), 1, scope=2) == ERR_INVALID_ARG
        assert raw(e, R.ptr(np.array([len(t.nodes)], np.uint32)), 1) == ERR_INVALID_ARG
        assert raw(e, R.ptr(np.array([t.n_domains], np.uint32)), 1, R.DRAIN_DOMAINS) == ERR_INVALID_ARG
        assert raw(e, None, 1) == ERR_INVALID_ARG
        assert raw(e, R.ptr(one), 1, capacity=4) == ERR_INVALID_ARG
        # LWS or group rows patched without a sweep: not ready until the next sweep
        for table, vals in ((R.TABLE_LWS, t.lws[:1]), (R.TABLE_GROUPS, t.groups[:1])):
            e.resident_patch(table, [0], vals)
            assert raw(e, R.ptr(one), 1) == ERR_NOT_READY
            assert cost(e._h, R.DRAIN_DOMAINS, R.ptr(out)) == ERR_NOT_READY
            e.resident_tick(e.make_tick((), t.flags))
            assert raw(e, R.ptr(one), 1) == 0
        fl = t.flags & R.SWEEP_GANG
        base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl)[:2]
        d = list(range(t.n_domains // 2))
        ref_rows, ref = drain_budget_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes,
                                         domain_nodes(t.nodes, t.n_domains, d), fl, base=base)
        assert ref["n_touched"] > 10
        small = e.resident_drain_budget(domains=d, capacity=7)
        assert len(small["rows"]) == 7 and all(small[k] == ref[k] for k in TOTALS)
        for r in small["rows"]:
            assert r.tobytes() == ref_rows[np.searchsorted(ref_rows["lws"], r["lws"])].tobytes()
        assert len(e.resident_drain_budget(domains=d, capacity=0)["rows"]) == 0
    finally:
        e.close()


def test_informer_domains(engine):
    """whatif_drain_domains → the set form equals the drain of the domain's node rows; the report names objects."""
    from informer_world import make_world

    items, cluster = make_world(7, n_lws=18, n_nodes=40)
    enc = informer.IncrementalEncoder(items, cluster, "zone", spare=1.0, node_spare=8)
    lws, groups, pst, pid, _ = enc.full_tables()
    load(engine, lws, groups, pst, pid, enc.node_rec, enc.n_domains)
    vals = sorted(enc._domain_ids)[:2]
    by_dom = engine.resident_drain_budget(domains=enc.whatif_drain_domains(vals))
    rows = domain_nodes(enc.node_rec, enc.n_domains, enc.whatif_drain_domains(vals))
    by_node = engine.resident_drain_budget(nodes=rows)
    assert all(by_dom[k] == by_node[k] for k in TOTALS)
    assert by_dom["rows"][np.argsort(by_dom["rows"]["lws"])].tobytes() == \
           by_node["rows"][np.argsort(by_node["rows"]["lws"])].tobytes()
    for r, rep in zip(by_dom["rows"], enc.drain_budget_report(by_dom)):
        assert (rep["namespace"], rep["name"]) == enc.object_of_lws_row(int(r["lws"]))
