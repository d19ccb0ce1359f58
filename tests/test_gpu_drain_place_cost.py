"""Drain placement on the device (lwse_resident_drain_place_cost): every key of the CPU worlds (the built world of
the locality rule's edges, namespaces past kNsCache unpinned requests and past kNsKeep x 512 rows, seeded informer
worlds), both scopes, byte for byte against the pruned reference (tests/drain_place_ref.py); at C3 every domain key
and every node key against the engine's own three-call composition (drain what-if → unpin → place what-if), with
more items than resident CTAs, and groups_restarted against the drain budget; isolation from a tick in flight;
the errors."""
import numpy as np
import pytest

from drain_place_ref import drain_place_ref
from lws_b200 import synth
from lws_b200 import records as R
from test_drain_place_cost import WORLDS

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7
RESTART = R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def c3():
    return synth.make("C3", 1.0, seed=synth.SEED)


def load(engine, lws, groups, pst, pid, nodes, nd, reqs, n_ns, flags=0):
    engine.upload_nodes(nodes, nd)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, n_ns)
    engine.resident_tick(engine.make_tick((), flags | R.TICK_PLACE))


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", list(WORLDS))
def test_every_key_matches_the_reference(engine, name, by_domain):
    lws, groups, pst, pid, nodes, nd, _, reqs, n_ns = WORLDS[name]()
    load(engine, lws, groups, pst, pid, nodes, nd, reqs, n_ns)
    occ = engine.resident_occupancy()
    got = engine.resident_drain_place_cost("domains" if by_domain else "nodes")
    ref = drain_place_ref(lws, groups, pst, pid, nodes, nd, occ, reqs, n_ns, by_domain, pruned=True,
                          base_place=engine.resident_place_outputs())
    for k in range(len(ref)):
        assert got[k].tobytes() == ref[k].tobytes(), (name, by_domain, k, got[k], ref[k])
    if name == "big_namespaces":
        assert got["unpinned"].max() >= 257
    if name == "built":  # the full node is full on the device too, and the capacity clause's holders move
        assert int(occ[3]) == int(nodes["capacity"][3])
        if not by_domain:
            assert got["n_moved"][:2].any() or got["n_lost"][:2].any()


def composition(engine, t, reqs, drained):
    """The three calls for one drain set: restarted groups, their requests and the drained nodes' leaders
    unpinned, the place what-if with the cordon → DRAIN_PLACE_COST fields (namespaces_solved left 0)."""
    wf = engine.resident_drain_whatif(drained)
    hit = ((wf["before"]["flags"] & RESTART) == 0) & ((wf["after"]["flags"] & RESTART) != 0)
    restarted = wf["rows"][hit].astype(np.int64)
    leader = reqs["leader_node"].astype(np.int64)
    g = reqs["group"].astype(np.int64)
    u = np.flatnonzero((leader != R.NONE) & (np.isin(leader, drained) | ((g < len(t.groups)) & np.isin(g, restarted))))
    nrows = np.asarray(sorted(set(int(n) for n in drained)), dtype=np.uint32)
    nv = R.aligned_empty(len(nrows), R.NODE_REC)
    nv[:] = t.nodes[nrows]
    nv["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
    rv = R.aligned_empty(len(u), R.PLACE_REQ)
    rv[:] = reqs[u]
    rv["leader_node"] = R.NONE
    segs = [(R.TABLE_NODES, nrows, nv)] + ([(R.TABLE_PLACE_REQS, u.astype(np.uint32), rv)] if len(u) else [])
    q = engine.resident_place_whatif(segs)
    before = engine.resident_place_outputs()
    after = before.copy()
    after[q["rows"]] = q["after"]
    in_u = np.zeros(len(reqs), bool)
    in_u[u] = True
    was, now = (before["flags"] & R.PLACE_PLACED) != 0, (after["flags"] & R.PLACE_PLACED) != 0
    row = np.zeros(1, R.DRAIN_PLACE_COST)[0]
    row["groups_restarted"] = wf["n_groups_restarted"]
    row["unpinned"] = len(u)
    row["stranded"] = int((in_u & ~now).sum())
    row["bumped"] = int((~in_u & was & ~now).sum())
    for f in ("n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict"):
        row[f] = q[f]
    return row


@pytest.mark.parametrize("scope", ["domains", "nodes"])
def test_c3_matches_the_three_call_composition(engine, c3, scope):
    t = c3
    reqs = t.place_requests()
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, reqs, t.n_namespaces, t.flags)
    got = engine.resident_drain_place_cost(scope)
    budget = engine.resident_drain_budget_cost(scope)
    assert np.array_equal(got["groups_restarted"], budget["groups_restarted"])
    if scope == "nodes":
        assert np.array_equal(got["groups_restarted"], engine.resident_drain_cost()["groups_restarted"])
        keys = range(len(t.nodes))
    else:
        keys = range(t.n_domains)
    d = t.nodes["domain_id"].astype(np.int64)
    for k in keys:
        drained = np.array([k]) if scope == "nodes" else np.flatnonzero(d == k)
        want = composition(engine, t, reqs, drained)
        row = got[k].copy()
        row["namespaces_solved"] = 0
        assert row.tobytes() == want.tobytes(), (scope, k, got[k], want)
    assert got["unpinned"].any() and got["n_changed"].any()


def test_isolation_from_a_tick_in_flight(engine, c3):
    t = c3
    reqs = t.place_requests()
    load(engine, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, reqs, t.n_namespaces, t.flags)
    want = engine.resident_drain_place_cost("domains")
    rows = np.asarray([3, 7, 11], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = reqs[rows]
    vals["size"] += 1
    seg = (R.TABLE_PLACE_REQS, rows, vals)
    # the reference run: the tick alone
    engine.resident_tick_submit(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    engine.resident_tick_wait()
    ref_out = engine.resident_place_outputs().copy()
    vals["size"] -= 1
    engine.resident_tick(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    base = engine.resident_place_outputs().copy()
    # the same tick with the call between its submit and wait: its snapshot orders behind the tick
    vals["size"] += 1
    engine.resident_tick_submit(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    mid = engine.resident_drain_place_cost("domains")
    engine.resident_tick_wait()
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    vals["size"] -= 1
    engine.resident_tick(engine.make_tick([seg], t.flags | R.TICK_PLACE))
    assert engine.resident_place_outputs().tobytes() == base.tobytes()
    assert engine.resident_drain_place_cost("domains").tobytes() == want.tobytes()
    assert mid["groups_restarted"].tobytes() == want["groups_restarted"].tobytes()


def test_errors(c3):
    import ctypes as C

    from lws_b200.engine import Engine, LwseError, lib

    t = c3
    reqs = t.place_requests()
    e = Engine(0)
    try:
        e.upload_nodes(t.nodes, t.n_domains)
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        with pytest.raises(LwseError) as ei:
            e.resident_drain_place_cost("nodes")  # no placement round yet
        assert ei.value.status == ERR_NOT_READY
        out = R.aligned_empty(len(t.nodes), R.DRAIN_PLACE_COST)
        e.resident_place_load(reqs, t.n_namespaces)
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        assert lib().lwse_resident_drain_place_cost(e._h, C.c_uint32(7), R.ptr(out)) == ERR_INVALID_ARG
        e.upload_nodes(t.nodes, 5457)  # the domains do not fit one CTA: the namespace form is not offered
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        with pytest.raises(LwseError) as ei:
            e.resident_drain_place_cost("domains")
        assert ei.value.status == ERR_UNSUPPORTED
    finally:
        e.close()
