"""Scale headroom on the device (lwse_resident_scale_headroom): byte for byte against tests/scale_headroom_ref.py on the
edge worlds and the fuzz worlds, both masks, with and without ceilings; every SOLVED entry against the engine's own
composition (resident_rollout_place of the scale-only proposals P(H) and P(probe)), on those worlds and on every
exclusive C3 object; the current rows; a tick in flight; the launches of one call; the refusals."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import synth
from lws_b200 import records as R
from rollout_place_ref import fuzz_world
from scale_headroom_ref import COUNTERS, edge_queries, fuzz_query, headroom_world, scale_headroom_ref, triggers

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7
MASKS = (R.RPW_STRANDED, R.RPW_ALL)


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def load(engine, w):
    engine.upload_nodes(w.nodes, w.n_domains)
    engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    engine.resident_place_load(w.reqs, w.n_ns)
    engine.resident_tick(engine.make_tick((), w.flags | R.TICK_PLACE))


def _same_rows(g, x, where):
    bad = np.flatnonzero((g.view(np.uint8).reshape(len(g), 64) != x.view(np.uint8).reshape(len(x), 64)).any(axis=1))
    assert len(bad) == 0, f"{where}: entries {bad[:8].tolist()} differ: got {g[bad[:2]]}, want {x[bad[:2]]}"


def _same(got, want, where):
    _same_rows(got["rows"], want["rows"], where)
    for k in ("n_solved", "n_blocked", "n_at_ceiling", "headroom"):
        assert got[k] == want[k], f"{where}: {k}"


def _proposals(lws, rows, reps):
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = lws[np.asarray(rows, dtype=np.int64)]
    recs["replicas"] = reps
    return recs


def check_composition(engine, lws, rows, ns, got, mask, where):
    """Every SOLVED entry that is not BLOCKED: P(H) is clean, and P(probe) gives the answer row's counters (two
    batched rollout placements of the scale-only proposals)."""
    out = got["rows"]
    sel = np.flatnonzero(((out["flags"] & R.SHR_SOLVED) != 0) & ((out["flags"] & R.SHR_BLOCKED) == 0))
    assert len(sel) > 0, where
    r, v = rows[sel], ns[sel]
    at_h = engine.resident_rollout_place(r, v, _proposals(lws, r, out["max_replicas"][sel]))["rows"]
    at_p = engine.resident_rollout_place(r, v, _proposals(lws, r, out["probe"][sel]))["rows"]
    assert (at_h["peak"] == out["max_replicas"][sel]).all() and (at_p["peak"] == out["probe"][sel]).all(), where
    for j, i in enumerate(sel.tolist()):
        assert not triggers(at_h[j], mask), f"{where}: entry {i} triggers at H"
        ceil = bool(out["flags"][i] & R.SHR_AT_CEILING)
        assert triggers(at_p[j], mask) != ceil, f"{where}: entry {i} at its probe"
        for k in COUNTERS:
            assert int(at_p[j][k]) == int(out[i][k]), f"{where}: entry {i} {k}"
    blocked = np.flatnonzero((out["flags"] & R.SHR_BLOCKED) != 0)
    if len(blocked):
        cur = engine.resident_rollout_place(rows[blocked], ns[blocked])["rows"]
        assert all(triggers(c, mask) for c in cur), where


@pytest.mark.parametrize("fit_all", [False, True])
def test_edge_worlds_equal_the_reference(engine, fit_all):
    w, rows = headroom_world(fit_all)
    rr, nn, cc, _ = edge_queries(w, rows)
    load(engine, w)
    for mask in MASKS:
        for c in (None, cc):
            want = scale_headroom_ref(w, rr, nn, c, mask)
            got = engine.resident_scale_headroom(rr, nn, c, mask, current=True)
            _same(got, want, f"edge {fit_all} {mask} {c is not None}")
            _same_rows(got["current"], want["current"], "current rows")
            check_composition(engine, w.lws, rr, nn, got, mask, f"edge {fit_all} {mask}")
    assert got["rounds"] > 0


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_worlds_equal_the_reference(engine, seed):
    w = fuzz_world(seed)
    load(engine, w)
    rows, ns, ceil = fuzz_query(w, seed, n=200)
    for mask in MASKS:
        for c in (None, ceil):
            got = engine.resident_scale_headroom(rows, ns, c, mask, current=True)
            _same(got, scale_headroom_ref(w, rows, ns, c, mask), f"fuzz {seed} {mask} {c is not None}")
            _same_rows(got["current"], engine.resident_rollout_place(rows, ns)["rows"], "current rows")
            check_composition(engine, w.lws, rows, ns, got, mask, f"fuzz {seed}")


def test_c3_every_exclusive_object_equals_the_composition(engine):
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    rows = np.flatnonzero(t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY).astype(np.uint32)
    ns = t.ns_of_lws[rows].astype(np.uint32)
    for mask, ceil in ((R.RPW_STRANDED, None), (R.RPW_ALL, t.lws["replicas"][rows] + 8)):
        got = engine.resident_scale_headroom(rows, ns, ceil, mask)
        assert got["n_solved"] == int(((got["rows"]["flags"] & R.SHR_SOLVED) != 0).sum())
        check_composition(engine, t.lws, rows, ns, got, mask, f"C3 {mask}")


def test_tick_in_flight_is_isolated(engine):
    w = fuzz_world(2)
    load(engine, w)
    rows, ns, ceil = fuzz_query(w, 2, n=300)
    prow = np.asarray([1, 5, 9], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = w.reqs[prow]
    vals["leader_node"] = R.NONE
    seg = (R.TABLE_PLACE_REQS, prow, vals)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    engine.resident_tick_wait()
    ref_out = engine.resident_place_outputs().copy()
    after = engine.resident_scale_headroom(rows, ns, ceil)
    load(engine, w)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    mid = engine.resident_scale_headroom(rows, ns, ceil)  # behind the submitted tick
    engine.resident_tick_wait()
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    assert mid["rows"].tobytes() == after["rows"].tobytes()


def test_launches_of_one_call(engine):
    """Beyond the resident forecast's own launches: the rollout placement's setup with items (count, baseline totals,
    namespace index (3), scan, fill, capacities and solve (2), finish: 10), the setup and the finish kernels (2), and
    per round the round kernel, the scan, the fill, the capacities and the solve (2), the finish and the commit (7)."""
    w, rows = headroom_world()
    rr, nn, cc, _ = edge_queries(w, rows)
    load(engine, w)
    c0 = engine.launch_count
    engine.resident_forecast(steps=False)
    c1 = engine.launch_count
    got = engine.resident_scale_headroom(rr, nn, cc)
    c2 = engine.launch_count
    assert got["rounds"] > 0
    assert (c2 - c1) - (c1 - c0) == 12 + 7 * got["rounds"]


def _raw(engine, rows, ns, ceil=None, n=None, out=None, constraints=R.RPW_STRANDED, reserved=0):
    from lws_b200.engine import lib

    q = R.ScaleHeadroomQuery()
    q.rows = R.ptr(rows) if rows is not None else None
    q.ns = R.ptr(ns) if ns is not None else None
    q.ceilings = R.ptr(ceil) if ceil is not None else None
    q.n = len(rows) if n is None else n
    q.constraints, q.reserved = constraints, reserved
    o = R.aligned_empty(max(q.n, 1), R.SCALE_HEADROOM) if out is None else out
    q.out = R.ptr(o) if out is not False else None
    return lib().lwse_resident_scale_headroom(engine._h, C.byref(q))


def test_refusals():
    from lws_b200.engine import Engine, lib

    w = fuzz_world(3, 0.1)
    rows = np.arange(4, dtype=np.uint32)
    ns = np.zeros(4, np.uint32)
    e = Engine(0)
    try:
        assert _raw(e, rows, ns) == ERR_NOT_READY  # nothing loaded
        e.upload_nodes(w.nodes, w.n_domains)
        e.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        e.resident_sweep(w.flags)
        assert _raw(e, rows, ns) == ERR_NOT_READY  # no placement round
        e.resident_place_load(w.reqs, w.n_ns)
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns) == 0
        assert _raw(e, rows, ns, n=0) == 0
        q = R.ScaleHeadroomQuery()
        q.constraints, q.rounds, q.headroom = R.RPW_STRANDED, 7, 7
        assert lib().lwse_resident_scale_headroom(e._h, C.byref(q)) == 0 and (q.rounds, q.headroom) == (0, 0)
        assert _raw(e, None, ns, n=4) == ERR_INVALID_ARG
        assert _raw(e, rows, None, n=4) == ERR_INVALID_ARG
        assert _raw(e, rows, ns, out=False) == ERR_INVALID_ARG
        assert _raw(e, np.array([len(w.lws)], np.uint32), np.zeros(1, np.uint32)) == ERR_INVALID_ARG
        assert _raw(e, rows[:1], np.array([w.n_ns], np.uint32)) == ERR_INVALID_ARG
        for c in (0, R.RPW_BUMPED, R.RPW_ALL | 4):
            assert _raw(e, rows, ns, constraints=c) == ERR_INVALID_ARG
        assert _raw(e, rows, ns, reserved=1) == ERR_INVALID_ARG
        out = R.aligned_empty(4, R.SCALE_HEADROOM)
        out["flags"] = 0xABCD
        assert _raw(e, rows, ns, out=out, constraints=8) == ERR_INVALID_ARG
        assert (out["flags"] == 0xABCD).all()
        # a node table whose domains do not fit one CTA: the namespace form is not offered, nothing written
        e.upload_nodes(w.nodes, 5457)
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns, out=out) == ERR_UNSUPPORTED
        assert (out["flags"] == 0xABCD).all()
    finally:
        e.close()
    e = Engine(0)  # an engine with a peer exchange: refused
    try:
        e.upload_nodes(w.nodes, w.n_domains)
        e.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        e.resident_place_load(w.reqs, w.n_ns)
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns) == 0
        e.exchange_create(len(w.reqs) + 1, 1, 0)
        assert _raw(e, rows, ns) == ERR_UNSUPPORTED
    finally:
        e.close()
