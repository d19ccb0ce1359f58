"""Rollout placement on the device (lwse_resident_rollout_place): byte for byte against tests/rollout_place_ref.py on
the fuzz worlds and the edge world, in resident and proposal forms; every entry against the engine's own composition
(resident_forecast / resident_rollout_whatif → the informer's extra rows → resident_place_whatif) on an informer world
and on every C3 object with extra rows; a tick in flight; the refusals; the launches of one call."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import informer, synth
from lws_b200 import records as R
from rollout_place_ref import edge_queries, edge_world, extra_groups, fuzz_world, proposals, rollout_place_ref

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7


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


def _same(got, want, where):
    """Rows, totals and (when the call returned them) the extra rows, against the reference."""
    if "extra" in got:
        wx = [x for x in want["extra"] if len(x)]
        wx = np.concatenate(wx).view(R.PLACE_REQ) if wx else np.zeros(0, R.PLACE_REQ)
        assert got["extra"].tobytes() == wx.tobytes(), f"{where}: extra rows differ from the encoder's"
    g, x = got["rows"], want["rows"]
    bad = np.flatnonzero((g.view(np.uint8).reshape(len(g), 64) != x.view(np.uint8).reshape(len(x), 64)).any(axis=1))
    assert len(bad) == 0, f"{where}: entries {bad[:8].tolist()} differ: got {g[bad[:2]]}, want {x[bad[:2]]}"
    for k in R.ROLLOUT_PLACE_TOTALS:
        assert got[k] == want[k], f"{where}: {k}"


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_worlds_equal_the_reference(engine, seed):
    w = fuzz_world(seed)
    load(engine, w)
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, len(w.lws), 200).astype(np.uint32)
    ns = (rows.astype(np.int64) % w.n_ns).astype(np.uint32)
    _same(engine.resident_rollout_place(rows, ns, extra=True), rollout_place_ref(w, rows, ns), f"fuzz {seed}")
    recs = proposals(w.lws, rows, seed)[1]
    _same(engine.resident_rollout_place(rows, ns, recs, extra=True), rollout_place_ref(w, rows, ns, recs=recs),
          f"fuzz {seed} proposals")


def test_edge_world_equals_the_reference(engine):
    w, rows = edge_world()
    (rr, rn), (pr, pn, recs), labels = edge_queries(w, rows)
    load(engine, w)
    _same(engine.resident_rollout_place(rr, rn, extra=True), rollout_place_ref(w, rr, rn), "edge")
    _same(engine.resident_rollout_place(pr, pn, recs, extra=True), rollout_place_ref(w, pr, pn, recs=recs), "edge proposals")
    # a capacity below n_surge lists the first rows only
    full = engine.resident_rollout_place(pr, pn, recs, extra=True)
    xs = R.aligned_empty(4, R.PLACE_REQ)
    assert _raw(engine, pr, pn, recs=R.ptr(recs), extra=xs) == 0
    assert xs.tobytes() == full["extra"][:4].tobytes()


def composition(engine, lws, groups, rows, ns, recs=None):
    """The engine's own composition per entry → ROLLOUT_PLACE rows of the entries it solves (others zero)."""
    if recs is None:
        fc = engine.resident_forecast(steps=False)["lws"][np.asarray(rows, dtype=np.int64)]
    else:
        fc = engine.resident_rollout_whatif(rows, recs, steps=False)["lws"]
    out = np.zeros(len(rows), R.ROLLOUT_PLACE)
    for i, r in enumerate(np.asarray(rows).tolist()):
        rec = lws[r] if recs is None else recs[i]
        gb, gc = int(lws["group_base"][r]), int(lws["group_count"][r])
        w = type("W", (), {"lws": lws, "groups": groups})
        x = informer.IncrementalEncoder._whatif_requests(int(rec["uid_hash"]), int(rec["size"]), int(ns[i]),
                                                         extra_groups(w, r, int(fc[i]["peak_sts_replicas"])))
        x["group"] = (x["group"].astype(np.int64) + gb).astype(np.uint32)
        q = engine.resident_place_whatif(extra=x)
        o = out[i]
        o["surge"] = len(x)
        xp = (q["extra_out"]["flags"] & R.PLACE_PLACED) != 0
        o["placed"], o["stranded"] = int(xp.sum()), int((~xp).sum())
        lost = ((q["before"]["flags"] & R.PLACE_PLACED) != 0) & ((q["after"]["flags"] & R.PLACE_PLACED) == 0)
        grp = engine_reqs_group(engine)[q["rows"]].astype(np.int64)
        own = (grp >= gb) & (grp < gb + gc)
        o["own_lost"], o["bumped"] = int((lost & own).sum()), int((lost & ~own).sum())
        for k in ("n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict",
                  "namespaces_solved"):
            o[k] = q[k]
        out[i] = o
    return out


_REQS = {}


def engine_reqs_group(engine):
    return _REQS[id(engine)]["group"]


def _check_composition(engine, lws, groups, reqs, rows, ns, recs=None, where=""):
    _REQS[id(engine)] = reqs
    got = engine.resident_rollout_place(rows, ns, recs)["rows"]
    solved = (got["flags"] & R.RPL_SOLVED) != 0
    assert solved.any(), where
    want = composition(engine, lws, groups, rows[solved], ns[solved], None if recs is None else recs[solved])
    cols = ["surge", "placed", "stranded", "own_lost", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed",
            "n_unschedulable", "n_conflict", "namespaces_solved"]
    for c in cols:
        assert got[solved][c].tolist() == want[c].tolist(), f"{where}: {c}"


def test_informer_world_equals_the_composition(engine):
    from informer_world import make_world

    items, cluster = make_world(3, n_lws=14, n_nodes=28)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    lws, groups, pst, pid, reqs = enc.full_tables()
    engine.upload_nodes(enc.node_rec, enc.n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, enc.n_namespaces)
    engine.resident_tick(engine.make_tick((), R.TICK_PLACE))
    rows, ns = enc.rollout_place_query()
    _check_composition(engine, lws, groups, reqs, rows, ns, where="informer")
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    for i, k in enumerate(sorted(k for k in enc.slots if enc.slots[k].lws_row in set(rows.tolist()))):
        recs[i] = enc.rollout_place_proposal(enc.items[k])[1]
    recs["replicas"] += 2  # a scale-up per object: two more groups each
    _check_composition(engine, lws, groups, reqs, rows, ns, recs, where="informer proposals")
    enc.rollout_place_report(engine.resident_rollout_place(rows, ns, recs))


def test_c3_every_object_with_extra_rows_equals_the_composition(engine):
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    rows = np.arange(len(t.lws), dtype=np.uint32)
    ns = t.ns_of_lws.astype(np.uint32)
    got = engine.resident_rollout_place(rows, ns)
    sel = np.flatnonzero(got["rows"]["surge"] > 0)
    assert len(sel) > 0 and got["n_solved"] == int(((got["rows"]["flags"] & R.RPL_SOLVED) != 0).sum())
    _check_composition(engine, t.lws, t.groups, reqs, rows[sel], ns[sel], where="C3")


def test_tick_in_flight_is_isolated(engine):
    w = fuzz_world(2)
    load(engine, w)
    rows = np.arange(min(len(w.lws), 300), dtype=np.uint32)
    ns = (rows.astype(np.int64) % w.n_ns).astype(np.uint32)
    prow = np.asarray([1, 5, 9], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = w.reqs[prow]
    vals["leader_node"] = R.NONE
    seg = (R.TABLE_PLACE_REQS, prow, vals)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    engine.resident_tick_wait()
    ref_out = engine.resident_place_outputs().copy()
    after = engine.resident_rollout_place(rows, ns)
    load(engine, w)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    mid = engine.resident_rollout_place(rows, ns)  # behind the submitted tick
    engine.resident_tick_wait()
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    assert mid["rows"].tobytes() == after["rows"].tobytes()


def _raw(engine, rows, ns, recs=None, n=None, out=None, extra=None):
    from lws_b200.engine import lib

    q = R.RolloutPlaceQuery()
    q.rows = R.ptr(rows) if rows is not None else None
    q.ns = R.ptr(ns) if ns is not None else None
    q.recs = recs
    q.n = len(rows) if n is None else n
    o = R.aligned_empty(max(q.n, 1), R.ROLLOUT_PLACE) if out is None else out
    q.out = R.ptr(o)
    if extra is not None:
        q.extra, q.extra_capacity = R.ptr(extra), len(extra)
    return lib().lwse_resident_rollout_place(engine._h, C.byref(q))


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
        assert _raw(e, rows, ns) == ERR_NOT_READY  # no sweep, no placement round
        e.resident_sweep(w.flags)
        assert _raw(e, rows, ns) == ERR_NOT_READY  # no placement round
        e.resident_place_load(w.reqs, w.n_ns)
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns) == 0
        assert _raw(e, None, ns, n=4) == ERR_INVALID_ARG
        assert _raw(e, rows, None, n=4) == ERR_INVALID_ARG
        assert _raw(e, np.array([len(w.lws)], np.uint32), np.zeros(1, np.uint32)) == ERR_INVALID_ARG
        assert _raw(e, rows[:1], np.array([w.n_ns], np.uint32)) == ERR_INVALID_ARG
        recs = R.aligned_empty(5, R.LWS_REC)
        recs[:4] = w.lws[rows]
        assert _raw(e, rows, ns, recs=R.ptr(recs) + 4) == ERR_INVALID_ARG  # misaligned
        assert _raw(e, rows, ns, n=0) == 0
        q = R.RolloutPlaceQuery()  # extra rows asked for without a buffer
        q.rows, q.ns, q.n, q.out, q.extra_capacity = R.ptr(rows), R.ptr(ns), 4, R.ptr(R.aligned_empty(4, R.ROLLOUT_PLACE)), 8
        assert lib().lwse_resident_rollout_place(e._h, C.byref(q)) == ERR_INVALID_ARG
        # the proposals' slots reach the forecast's limit (2^31): 2 048 proposals of 2^20 slots each (C = replicas), nothing written
        big = np.zeros(2048, np.uint32)
        brecs = R.aligned_empty(2048, R.LWS_REC)
        brecs[:] = w.lws[0]
        brecs["replicas"] = 1 << 20
        brecs["max_surge"] = 0
        brecs["flags"] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT)
        out = R.aligned_empty(2048, R.ROLLOUT_PLACE)
        out["flags"] = 0xABCD
        q = R.RolloutPlaceQuery()
        q.rows, q.ns, q.recs, q.n, q.out = R.ptr(big), R.ptr(big), R.ptr(brecs), 2048, R.ptr(out)
        q.n_solved, q.n_surge = 77, 77
        assert lib().lwse_resident_rollout_place(e._h, C.byref(q)) == ERR_UNSUPPORTED
        assert (out["flags"] == 0xABCD).all() and q.n_solved == 77 and q.n_surge == 77  # nothing written
        # a what-if node table whose domains do not fit one CTA: the namespace form is not offered
        e.upload_nodes(w.nodes, 5457)
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns) == ERR_UNSUPPORTED
    finally:
        e.close()
    # an engine with a peer exchange (the shared-occupancy round): refused
    e = Engine(0)
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


def test_launches_of_one_call(engine):
    """Beyond the forecast's own launches (resident_forecast / resident_rollout_whatif, summaries only): the count
    kernel, the baseline totals, then with items the namespace index (3), the scan, the fill, the capacities and
    the solve (2) and the finish: 10; without items the solve's four are skipped: 5."""
    w, rows = edge_world()
    (rr, rn), (pr, pn, recs), _ = edge_queries(w, rows)
    load(engine, w)
    for q, fc in (((rr, rn), lambda: engine.resident_forecast(steps=False)),
                  ((pr, pn, recs), lambda: engine.resident_rollout_whatif(pr, recs, steps=False))):
        c0 = engine.launch_count
        fc()
        c1 = engine.launch_count
        engine.resident_rollout_place(*q)
        c2 = engine.launch_count
        assert (c2 - c1) - (c1 - c0) == 10
    sel = np.asarray([rows["A"]], np.uint32)  # A: no extra rows
    c0 = engine.launch_count
    engine.resident_forecast(steps=False)
    c1 = engine.launch_count
    engine.resident_rollout_place(sel, np.zeros(1, np.uint32))
    c2 = engine.launch_count
    assert (c2 - c1) - (c1 - c0) == 5
