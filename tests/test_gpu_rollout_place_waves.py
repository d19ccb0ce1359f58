"""Rollout placement waves on the device (lwse_resident_rollout_place_waves): byte for byte against
tests/rollout_place_waves_ref.py on the fuzz, edge and tie worlds in both query forms; the alone rows against
lwse_resident_rollout_place; every wave against the engine's own composition (resident_rollout_place's extra rows,
concatenated in query order, into one resident_place_whatif) and the first-fit property through it; every wave of a
C3 template bump; a tick in flight; the refusals."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import records as R
from lws_b200 import synth
from rollout_place_ref import fuzz_world, proposals
from rollout_place_waves_ref import ALL_MASKS, edge_queries, rollout_place_waves_ref, tie_world, waves_world
from test_rollout_place_waves import fuzz_query

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
    assert got["keys"].tobytes() == want["keys"].tobytes(), f"{where}: keys {got['keys']} != {want['keys']}"
    assert got["waves"].tobytes() == want["waves"].tobytes(), f"{where}: waves {got['waves']} != {want['waves']}"
    assert got["alone_rows"].tobytes() == want["alone_rows"].tobytes(), f"{where}: alone rows"
    for k in R.ROLLOUT_WAVES_TOTALS:
        assert got[k] == want[k], f"{where}: {k}"


def _run(engine, w, rows, ns, recs, cap, mask, where):
    got = engine.resident_rollout_place_waves(rows, ns, recs, max_waves=cap, constraints=mask, alone=True)
    _same(got, rollout_place_waves_ref(w, rows, ns, recs, max_waves=cap, constraints=mask, mode="ns"), where)
    return got


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_worlds_equal_the_reference(engine, seed):
    w = fuzz_world(seed)
    load(engine, w)
    rows, ns = fuzz_query(w, seed)
    for recs in (None, proposals(w.lws, rows, seed)[1]):
        for cap, mask in ((64, R.RPW_STRANDED), (2, R.RPW_BUMPED), (1, R.RPW_ALL)):
            _run(engine, w, rows, ns, recs, cap, mask, f"fuzz {seed} {cap} {mask}")


def test_edge_worlds_equal_the_reference(engine):
    w, rows = waves_world()
    load(engine, w)
    for label, (r, v, recs) in edge_queries(w, rows).items():
        for cap in (1, 2, 64):
            for mask in ALL_MASKS:
                _run(engine, w, r, v, recs, cap, mask, f"{label} {cap} {mask}")
    tw, r, v, recs = tie_world()
    load(engine, tw)
    for mask in ALL_MASKS:
        _run(engine, tw, r, v, recs, 64, mask, f"tie {mask}")
        _run(engine, tw, r[::-1].copy(), v, recs[::-1].copy(), 64, mask, f"tie reversed {mask}")


def test_alone_rows_equal_rollout_place(engine):
    w, rows = waves_world()
    load(engine, w)
    for label, (r, v, recs) in edge_queries(w, rows).items():
        got = engine.resident_rollout_place_waves(r, v, recs, alone=True)
        assert got["alone_rows"].tobytes() == engine.resident_rollout_place(r, v, recs)["rows"].tobytes(), label


def composition(engine, reqs, lws, rows, ns, recs, S):
    """The engine's own set form over the keys S (query order) → the wave's counts."""
    S = sorted(S)
    sub = engine.resident_rollout_place(rows[S], ns[S], None if recs is None else recs[S], extra=True)
    x = sub["extra"]
    q = engine.resident_place_whatif(extra=x)
    xp = (q["extra_out"]["flags"] & R.PLACE_PLACED) != 0
    lost = ((q["before"]["flags"] & R.PLACE_PLACED) != 0) & ((q["after"]["flags"] & R.PLACE_PLACED) == 0)
    grp = reqs["group"][q["rows"]].astype(np.int64)
    rns = reqs["ns"][q["rows"]].astype(np.int64)
    own = np.zeros(len(grp), bool)
    for i in S:
        gb, gc = int(lws["group_base"][rows[i]]), int(lws["group_count"][rows[i]])
        own |= (rns == int(ns[i])) & (grp >= gb) & (grp < gb + gc)
    c = {"n_keys": len(S), "surge": len(x), "placed": int(xp.sum()), "stranded": int((~xp).sum()),
         "own_lost": int((lost & own).sum()), "bumped": int((lost & ~own).sum()),
         "namespaces": len({int(ns[i]) for i in S})}
    for k in ("n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict"):
        c[k] = q[k]
    return c


def _verdicts(c):
    return (R.RPW_STRANDED if c["stranded"] else 0) | (R.RPW_BUMPED if c["own_lost"] or c["bumped"] else 0)


def _check_waves(engine, reqs, lws, rows, ns, recs, got, mask, where):
    for c, wave in enumerate(got["waves"]):
        S = np.flatnonzero((got["keys"]["status"] == R.ROLLW_PLANNED) & (got["keys"]["wave"] == c)).tolist()
        want = composition(engine, reqs, lws, rows, ns, recs, S)
        for k, v in want.items():
            assert int(wave[k]) == v, f"{where}: wave {c} {k}: {int(wave[k])} != {v}"
        assert not (_verdicts(want) & mask), f"{where}: wave {c} triggers"


def test_waves_equal_the_composition_and_first_fit_holds(engine):
    w, names = waves_world()
    load(engine, w)
    for label, (rows, ns, recs) in edge_queries(w, names).items():
        for mask in ALL_MASKS:
            got = engine.resident_rollout_place_waves(rows, ns, recs, constraints=mask)
            _check_waves(engine, w.reqs, w.lws, rows, ns, recs, got, mask, f"{label} {mask}")
            keys = got["keys"]
            for k in np.flatnonzero(keys["status"] == R.ROLLW_PLANNED).tolist():
                for c in range(int(keys["wave"][k])):  # every lower wave's probe at that point triggers
                    S = [i for i in range(k) if keys["status"][i] == R.ROLLW_PLANNED and keys["wave"][i] == c]
                    assert _verdicts(composition(engine, w.reqs, w.lws, rows, ns, recs, S + [k])) & mask, (label, k, c)


def test_c3_template_bump_of_every_exclusive_object(engine):
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    rows = np.flatnonzero(t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY).astype(np.uint32)
    ns = t.ns_of_lws[rows].astype(np.uint32)
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = t.lws[rows]
    recs["rev_hash"] ^= np.uint64(0x9E3779B97F4A7C15)
    recs["flags"] |= np.uint32(R.LWS_UPDATED)
    got = engine.resident_rollout_place_waves(rows, ns, recs, constraints=R.RPW_ALL)
    assert got["n_waves"] >= 1 and got["n_planned"] > 0
    assert got["n_planned"] + got["n_triggers_alone"] + got["n_no_wave"] + got["n_not_solved"] == len(rows)
    _check_waves(engine, reqs, t.lws, rows, ns, recs, got, R.RPW_ALL, "C3")


def test_tick_in_flight_is_isolated(engine):
    w = fuzz_world(2)
    load(engine, w)
    rows, ns = fuzz_query(w, 2)
    prow = np.asarray([1, 5, 9], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = w.reqs[prow]
    vals["leader_node"] = R.NONE
    seg = (R.TABLE_PLACE_REQS, prow, vals)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    engine.resident_tick_wait()
    ref_out = engine.resident_place_outputs().copy()
    after = engine.resident_rollout_place_waves(rows, ns, constraints=R.RPW_ALL)
    load(engine, w)
    engine.resident_tick_submit(engine.make_tick([seg], w.flags | R.TICK_PLACE))
    mid = engine.resident_rollout_place_waves(rows, ns, constraints=R.RPW_ALL)  # behind the submitted tick
    engine.resident_tick_wait()
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    assert mid["keys"].tobytes() == after["keys"].tobytes() and mid["waves"].tobytes() == after["waves"].tobytes()


def _raw(e, rows, ns, n=None, recs=None, max_waves=64, constraints=R.RPW_STRANDED, reserved=0, keys=True, waves=True):
    from lws_b200.engine import lib

    n = len(rows) if n is None else n
    q = R.RolloutPlaceWavesQuery()
    q.rows = R.ptr(rows) if rows is not None else None
    q.ns = R.ptr(ns) if ns is not None else None
    q.recs = recs
    q.n, q.max_waves, q.constraints, q.reserved = n, max_waves, constraints, reserved
    k = R.aligned_empty(max(n, 1), R.ROLLOUT_WAVE_KEY)
    k["status"] = 0xABCD
    wv = R.aligned_empty(64, R.ROLLOUT_WAVE)
    wv["n_keys"] = 0xABCD
    q.keys = R.ptr(k) if keys else None
    q.waves = R.ptr(wv) if waves else None
    q.n_waves = q.n_planned = 77
    rc = lib().lwse_resident_rollout_place_waves(e._h, C.byref(q))
    if rc != 0:  # a refused call writes nothing
        assert (k["status"] == 0xABCD).all() and (wv["n_keys"] == 0xABCD).all() and q.n_waves == 77 and q.n_planned == 77
    return rc


def test_refusals():
    from lws_b200.engine import Engine

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
        assert _raw(e, np.array([0, 1, 0], np.uint32), np.zeros(3, np.uint32)) == ERR_INVALID_ARG  # duplicate rows
        assert _raw(e, rows[:1], np.array([w.n_ns], np.uint32)) == ERR_INVALID_ARG  # ns out of range
        assert _raw(e, np.array([len(w.lws)], np.uint32), np.zeros(1, np.uint32)) == ERR_INVALID_ARG
        for kw in (dict(max_waves=0), dict(max_waves=65), dict(constraints=0), dict(constraints=4), dict(reserved=1),
                   dict(keys=False), dict(waves=False)):
            assert _raw(e, rows, ns, **kw) == ERR_INVALID_ARG, kw
        assert _raw(e, None, ns, n=4) == ERR_INVALID_ARG
        recs = R.aligned_empty(5, R.LWS_REC)
        recs[:4] = w.lws[rows]
        assert _raw(e, rows, ns, recs=R.ptr(recs) + 4) == ERR_INVALID_ARG  # misaligned
        # the 24-bit bound over the SOLVED entries' extra rows: proposals that add 2^23 groups between them
        big = np.flatnonzero(w.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY)[:64].astype(np.uint32)
        brecs = R.aligned_empty(len(big), R.LWS_REC)
        brecs[:] = w.lws[big]
        brecs["replicas"] = (1 << 25) // len(big)
        brecs["max_surge"] = 0
        brecs["flags"] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT)
        bns = np.zeros(len(big), np.uint32)
        surge = e.resident_rollout_place(big, bns, brecs)["n_surge"]  # (each entry alone stays below the bound)
        assert len(w.reqs) + surge >= 1 << 24, surge
        assert _raw(e, big, bns, recs=R.ptr(brecs)) == ERR_UNSUPPORTED
        e.upload_nodes(w.nodes, 5457)  # domains that do not fit one CTA: the namespace form is not offered
        e.resident_tick(e.make_tick((), w.flags | R.TICK_PLACE))
        assert _raw(e, rows, ns) == ERR_UNSUPPORTED
    finally:
        e.close()
    e = Engine(0)
    try:
        load(e, w)
        assert _raw(e, rows, ns) == 0
        e.exchange_create(len(w.reqs) + 1, 1, 0)
        assert _raw(e, rows, ns) == ERR_UNSUPPORTED
    finally:
        e.close()
