"""The rollout forecast on the device (lwse_ds_forecast_host / lwse_ds_resident_forecast) against the CPU
reference of tests/ds_forecast_ref.py, byte for byte: C4, fuzzed multi-role tables with BAD_TABLE rows,
the golden planner sequences and the reference flows, the resident tables after DS-tick patches (with
and without links), forecasts between DS ticks and inside pipelined LeaderWorkerSet ticks, truncated
trajectories and the error paths."""
import numpy as np
import pytest

import oracle
from ds_forecast_ref import ds_forecast
from lws_b200 import churn, encoder, synth
from lws_b200 import records as R
from test_ds_forecast import FLOWS, GOLDEN, SORT_REVISIONS, abc_item, golden_item, random_item

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6  # lwse_status


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def _same(got, want, where=""):
    assert got["ds"].tobytes() == want["ds"].tobytes(), f"{where}: per-DS forecast differs"
    assert got["roles"].tobytes() == want["roles"].tobytes(), f"{where}: per-role forecast differs"
    assert got["n_steps_needed"] == want["n_steps_needed"] and got["n_steps_written"] == want["n_steps_written"]
    if want["steps"] is None:
        assert got["steps"] is None
    else:
        assert got["steps"].tobytes() == want["steps"].tobytes(), f"{where}: trajectory rows differ"


def _fuzzed(n_ds, seed):
    t = synth.make_ds(n_ds, (2, 3, 5, 10), fuzz=0.05, seed=seed)
    ds = t.ds.copy()
    rng = np.random.default_rng(seed)
    bad = rng.choice(n_ds, size=max(n_ds // 200, 2), replace=False)
    ds["n_roles"][bad[0::2]] = 11
    ds["rev_base"][bad[1::2]] = len(t.revroles) - 1
    return ds, t.roles, t.revroles


def test_c4_equals_reference(engine):
    t = synth.make_ds(50_000, (2,))
    want = ds_forecast(t.ds, t.roles, t.revroles)
    got = engine.ds_forecast_host(t.ds, t.roles, t.revroles)
    _same(got, want, "C4")
    assert (got["ds"]["n_steps"] > 0).sum() > 10_000
    summ = engine.ds_forecast_host(t.ds, t.roles, t.revroles, steps=False)
    assert summ["ds"].tobytes() == got["ds"].tobytes() and summ["roles"].tobytes() == got["roles"].tobytes()
    assert summ["steps"] is None and summ["n_steps_written"] == 0


def test_fuzzed_multi_role_equals_reference(engine):
    ds, roles, rr = _fuzzed(20_000, 9)
    want = ds_forecast(ds, roles, rr)
    got = engine.ds_forecast_host(ds, roles, rr)
    _same(got, want, "fuzzed")
    assert ((got["ds"]["flags"] & R.DSF_BAD_TABLE) != 0).sum() >= 2


def test_golden_and_reference_flows_through_the_kernel(engine):
    items = [golden_item(c) for c in GOLDEN] + [abc_item(*f, o) for f in FLOWS for o in (("A", "B"), ("B", "A"))]
    from lws_b200 import api

    for revisions in SORT_REVISIONS:
        cfg = api.RollingUpdateConfiguration(maxSurge=1, maxUnavailable=0)
        n = len(revisions)
        ds = api.DisaggregatedSet("s", roles=[api.DisaggregatedRoleSpec("prefill", n, cfg),
                                              api.DisaggregatedRoleSpec("decode", n, cfg)])
        kids = []
        for h, tp, td in revisions:
            kids += [api.ChildLWS("prefill", h, 1, 1, float(tp)), api.ChildLWS("decode", h, 1, 1, float(td))]
        items.append(encoder.DsItem(ds, "new", kids))
    import random

    rng = random.Random(3)
    items += [random_item(rng) for _ in range(300)]
    t = encoder.encode_ds(items)
    _same(engine.ds_forecast_host(t.ds, t.roles, t.revroles), ds_forecast(t.ds, t.roles, t.revroles), "flows")


def _patches(rng, ds, roles, rr):
    """A DS tick's worth of revision-role patches (scattered) and one range of them, disjoint."""
    first = int(rng.integers(0, len(rr) - 64))
    rows = np.unique(rng.choice(len(rr), size=len(rr) // 100, replace=False)).astype(np.uint32)
    rows = rows[(rows < first) | (rows >= first + 64)]
    v = rr[rows].copy()
    v["ready_replicas"] = rng.integers(0, 33, size=len(rows))
    v["replicas"] = np.where(rng.random(len(rows)) < 0.3, rng.integers(0, 33, size=len(rows)), v["replicas"])
    rv = rr[first: first + 64].copy()
    rv["replicas"] = rng.integers(0, 33, size=64)
    return [(R.TABLE_DS_REVROLES, rows, v), (R.TABLE_DS_REVROLES, first, rv, True)]


@pytest.mark.parametrize("linked", [False, True])
def test_resident_forecast_after_patches(engine, linked):
    ds, roles, rr = _fuzzed(20_000, 21)
    rr = rr.copy()
    engine.ds_resident_load(ds, roles, rr)
    first = engine.ds_resident_tick()
    if linked:  # a link table makes the tick run the linked sweep; the forecast ignores links
        links = np.zeros(len(rr), R.DS_LINK)
        links["lws_row"] = np.where(np.arange(len(rr)) % 3 == 0, 5, 0xFFFFFFFF)
        engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)])
    rng = np.random.default_rng(2)
    for k in range(4):
        segs = _patches(rng, ds, roles, rr)
        for sg in segs:
            if len(sg) == 4:
                rr[sg[1]: sg[1] + len(sg[2])] = sg[2]
            else:
                rr[sg[1]] = sg[2]
        res = engine.ds_resident_tick(segs)
        mirror = {k2: res[k2].copy() for k2 in ("ds_out", "role_out", "revrole_out")}
        listed = res["rows"].copy()
        got = engine.ds_resident_forecast(steps=k % 2 == 0)
        _same(got, ds_forecast(ds, roles, rr, steps=k % 2 == 0), f"resident tick {k}")
        for k2 in mirror:  # the tick's outputs are untouched by the forecast
            assert res[k2].tobytes() == mirror[k2].tobytes()
        assert np.array_equal(res["rows"], listed)
    assert first["n_changed"] == len(ds)


def test_forecasts_between_ticks_change_no_tick(engine):
    """DS ticks with and without forecasts in between list the same rows and hold the same mirrors, and
    a forecast between an LWS submit and wait changes neither tick."""
    ds, roles, rr = _fuzzed(8000, 33)

    def run(with_forecast):
        r = rr.copy()
        engine.ds_resident_load(ds, roles, r)
        out = [engine.ds_resident_tick()]
        rng = np.random.default_rng(8)
        for k in range(5):
            segs = _patches(rng, ds, roles, r)
            if with_forecast:
                engine.ds_resident_forecast()
            res = engine.ds_resident_tick(segs)
            out.append((np.sort(res["rows"]).copy(), res["ds_out"].copy(), res["revrole_out"].copy()))
        return out[1:]

    a, b = run(False), run(True)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert u.tobytes() == v.tobytes()
    # inside pipelined LWS ticks
    t = synth.make("C3-steady", 0.02)
    t.ns_of_lws[:] = 0
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    reqs = encoder.encode_place_requests(t.lws, t.groups)
    engine.resident_place_load(reqs, 1)
    flags = t.flags | R.TICK_PLACE
    engine.resident_tick(engine.make_tick((), flags))
    occ = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, flags=t.flags, want_occupancy=True)[2]
    plan = churn.make_plan(t, reqs, oracle.place(t.nodes, occ, t.n_domains, 1, reqs), 0.02, 0.05, n_sets=2, seed=3)
    ticks = churn.ArenaPlan(engine, plan, flags).ticks
    pst, grp, rq = t.pod_state.copy(), t.groups.copy(), reqs.copy()
    rr2 = rr.copy()
    engine.ds_resident_load(ds, roles, rr2)
    engine.ds_resident_tick()
    for k in range(2):
        churn.apply_to_mirror(plan[k], pst, grp, rq)
        engine.resident_tick_submit(ticks[k])
        _same(engine.ds_resident_forecast(), ds_forecast(ds, roles, rr2), f"inside LWS tick {k}")
        engine.resident_tick_wait()
    w = oracle.sweep_lws(t.lws, grp, pst, t.pod_ident, t.nodes, flags=t.flags)
    g = engine.resident_outputs()
    assert g[0].tobytes() == w[0].tobytes() and g[1].tobytes() == w[1].tobytes()


def test_truncated_trajectory_keeps_guard_and_summaries(engine):
    ds, roles, rr = _fuzzed(5000, 5)
    full = ds_forecast(ds, roles, rr)
    cap = full["n_steps_needed"] // 3
    want = ds_forecast(ds, roles, rr, step_capacity=cap)
    # the engine fills a buffer with a guard region behind step_capacity
    import ctypes as C
    from lws_b200 import engine as E

    fc = R.aligned_empty(len(ds), R.DS_FORECAST)
    fr = R.aligned_empty(len(roles), R.DS_FORECAST_ROLE)
    buf = R.aligned_empty(cap + 4096, R.DS_ROLE_OUT)
    buf.view(np.uint8)[:] = 0xA5
    t = R.DsTables(R.ptr(ds), len(ds), R.ptr(roles), len(roles), R.ptr(rr), len(rr), None, None, None)
    out = R.DsForecastOut(R.ptr(fc), R.ptr(fr), R.ptr(buf), cap, 0, 0)
    assert E.lib().lwse_ds_forecast_host(engine._h, C.byref(t), C.byref(out)) == 0
    assert fc.tobytes() == want["ds"].tobytes() and fr.tobytes() == want["roles"].tobytes()
    assert out.n_steps_written == want["n_steps_written"] and out.n_steps_needed == full["n_steps_needed"]
    assert buf[: out.n_steps_written].tobytes() == want["steps"].tobytes()
    assert (buf.view(np.uint8)[out.n_steps_written * 8:] == 0xA5).all()
    trunc = (fc["flags"] & R.DSF_TRUNCATED) != 0
    assert trunc.any() and not trunc.all()
    fc["flags"] &= ~np.uint32(R.DSF_TRUNCATED)
    assert fc.tobytes() == full["ds"].tobytes()


def test_error_paths_change_nothing(engine):
    import ctypes as C
    from lws_b200 import engine as E
    from lws_b200.engine import Engine

    fresh = Engine(0)
    try:
        fc = R.aligned_empty(4, R.DS_FORECAST)
        fc.view(np.uint8)[:] = 0x5A
        out = R.DsForecastOut(R.ptr(fc), None, None, 0, 7, 9)
        assert E.lib().lwse_ds_resident_forecast(fresh._h, C.byref(out)) == ERR_NOT_READY
        assert (fc.view(np.uint8) == 0x5A).all() and out.n_steps_written == 7 and out.n_steps_needed == 9
    finally:
        fresh.close()
    ds, roles, rr = _fuzzed(2000, 6)
    engine.ds_resident_load(ds, roles, rr)
    before = engine.ds_resident_tick()
    mirror = before["revrole_out"].copy()
    assert E.lib().lwse_ds_resident_forecast(engine._h, None) == ERR_INVALID_ARG
    out = R.DsForecastOut(None, None, None, 0, 7, 9)  # n_ds > 0 but no per-DS output
    assert E.lib().lwse_ds_resident_forecast(engine._h, C.byref(out)) == ERR_INVALID_ARG
    assert out.n_steps_written == 7 and out.n_steps_needed == 9
    t = R.DsTables(R.ptr(ds), len(ds), R.ptr(roles), len(roles), R.ptr(rr), len(rr), None, None, None)
    assert E.lib().lwse_ds_forecast_host(engine._h, C.byref(t), C.byref(out)) == ERR_INVALID_ARG
    assert E.lib().lwse_ds_forecast_host(engine._h, None, C.byref(out)) == ERR_INVALID_ARG
    again = engine.ds_resident_tick()
    assert again["n_changed"] == 0 and again["revrole_out"].tobytes() == mirror.tobytes()
    _same(engine.ds_resident_forecast(), ds_forecast(ds, roles, rr), "after errors")


def test_overlapping_ranges_write_only_their_reserved_rows(engine):
    """DS whose row ranges overlap another DS's get unspecified results, but no DS writes outside the
    trajectory rows the scan reserved for it: the guard region behind step_capacity stays untouched, and
    the DS with rows of their own still equal the reference."""
    import ctypes as C
    from lws_b200 import engine as E

    t = synth.make_ds(4000, (2, 3, 5), seed=12)
    ds = t.ds.copy()
    shared = np.arange(0, 4000 - 64, 16)  # DS d takes the ranges of DS d + 40 (another warp, not in `shared`)
    for f in ("role_base", "n_roles", "n_spec_roles", "rev_base", "n_old_revs"):
        ds[f][shared] = ds[f][shared + 40]
    own = np.ones(len(ds), bool)
    own[shared] = own[shared + 40] = False
    want = ds_forecast(t.ds, t.roles, t.revroles)
    tabs = R.DsTables(R.ptr(ds), len(ds), R.ptr(t.roles), len(t.roles), R.ptr(t.revroles), len(t.revroles),
                      None, None, None)
    for k in range(3):
        fc = R.aligned_empty(len(ds), R.DS_FORECAST)
        fr = R.aligned_empty(len(t.roles), R.DS_FORECAST_ROLE)
        probe = R.DsForecastOut(R.ptr(fc), R.ptr(fr), None, 0, 0, 0)
        assert E.lib().lwse_ds_forecast_host(engine._h, C.byref(tabs), C.byref(probe)) == 0
        cap = int(probe.n_steps_needed) // (k + 1)
        buf = R.aligned_empty(cap + 4096, R.DS_ROLE_OUT)
        buf.view(np.uint8)[:] = 0xA5
        out = R.DsForecastOut(R.ptr(fc), R.ptr(fr), R.ptr(buf), cap, 0, 0)
        assert E.lib().lwse_ds_forecast_host(engine._h, C.byref(tabs), C.byref(out)) == 0
        assert out.n_steps_written <= cap
        assert (buf.view(np.uint8)[out.n_steps_written * 8:] == 0xA5).all()
        for d in np.nonzero(own)[0]:
            got, exp = fc[d].copy(), want["ds"][d].copy()
            got["step_base"] = exp["step_base"] = 0
            got["flags"] &= ~np.uint32(R.DSF_TRUNCATED)
            assert got.tobytes() == exp.tobytes(), f"DS {d}"
            b, n = int(ds["role_base"][d]), int(ds["n_roles"][d])
            assert fr[b: b + n].tobytes() == want["roles"][b: b + n].tobytes()
            if fc[d]["n_steps"] and not fc[d]["flags"] & R.DSF_TRUNCATED:
                s0, s1 = int(fc[d]["step_base"]), int(want["ds"][d]["step_base"])
                m = int(fc[d]["n_steps"]) * n
                assert buf[s0: s0 + m].tobytes() == want["steps"][s1: s1 + m].tobytes()
