"""The four paths of the DS sweep body (the stateless ``lwse_sweep_ds_*``, the resident DS tick, the
linked DS tick and the rollout forecast) on the limit tables of ``ds_limits_world``: 32 old revisions,
10 roles with removed ones, creation stamps out of row order, bit 31 of ``drained_revs`` /
``ready_revs``, targets near 10^5 with percent surges, and DS rows just past the format.  Every check
is a byte comparison with ``oracle.sweep_ds`` or ``ds_forecast_ref.ds_forecast``."""
import numpy as np
import pytest

import ds_limits_world as W
import oracle
from ds_forecast_ref import ds_forecast
from ds_link_world import child_lws_tables, flip_ready, linked_revroles
from lws_b200 import records as R
from test_ds_limits import newest_first, zeroed_revisions

pytestmark = pytest.mark.gpu

TABLES = ("v_sweep", "stamps", "bit31", "rounding", "mixed")


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def _table(name):
    return W.mixed() if name == "mixed" else W.FAMILIES[name]()


def _same(got, want, where):
    for k, name in enumerate(("ds_out", "role_out", "revrole_out")):
        assert got[k].tobytes() == want[k].tobytes(), f"{where}: {name} differs from the oracle"


def _same_owned(got, want, ds, where):
    """As _same, over the role and revision-role rows of the DS inside the format: the rows of a
    BAD_TABLE DS are neither read nor written, so they hold whatever the output buffer held."""
    bad = (want[0]["flags"] & R.DOUT_BAD_TABLE) != 0
    role, rrm = _valid_masks(ds, bad, len(want[1]), len(want[2]))
    assert got[0].tobytes() == want[0].tobytes(), f"{where}: ds_out differs from the oracle"
    assert got[1][role].tobytes() == want[1][role].tobytes(), f"{where}: role_out differs from the oracle"
    assert got[2][rrm].tobytes() == want[2][rrm].tobytes(), f"{where}: revrole_out differs from the oracle"


def _mirrors(res):
    return res["ds_out"], res["role_out"], res["revrole_out"]


def _changed_ds(before, after, ds):
    """The DS a tick lists (the rule of test_gpu_ds_tick.py): its ds_out row, or a role_out or revrole_out
    row of its ranges, differs.  The ranges of a BAD_TABLE DS are not compared."""
    ch = (before[0].view(np.uint8).reshape(len(ds), -1) != after[0].view(np.uint8).reshape(len(ds), -1)).any(1)
    ok = (after[0]["flags"] & R.DOUT_BAD_TABLE) == 0
    n = ds["n_roles"].astype(np.int64)
    for diff, base, count in ((before[1].view(np.uint64) != after[1].view(np.uint64), ds["role_base"], n),
                              (before[2] != after[2], ds["rev_base"], (ds["n_old_revs"].astype(np.int64) + 1) * n)):
        cs = np.concatenate([[0], np.cumsum(diff)])
        b = np.where(ok, base.astype(np.int64), 0)
        ch |= ok & (cs[b + np.where(ok, count, 0)] > cs[b])
    return np.flatnonzero(ch).astype(np.uint32)


def _device_sweep(engine, ds, roles, rr):
    import torch

    up = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()
    d = [up(ds), up(roles), up(rr)]
    o = [torch.zeros(len(ds) * R.DS_OUT.itemsize, dtype=torch.uint8, device="cuda"),
         torch.zeros(len(roles) * R.DS_ROLE_OUT.itemsize, dtype=torch.uint8, device="cuda"),
         torch.zeros(len(rr) * 4, dtype=torch.uint8, device="cuda")]
    torch.cuda.synchronize()
    engine.sweep_ds_device(d[0], len(ds), d[1], len(roles), d[2], len(rr), *o, stream=engine.stream)
    torch.cuda.synchronize()
    return tuple(x.cpu().numpy().view(dt) for x, dt in zip(o, (R.DS_OUT, R.DS_ROLE_OUT, R.DS_REVROLE_OUT)))


def _coverage(ds, roles, rr, out):
    """What the limit tables are for, read from the results: V = 32, drained bit 31, 10 roles with a
    removed one, a drain that is not the last revision row."""
    assert (ds["n_old_revs"] == 32).any()
    assert ((ds["n_roles"] == 10) & (ds["n_spec_roles"] < 10)).any()
    assert ((out[0]["drained_revs"] >> 31) & 1).any() and ((out[0]["ready_revs"] >> 31) & 1).any()
    off_order = 0
    for d in np.flatnonzero((out[0]["flags"] & R.DOUT_STEP) != 0):
        z = zeroed_revisions(ds, rr, out[2], d)
        V = int(ds["n_old_revs"][d])
        off_order += bool(z) and max(z) != V - 1 and z[0] == newest_first(ds, rr, d)[0]
    assert off_order > 0


# --------------------------------------------------------------------------------------------------
# 1. the stateless sweep
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", TABLES)
def test_stateless_sweep_at_the_limits(engine, name):
    ds, roles, rr = _table(name)
    want = oracle.sweep_ds(ds, roles, rr)
    _same(engine.sweep_ds_host(ds, roles, rr), want, f"{name} host")
    _same(_device_sweep(engine, ds, roles, rr), want, f"{name} device")
    if name == "mixed":
        _coverage(ds, roles, rr, want)


# --------------------------------------------------------------------------------------------------
# 2. the resident tick
# --------------------------------------------------------------------------------------------------
def _drain_ds_row(ds, roles, rr, out):
    """A V = 32, n = 10 drain DS (ds_limits_world.drain_ds) that zeroes one revision."""
    for d in np.flatnonzero((ds["n_old_revs"] == 32) & (ds["n_roles"] == 10) & (ds["n_spec_roles"] == 10)):
        if out[0]["flags"][d] & R.DOUT_STEP and roles["target_replicas"][int(ds["role_base"][d])] == 32:
            if len(zeroed_revisions(ds, rr, out[2], d)) == 1:
                return int(d)
    raise AssertionError("no V = 32, n = 10 drain DS in the table")


def test_resident_tick_at_the_limits(engine):
    ds, roles, rr = W.mixed()
    roles, rr = roles.copy(), rr.copy()
    engine.ds_resident_load(ds, roles, rr)
    res = engine.ds_resident_tick()
    prev = oracle.sweep_ds(ds, roles, rr)
    assert res["n_changed"] == len(ds)
    assert np.array_equal(np.sort(res["rows"]), np.arange(len(ds), dtype=np.uint32))
    _same(_mirrors(res), prev, "first tick")
    d = _drain_ds_row(ds, roles, rr, prev)
    vb, rb = int(ds["rev_base"][d]), int(ds["role_base"][d])

    def tick(table, rows, values, what):
        nonlocal prev
        rows = np.asarray(rows, np.uint32)
        (rr if table == R.TABLE_DS_REVROLES else roles)[rows] = values
        got = engine.ds_resident_tick([(table, rows, values)])
        want = oracle.sweep_ds(ds, roles, rr)
        expect = _changed_ds(prev, want, ds)
        assert expect.tolist() == [d], f"{what}: the patch should change DS {d} only, changes {expect[:8]}"
        assert np.sort(got["rows"]).tolist() == [d], what
        _same(_mirrors(got), want, what)
        prev = want

    # the last revision-role row of the DS (the new revision, role 9): not ready, then ready again
    last = np.array([vb + 329])
    v = rr[last].copy()
    v["ready_replicas"] = 0
    keep = rr[last].copy()
    tick(R.TABLE_DS_REVROLES, last, v, "row rev_base + 329")
    tick(R.TABLE_DS_REVROLES, last, keep, "row rev_base + 329 back")
    # revision 31: every row drained, then back
    r31 = np.arange(vb + 310, vb + 320)
    v, keep = rr[r31].copy(), rr[r31].copy()
    v["replicas"] = 0
    tick(R.TABLE_DS_REVROLES, r31, v, "revision 31 drained")
    assert (prev[0]["drained_revs"][d] >> 31) & 1
    tick(R.TABLE_DS_REVROLES, r31, keep, "revision 31 back")
    # a role row: target 64 doubles the steps, and the new revision may scale up again
    one = np.array([rb])
    v, keep = roles[one].copy(), roles[one].copy()
    v["target_replicas"] = 64
    tick(R.TABLE_DS_ROLES, one, v, "role row")
    tick(R.TABLE_DS_ROLES, one, keep, "role row back")
    # a stamp-only patch: another revision becomes the newest, and the drain moves to it
    z0 = zeroed_revisions(ds, rr, prev[2], d)
    assert z0 == [newest_first(ds, rr, d)[0]]
    r1 = (z0[0] + 7) % 32
    rows = np.arange(vb + r1 * 10, vb + r1 * 10 + 10)
    v = rr[rows].copy()
    v["flags"] = (v["flags"] & np.uint32(3)) | np.uint32(W.TS_MAX << R.RR_TS_SHIFT)
    tick(R.TABLE_DS_REVROLES, rows, v, "stamp")
    assert zeroed_revisions(ds, rr, prev[2], d) == [r1]
    m = engine.ds_resident_tick()["revrole_out"]
    assert (m[vb + r1 * 10: vb + r1 * 10 + 10] == 0).all() and (m[vb + z0[0] * 10: vb + z0[0] * 10 + 10] == 1).all()


# --------------------------------------------------------------------------------------------------
# 3. the linked tick
# --------------------------------------------------------------------------------------------------
def _valid_links(links, ds, bad, n_rr):
    """Links of the rows a valid DS reaches (the engine counts only those)."""
    own = np.zeros(n_rr, bool)
    for d in np.flatnonzero(~bad):
        vb = int(ds["rev_base"][d])
        own[vb: vb + (int(ds["n_old_revs"][d]) + 1) * int(ds["n_roles"][d])] = True
    out = links.copy()
    out["lws_row"] = np.where(own, out["lws_row"], R.NONE)
    return out


def test_linked_tick_at_the_limits(engine):
    base = W.mixed(with_rounding=False)
    ds, roles, rr, bad = W.past_limits(*base)
    rng = np.random.default_rng(4)
    lws, groups, pst, pid, links = child_lws_tables(rr, rng)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick(()))
    engine.ds_resident_load(ds, roles, rr)
    res = engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)])
    counted = _valid_links(links, ds, bad, len(rr))
    prev = None
    for k in range(4):
        if k:
            rows, v = flip_ready(groups, rng, 0.02)
            groups[rows] = v
            engine.resident_tick(engine.make_tick([(R.TABLE_GROUPS, rows, v)]))
            res = engine.ds_resident_tick()
        lo = oracle.sweep_lws(lws, groups, pst, pid)[0]
        sub, took, fell = linked_revroles(rr, counted, lws, lo)
        want = oracle.sweep_ds(ds, roles, sub)
        _same_owned(_mirrors(res), want, ds, f"linked tick {k}")
        assert (want[0]["flags"][bad] == R.DOUT_BAD_TABLE).all() and (res["ds_out"]["flags"][bad] == R.DOUT_BAD_TABLE).all()
        info = engine.ds_resident_tick_info()
        assert info["linked"] and (info["rows_from_lws"], info["rows_fallback"]) == (took, fell), k
        if k == 0:
            assert took == int(((counted["lws_row"] != R.NONE) & ((rr["flags"] & R.RR_EXISTS) != 0)).sum()) and fell == 0
            assert len(res["rows"]) == len(ds)
        else:
            assert np.array_equal(np.sort(res["rows"]), _changed_ds(prev, want, ds)), k
        prev = want
    _coverage(ds[~bad], roles, sub, oracle.sweep_ds(ds[~bad], roles, sub))


# --------------------------------------------------------------------------------------------------
# 4. the forecast
# --------------------------------------------------------------------------------------------------
def _same_forecast(got, want, where):
    assert got["ds"].tobytes() == want["ds"].tobytes(), f"{where}: per-DS forecast differs"
    assert got["roles"].tobytes() == want["roles"].tobytes(), f"{where}: per-role forecast differs"
    assert (got["n_steps_needed"], got["n_steps_written"]) == (want["n_steps_needed"], want["n_steps_written"]), where
    assert got["steps"].tobytes() == want["steps"].tobytes(), f"{where}: trajectory rows differ"


@pytest.mark.parametrize("name", ["v_sweep", "stamps", "bit31"])
def test_forecast_at_the_limits(engine, name):
    ds, roles, rr = _table(name)
    want = ds_forecast(ds, roles, rr)
    _same_forecast(engine.ds_forecast_host(ds, roles, rr), want, f"{name} host")
    engine.ds_resident_load(ds, roles, rr)
    engine.ds_resident_tick()
    _same_forecast(engine.ds_resident_forecast(), want, f"{name} resident")
    fl = want["ds"]["flags"]
    assert (fl & R.DSF_DONE).any() and (want["ds"]["n_steps"][ds["n_old_revs"] == 32] > 0).any()


def test_forecast_stops_at_the_cycle_cap(engine):
    """One DS of two roles moving 40 000 replicas one at a time needs about 80 000 cycles: the replay
    stops at LWSE_DS_FORECAST_MAX_CYCLES and reports UNFINISHED; a small DS beside it finishes."""
    rng = np.random.default_rng(1)
    x = W._empty(2, 0, 1)
    x.roles["target_replicas"] = 40_000
    for i in range(2):
        W._put(x, 0, i, 40_000, 40_000, 40_000, stamp=1)
        W._put(x, 1, i, 0, -1, 0, stamp=2)
    ds, roles, rr = W.assemble([x, W.drain_ds(rng, 3, 5, "perm")])
    want = ds_forecast(ds, roles, rr)
    got = engine.ds_forecast_host(ds, roles, rr)
    _same_forecast(got, want, "cycle cap")
    assert got["ds"]["flags"][0] & R.DSF_UNFINISHED and got["ds"]["cycles"][0] == R.DS_FORECAST_MAX_CYCLES
    assert got["ds"]["flags"][1] & R.DSF_DONE


# --------------------------------------------------------------------------------------------------
# 5. just past the limits
# --------------------------------------------------------------------------------------------------
def _valid_masks(ds, bad, n_roles, n_rr):
    role, rrm = np.zeros(n_roles, bool), np.zeros(n_rr, bool)
    for d in np.flatnonzero(~bad):
        rb, n, vb = int(ds["role_base"][d]), int(ds["n_roles"][d]), int(ds["rev_base"][d])
        role[rb: rb + n] = True
        rrm[vb: vb + (int(ds["n_old_revs"][d]) + 1) * n] = True
    return role, rrm


def _same_valid(with_bad, without, ds, bad, where):
    """The DS of the format: the same rows in a run with the rows past it and in one without them."""
    role, rrm = _valid_masks(ds, bad, len(with_bad[1]), len(with_bad[2]))
    assert with_bad[0][~bad].tobytes() == without[0].tobytes(), f"{where}: ds_out"
    assert with_bad[1][role].tobytes() == without[1][role].tobytes(), f"{where}: role_out"
    assert with_bad[2][rrm].tobytes() == without[2][rrm].tobytes(), f"{where}: revrole_out"
    bd = with_bad[0][bad]
    assert (bd["flags"] == R.DOUT_BAD_TABLE).all() and not bd["drained_revs"].any() and not bd["ready_revs"].any(), where


def test_rows_past_the_limits_are_bad_table_on_every_path(engine):
    ds, roles, rr, bad = W.past_limits(*W.mixed(copies=1, with_rounding=False))
    h = ds[bad]
    assert (h["n_old_revs"] == 33).any() and ((h["n_roles"] == 11) & (h["n_spec_roles"] == 10)).any()
    assert (h["n_spec_roles"] > h["n_roles"]).any()
    end = ds["rev_base"].astype(np.int64) + (ds["n_old_revs"].astype(np.int64) + 1) * ds["n_roles"]
    assert (end[bad] == len(rr) + 1).any() and (end[~bad] == len(rr)).any()
    good = ds[~bad].copy()
    want = oracle.sweep_ds(ds, roles, rr)
    _same_valid(want, oracle.sweep_ds(good, roles, rr), ds, bad, "oracle")
    # the stateless sweep, host and device
    got = engine.sweep_ds_host(ds, roles, rr)
    _same_owned(got, want, ds, "host")
    _same_valid(got, engine.sweep_ds_host(good, roles, rr), ds, bad, "host")
    dev = _device_sweep(engine, ds, roles, rr)
    _same_owned(dev, want, ds, "device")
    _same_valid(dev, _device_sweep(engine, good, roles, rr), ds, bad, "device")
    # the resident tick: the first tick's mirrors
    engine.ds_resident_load(good, roles, rr)
    alone = tuple(x.copy() for x in _mirrors(engine.ds_resident_tick()))
    engine.ds_resident_load(ds, roles, rr)
    res = engine.ds_resident_tick()
    assert res["n_changed"] == len(ds)
    _same_owned(_mirrors(res), want, ds, "tick")
    _same_valid(_mirrors(res), alone, ds, bad, "tick")
    # the forecast, host and resident (the last load: the table with the rows past the format)
    fw = ds_forecast(ds, roles, rr)
    fg = engine.ds_forecast_host(ds, roles, rr)
    _same_forecast(fg, fw, "forecast")
    assert (fg["ds"]["flags"][bad] == R.DSF_BAD_TABLE).all()
    _same_forecast(engine.ds_resident_forecast(), fw, "resident forecast")
    fa = engine.ds_forecast_host(good, roles, rr)
    role, _ = _valid_masks(ds, bad, len(roles), len(rr))
    assert fg["ds"][~bad].tobytes() == fa["ds"].tobytes()
    assert fg["roles"][role].tobytes() == fa["roles"][role].tobytes() and not fg["roles"][~role].view(np.uint8).any()
    assert fg["steps"].tobytes() == fa["steps"].tobytes()
