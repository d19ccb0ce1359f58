"""The DS rollout what-if on the device (lwse_resident_ds_rollout_whatif) against the CPU reference of
tests/ds_rollout_whatif_ref.py, byte for byte (now, now_roles, the forecast rows and the trajectory): fuzzed and
limit tables with mixed flags, duplicate and BAD rows; identity proposals at C4 against the DS tick and the resident
forecast; a template bump of every DS at C4 and a grid of 16 settings x 1 000 DS; linked, unlinked and unswept
engines; the warp, CTA and scan-block sizes, truncated trajectories and every refusal; and isolation from the ticks."""
import ctypes as C
import functools

import numpy as np
import pytest

from ds_drain_ref import ds_drain_world
from ds_limits_world import mixed, past_limits
from ds_rollout_whatif_ref import M, ds_rollout_whatif
from lws_b200 import engine as E
from lws_b200 import records as R
from lws_b200 import synth
from test_gpu_ds_drain import load, resident_tables
from test_gpu_node_events import Arena

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def world(name):
    if name == "C4":
        return ds_drain_world(n_ds=50_000, n_nodes=2048, seed=23, nodes_per_domain=16, roles=(2,))
    return ds_drain_world(n_ds=300, n_nodes=48, seed=31)


def _same(got, want, where=""):
    for k in ("now", "now_roles", "ds", "roles"):
        assert got[k].tobytes() == want[k].tobytes(), f"{where}: {k} differs"
    assert got["n_steps_needed"] == want["n_steps_needed"] and got["n_steps_written"] == want["n_steps_written"], where
    if want["steps"] is None:
        assert got["steps"] is None
    else:
        assert got["steps"].tobytes() == want["steps"].tobytes(), f"{where}: trajectory rows differ"


def random_proposals(ds, roles, n, seed):
    """n proposals on random DS rows (several per row): flags 0, NEW_REVISION, ROLES with new targets and rollout
    settings (integer and percent, invalid intstr), and both."""
    rng = np.random.default_rng(seed)
    props = np.zeros(n, R.DS_PROPOSAL)
    props["ds"] = rng.integers(0, len(ds), n)
    props["flags"] = rng.integers(0, 4, n)
    q = R.aligned_empty(n * M, R.DS_ROLE_REC)
    q["target_replicas"] = rng.integers(0, 12, n * M)
    q["max_surge"] = rng.integers(0, 4, n * M)
    q["max_unavailable"] = rng.integers(0, 3, n * M)
    q["flags"] = (rng.integers(0, 64, n * M) | R.ROLE_IN_SPEC).astype(np.uint32)
    # the spec / removed split of the resident rows stays
    for i in np.flatnonzero(props["flags"] & R.DSP_ROLES):
        d = ds[props["ds"][i]]
        nr, S = min(int(d["n_roles"]), M), min(int(d["n_spec_roles"]), M)
        q["flags"][i * M + S: i * M + nr] &= ~np.uint32(R.ROLE_IN_SPEC)
    return props, q


def _tables(seed):
    if seed == 0:  # the table limits: V up to 32, 10 roles with removed ones, rows past the limits
        return past_limits(*mixed(seed=5, copies=1, with_rounding=False))[:3]
    t = synth.make_ds(400, n_roles_choices=(2, 3, 10), max_old_revs=33 if seed == 2 else 3, seed=seed, fuzz=0.2)
    t.ds["n_spec_roles"][::97] = t.ds["n_roles"][::97] + 1  # past the limits
    return t.ds, t.roles, t.revroles


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fuzzed_tables_equal_reference(engine, seed):
    ds0, roles, rr = _tables(seed)
    ds = R.aligned_empty(len(ds0) + 2, R.DS_REC)  # two vacant (zeroed) rows at the end
    ds[: len(ds0)] = ds0
    engine.ds_resident_load(ds, roles, rr)
    engine.ds_resident_tick([])
    props, q = random_proposals(ds, roles, 3000, seed)
    want = ds_rollout_whatif(ds, roles, rr, None, props, q)
    assert want["bad"].any() and not want["bad"].all()
    assert (want["ds"]["flags"] & R.DSF_DONE).any() and (want["now"]["flags"] & R.DOUT_INIT).any()
    _same(engine.resident_ds_rollout_whatif(props, q), want, f"seed {seed}")
    summ = engine.resident_ds_rollout_whatif(props, q, steps=False)
    assert summ["ds"].tobytes() == want["ds"].tobytes() and summ["steps"] is None


def test_old_revision_limit(engine):
    """V = 31 becomes 32 after a bump (valid, ready_revs bit 31 for the retired revision); V = 32 becomes BAD."""
    from ds_limits_world import _empty, _put, assemble

    items = []
    for V in (31, 32):
        x = _empty(2, 1, V)
        for r in range(V + 1):
            for i in range(3):
                _put(x, r, i, 2 if r == V and i < 2 else 0, stamp=r + 1)
        items.append(x)
    ds, roles, rr = assemble(items)
    engine.ds_resident_load(ds, roles, rr)
    engine.ds_resident_tick([])
    props = np.zeros(4, R.DS_PROPOSAL)
    props["ds"] = [0, 0, 1, 1]
    props["flags"] = [0, R.DSP_NEW_REVISION] * 2
    want = ds_rollout_whatif(ds, roles, rr, None, props)
    assert want["bad"].tolist() == [False, False, False, True]
    assert int(want["now"][1]["ready_revs"]) >> 31 == 1
    _same(engine.resident_ds_rollout_whatif(props), want, "limits")


def test_identity_is_the_tick(engine):
    """Flags 0 for every DS at C4 after an LWS tick and a linked DS tick: `now` is the DS tick's output, the forecast
    the resident forecast's rows, re-strided."""
    w = world("C4")
    tick = load(engine, w)
    props = np.zeros(len(w.ds), R.DS_PROPOSAL)
    props["ds"] = np.arange(len(w.ds))
    got = engine.resident_ds_rollout_whatif(props)
    fc = engine.ds_resident_forecast()
    assert got["now"].tobytes() == tick["ds_out"].tobytes()
    ok = (tick["ds_out"]["flags"] & R.DOUT_BAD_TABLE) == 0
    n = w.ds["n_roles"].astype(np.int64)
    for d in np.flatnonzero(ok):
        rb, k = int(w.ds["role_base"][d]), int(n[d])
        assert got["now_roles"][d * M: d * M + k].tobytes() == tick["role_out"][rb: rb + k].tobytes(), d
        assert got["roles"][d * M: d * M + k].tobytes() == fc["roles"][rb: rb + k].tobytes(), d
    assert got["ds"].tobytes() == fc["ds"].tobytes()
    assert got["steps"].tobytes() == fc["steps"].tobytes() and got["n_steps_needed"] == fc["n_steps_needed"]


def _linked_ref(w, props, q=None, lws_results=True, **kw):
    return ds_rollout_whatif(w.ds, w.roles, w.revroles, w.links, props, q, lws=w.lws if lws_results else None,
                             lws_out=w.base[0] if lws_results else None, **kw)


def test_fleet_template_bump(engine):
    """A new template for every DS at C4 (50 000 proposals) on the linked world."""
    w = world("C4")
    load(engine, w)
    props = np.zeros(len(w.ds), R.DS_PROPOSAL)
    props["ds"] = np.arange(len(w.ds))
    props["flags"] = R.DSP_NEW_REVISION
    want = _linked_ref(w, props)
    assert (want["ds"]["flags"] & R.DSF_DONE).sum() > len(w.ds) // 2
    _same(engine.resident_ds_rollout_whatif(props), want, "C4 bump")


def test_settings_grid(engine):
    """16 rollout settings x 1 000 DS: maxSurge {0, 1, 2, 25%} x maxUnavailable {0, 1, 2, 50%}, with a template
    edit, on the first 1 000 DS of C4."""
    w = world("C4")
    load(engine, w)
    grid = [(s, u) for s in (0, 1, 2, 25) for u in (0, 1, 2, 50)]
    n_ds = 1000
    props = np.zeros(len(grid) * n_ds, R.DS_PROPOSAL)
    props["ds"] = np.tile(np.arange(n_ds), len(grid))
    props["flags"] = R.DSP_NEW_REVISION | R.DSP_ROLES
    q = R.aligned_empty(len(props) * M, R.DS_ROLE_REC)
    for g, (s, u) in enumerate(grid):
        for d in range(n_ds):
            i, rb, nr = g * n_ds + d, int(w.ds["role_base"][d]), min(int(w.ds["n_roles"][d]), M)
            rows = w.roles[rb: rb + nr].copy()
            spec = (rows["flags"] & R.ROLE_IN_SPEC) != 0
            rows["max_surge"] = np.where(spec, s, rows["max_surge"])
            rows["max_unavailable"] = np.where(spec, u, rows["max_unavailable"])
            pct = (R.ROLE_SURGE_IS_PERCENT if s == 25 else 0) | (R.ROLE_UNAVAIL_IS_PERCENT if u == 50 else 0)
            keep = rows["flags"] & ~np.uint32(R.ROLE_SURGE_IS_PERCENT | R.ROLE_UNAVAIL_IS_PERCENT | R.ROLE_SURGE_INVALID
                                               | R.ROLE_UNAVAIL_INVALID)
            rows["flags"] = np.where(spec, keep | R.ROLE_HAS_ROLLING_CONFIG | pct, rows["flags"])
            q[i * M: i * M + nr] = rows
    want = _linked_ref(w, props, q)
    _same(engine.resident_ds_rollout_whatif(props, q), want, "grid")
    cyc = want["ds"]["cycles"].reshape(len(grid), n_ds).astype(np.int64).sum(axis=1)
    assert len(set(cyc.tolist())) > 4  # the settings make different rollouts


def test_links():
    """A linked world whose LWS ready counts differ from the revision-role rows: `now` follows the LWS values
    (the retired revision's rows too); an unlinked engine and one whose LWS rows are not swept use the rows' own."""
    w = world("small")
    props, q = random_proposals(w.ds, w.roles, 2000, 7)
    for mode in ("linked", "unlinked", "unswept"):
        e = E.Engine(0)
        try:
            e.upload_nodes(w.nodes, w.n_domains)
            e.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
            if mode != "unswept":
                e.resident_tick(e.make_tick((), w.flags))
            e.ds_resident_load(w.ds, w.roles, w.revroles)
            e.ds_resident_tick([] if mode == "unlinked" else [(R.TABLE_DS_LINKS, 0, w.links, True)])
            want = _linked_ref(w, props, q, lws_results=mode == "linked")
            _same(e.resident_ds_rollout_whatif(props, q), want, mode)
            if mode == "linked":
                own = _linked_ref(w, props, q, lws_results=False)
                assert own["now"].tobytes() != want["now"].tobytes()
                assert own["ds"].tobytes() == want["ds"].tobytes()  # the forecast ignores links
        finally:
            e.close()


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025])
def test_sizes(engine, n):
    w = world("small")
    load(engine, w)
    props, q = random_proposals(w.ds, w.roles, n, 100 + n)
    got = engine.resident_ds_rollout_whatif(props, q)
    if n == 0:
        assert len(got["now"]) == 0 and got["n_steps_needed"] == 0 and got["n_steps_written"] == 0
        return
    _same(got, _linked_ref(w, props, q), f"n={n}")


def test_truncated(engine):
    w = world("small")
    load(engine, w)
    props, q = random_proposals(w.ds, w.roles, 1500, 9)
    need = _linked_ref(w, props, q)["n_steps_needed"]
    assert need > 10
    for cap in (0, 1, need // 2, need - 1, need):
        _same(engine.resident_ds_rollout_whatif(props, q, step_capacity=cap), _linked_ref(w, props, q, step_capacity=cap),
              f"capacity {cap}")
    _same(engine.resident_ds_rollout_whatif(props, q, steps=False), _linked_ref(w, props, q, steps=False), "no steps")


def _raw(e, props=None, n=0, roles=None, now=None, fc_ds=None, fc_roles=None, reserved=0, now_roles=None):
    o = R.DsForecastOut(fc_ds, fc_roles, None, 0, 0, 0)
    q = R.DsRolloutWhatIf(props, roles, n, reserved, now, now_roles, o)
    return E.lib().lwse_resident_ds_rollout_whatif(e._h, C.byref(q))


def test_refusals_write_nothing():
    w = world("small")
    e = E.Engine(0)
    try:
        props = np.zeros(4, R.DS_PROPOSAL)
        props["ds"] = [0, 1, 2, 3]
        q = R.aligned_empty(4 * M + 1, R.DS_ROLE_REC)
        now, now_roles = R.aligned_empty(4, R.DS_OUT), R.aligned_empty(4 * M, R.DS_ROLE_OUT)
        fc, fr = R.aligned_empty(4, R.DS_FORECAST), R.aligned_empty(4 * M, R.DS_FORECAST_ROLE)
        outs = (now, now_roles, fc, fr)
        for a in outs:
            a.view(np.uint8)[:] = 0xA5
        p = dict(props=R.ptr(props), n=4, roles=R.ptr(q), now=R.ptr(now), now_roles=R.ptr(now_roles),
                 fc_ds=R.ptr(fc), fc_roles=R.ptr(fr))
        assert _raw(e, **p) == ERR_NOT_READY
        assert E.lib().lwse_resident_ds_rollout_whatif(e._h, None) == ERR_INVALID_ARG
        e.ds_resident_load(w.ds, w.roles, w.revroles)
        assert E.lib().lwse_resident_ds_rollout_whatif(e._h, None) == ERR_INVALID_ARG
        for k in ("props", "now", "fc_ds", "fc_roles"):
            assert _raw(e, **dict(p, **{k: None})) == ERR_INVALID_ARG, k
        assert _raw(e, **dict(p, reserved=1)) == ERR_INVALID_ARG
        for field, v in (("ds", len(w.ds)), ("flags", 4), ("flags", 1 << 31)):
            bad = props.copy()
            bad[field][2] = v
            assert _raw(e, **dict(p, props=R.ptr(bad))) == ERR_INVALID_ARG, (field, v)
        roles_props = props.copy()
        roles_props["flags"][1] = R.DSP_ROLES
        assert _raw(e, **dict(p, props=R.ptr(roles_props), roles=None)) == ERR_INVALID_ARG
        assert _raw(e, **dict(p, props=R.ptr(roles_props), roles=R.ptr(q) + 8)) == ERR_INVALID_ARG
        # n past the cap, with small arrays: refused before any array is read
        assert _raw(e, **dict(p, n=R.DS_WHATIF_MAX_PROPOSALS + 1)) == ERR_UNSUPPORTED
        assert _raw(e, **dict(p, n=0xFFFFFFFF)) == ERR_UNSUPPORTED
        for a in outs:
            assert (a.view(np.uint8) == 0xA5).all()
        # without ROLES proposals `roles` is not read; now_roles may be NULL
        assert _raw(e, **dict(p, roles=None, now_roles=None)) == 0
        want = ds_rollout_whatif(w.ds, w.roles, w.revroles, None, props, steps=False)
        assert now.tobytes() == want["now"].tobytes() and fc.tobytes() == want["ds"].tobytes()
        assert (now_roles.view(np.uint8) == 0xA5).all()
        assert _raw(e, n=0) == 0
    finally:
        e.close()


def test_isolation(engine):
    """What-ifs between the submit and wait of LWS ticks in flight and before each DS tick: every LWS tick's change
    lists, every DS tick's rows, outputs and tick info and the DS forecast equal a run without them, and every
    resident table and the link table read back are unchanged."""
    w = world("small")
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(5):
        rows = np.sort(rng.choice(len(w.groups), size=100, replace=False)).astype(np.uint32)
        v = w.groups[rows].copy()
        v["flags"] ^= np.uint32(R.GRP_POD_READY)
        sets.append([(R.TABLE_GROUPS, rows, v)])
    props, q = random_proposals(w.ds, w.roles, 700, 13)

    def snap(r):
        return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()}

    def run(with_whatif):
        first = snap(load(engine, w))
        first["info"] = engine.ds_resident_tick_info()
        arena = Arena(engine)
        lws_out, ds_out = [], [first]
        for k, segs in enumerate(sets):
            engine.resident_tick_submit(engine.make_tick(arena.put(segs, k & 1), w.flags))
            if with_whatif:
                engine.resident_ds_rollout_whatif(props, q)
            lws_out.append(snap(engine.resident_tick_wait()))
            if with_whatif:
                engine.resident_ds_rollout_whatif(props, q, steps=False)
            ds_out.append(snap(engine.ds_resident_tick([])))
            ds_out[-1]["info"] = engine.ds_resident_tick_info()
        return lws_out, ds_out, [x.copy() for x in engine.resident_outputs()], engine.ds_resident_forecast()

    a = run(True)
    tables = resident_tables(engine, w)
    b = run(False)
    assert resident_tables(engine, w) == tables
    before = resident_tables(engine, w)
    engine.resident_ds_rollout_whatif(props, q)
    assert resident_tables(engine, w) == before
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
    assert all(a[3][k].tobytes() == b[3][k].tobytes() for k in ("ds", "roles", "steps"))
    # the last what-if of the run saw the last LWS tick: it equals the reference over that tick's results
    got = engine.resident_ds_rollout_whatif(props, q)
    lws_out = engine.resident_outputs()[0]
    _same(got, ds_rollout_whatif(w.ds, w.roles, w.revroles, w.links, props, q, lws=w.lws, lws_out=lws_out), "after")
