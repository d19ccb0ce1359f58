"""The rollout what-if on the device (lwse_resident_rollout_whatif) against the CPU reference of
tests/rollout_whatif_ref.py, byte for byte: fuzzed proposals on fuzzed worlds, identity proposals against
the resident sweep and forecast at C3 and C5, a fleet template bump at C5, the table, slot and argument
edges, and what-ifs between pipelined ticks, which must change no tick."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import churn, synth
from lws_b200 import records as R
from rollout_whatif_ref import foreign_owners, layers, replaced, rollout_whatif
from test_gpu_lws_forecast import _resident_world, _tick_lists

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def _same(got, want, where=""):
    assert got["now"].tobytes() == want["now"].tobytes(), f"{where}: now differs"
    assert got["lws"].tobytes() == want["lws"].tobytes(), f"{where}: per-proposal forecast differs"
    assert got["n_steps_needed"] == want["n_steps_needed"] and got["n_steps_written"] == want["n_steps_written"], where
    if want["steps"] is None:
        assert got["steps"] is None
    else:
        assert got["steps"].tobytes() == want["steps"].tobytes(), f"{where}: trajectory rows differ"


def _load(engine, t):
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_sweep(t.flags)


def proposals(lws, n, seed):
    """n proposals on random rows (several per row): template edits, replicas up and down, spec partitions,
    integer and percent surge / unavailable (percentages past 100), INTSTR_INVALID, IRREGULAR, size and
    restart-policy changes, and identity proposals.  maxUnavailable stays >= 0 (the webhook rejects a
    negative one, and the C oracle's partition walk assumes it)."""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, len(lws), n).astype(np.uint32)
    recs = R.aligned_empty(n, R.LWS_REC)
    recs[:] = lws[rows]
    kind = rng.integers(0, 8, n)
    tmpl = (kind == 0) | (kind == 1)
    recs["rev_hash"][tmpl] = rng.integers(1, 2**63, int(tmpl.sum()), dtype=np.uint64)
    recs["flags"][tmpl] |= np.uint32(R.LWS_UPDATED)
    sc = kind == 2
    recs["replicas"][sc] = np.maximum(recs["replicas"][sc] + rng.integers(-4, 6, int(sc.sum())), 0)
    pt = kind == 3
    recs["partition"][pt] = rng.integers(0, 8, int(pt.sum()))
    st = kind == 4
    pct_s, pct_u = rng.random(n) < 0.5, rng.random(n) < 0.5
    recs["max_surge"][st] = np.where(pct_s, rng.integers(0, 160, n), rng.integers(0, 5, n))[st]
    recs["max_unavailable"][st] = np.where(pct_u, rng.integers(0, 160, n), rng.integers(0, 5, n))[st]
    f = recs["flags"]
    f[st] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT | R.LWS_UNAVAIL_IS_PERCENT)
    f[st] |= (np.where(pct_s, R.LWS_SURGE_IS_PERCENT, 0) | np.where(pct_u, R.LWS_UNAVAIL_IS_PERCENT, 0)).astype(np.uint32)[st]
    odd = kind == 5
    f[odd] ^= np.where(rng.random(n) < 0.5, R.LWS_INTSTR_INVALID, R.LWS_IRREGULAR).astype(np.uint32)[odd]
    sz = kind == 6
    recs["size"][sz] = rng.choice([1, 2, 3, 8], int(sz.sum()))
    f[sz] = (f[sz] & ~np.uint32(R.LWS_RESTART_MASK)) | (rng.integers(0, 3, int(sz.sum())) << R.LWS_RESTART_SHIFT).astype(np.uint32)
    recs["flags"] = f
    # kind 7: identity; and every proposal's own range is ignored
    recs["group_base"] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    recs["group_count"] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    return rows, recs


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzzed_proposals_equal_reference(engine, seed):
    t = synth.make(synth.profile("fuzz", 0.5), seed=seed)
    _load(engine, t)
    rows, recs = proposals(t.lws, 3000, seed)
    want = rollout_whatif(t, rows, recs)
    _same(engine.resident_rollout_whatif(rows, recs), want, f"fuzz {seed}")
    summ = engine.resident_rollout_whatif(rows, recs, steps=False)
    assert summ["lws"].tobytes() == want["lws"].tobytes() and summ["now"].tobytes() == want["now"].tobytes()
    f = want["lws"]["flags"]
    for bit in (R.LWSF_ROLLING, R.LWSF_WAITING, R.LWSF_DONE, R.LWSF_NOT_FORECAST):
        assert (f & bit).any(), bit
    assert len(np.unique(rows)) < len(rows)  # several proposals per row


def test_truncated_trajectories(engine):
    t = synth.make(synth.profile("fuzz", 0.5), seed=4)
    _load(engine, t)
    rows, recs = proposals(t.lws, 1500, 4)
    need = rollout_whatif(t, rows, recs)["n_steps_needed"]
    for cap in (0, 1, need // 2, need - 1, need):
        want = rollout_whatif(t, rows, recs, step_capacity=cap)
        _same(engine.resident_rollout_whatif(rows, recs, step_capacity=cap), want, f"capacity {cap}")


@pytest.mark.parametrize("name", ["C3", "C5"])
def test_identity_is_the_baseline(engine, name):
    t = synth.make(name)
    _load(engine, t)
    rows = np.arange(len(t.lws), dtype=np.uint32)
    got = engine.resident_rollout_whatif(rows, t.lws)
    lo, _ = engine.resident_outputs()
    assert got["now"].tobytes() == lo.tobytes()
    base = engine.resident_forecast()
    assert got["lws"].tobytes() == base["lws"].tobytes()
    assert got["steps"].tobytes() == base["steps"].tobytes()
    assert got["n_steps_needed"] == base["n_steps_needed"] > 0


def test_fleet_template_bump_c5(engine):
    t = synth.make("C5")
    _load(engine, t)
    rows = np.arange(len(t.lws), dtype=np.uint32)
    recs = t.lws.copy()
    recs["rev_hash"] ^= np.uint64(0x5DEECE66D)
    recs["flags"] |= np.uint32(R.LWS_UPDATED)
    want = rollout_whatif(t, rows, recs)
    _same(engine.resident_rollout_whatif(rows, recs), want, "fleet")
    _same(engine.resident_rollout_whatif(rows, recs, steps=False), dict(want, steps=None, n_steps_written=0),
          "fleet, summaries")
    assert (want["lws"]["n_steps"] > 0).sum() > len(rows) // 2


def edge_world():
    """A fuzz world with an object whose range also holds the first rows of the next object (foreign-owned
    rows), one whose range ends past the group table, and proposals on both, on their neighbours, and one
    with more slots than LWSE_LWS_FORECAST_MAX_SLOTS."""
    t = synth.make(synth.profile("fuzz", 0.3), seed=9)
    lws = t.lws
    end = lws["group_base"].astype(np.int64) + lws["group_count"]
    a = next(i for i in range(len(lws) - 1) if end[i] == lws["group_base"][i + 1] and lws["group_count"][i + 1] >= 2
             and lws["group_count"][i] >= 1)
    lws["group_count"][a] += 2
    b = len(lws) - 1 if a != len(lws) - 1 else 0
    lws["group_base"][b] = len(t.groups) - 1
    lws["group_count"][b] = 5
    rows = np.array([a, a, a + 1, b, b, 0], np.uint32)
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = lws[rows]
    recs["rev_hash"][[0, 2, 3]] ^= np.uint64(77)
    recs["flags"][[0, 2, 3]] |= np.uint32(R.LWS_UPDATED)
    recs["replicas"][1] += 2
    recs["replicas"][5] = R.LWS_FORECAST_MAX_SLOTS + 1
    return t, rows, recs


def test_edges(engine):
    """Against the definition itself: the engine's own sweep of the resident tables with one row replaced,
    and its forecast of that row.  (The C oracle's updateConditions judges a group row in a range against
    the range's object, the engine's group pass against the row's owner; the two agree unless a range holds
    another object's rows, which is this world's point.)"""
    t, rows, recs = edge_world()
    _load(engine, t)
    got = engine.resident_rollout_whatif(rows, recs)
    assert got["now"]["flags"][3] & R.LOUT_BAD_TABLE and got["lws"]["flags"][3] == R.LWSF_BAD_TABLE
    assert got["lws"]["flags"][5] == R.LWSF_NOT_FORECAST
    a = int(rows[0])
    own = t.groups["lws_index"][int(t.lws["group_base"][a]): int(t.lws["group_base"][a] + t.lws["group_count"][a])]
    assert (own != a).sum() == 2
    for i in range(len(rows)):
        lws = replaced(t.lws, rows, recs, [i])
        lo, go = engine.sweep_lws_host(lws, t.groups, t.pod_state, t.pod_ident, flags=t.flags)[:2]
        r = int(rows[i])
        assert got["now"][i].tobytes() == lo[r].tobytes(), i
        f = engine.lws_forecast(lws[r: r + 1], go)
        assert got["lws"][i]["step_base"] == got["lws"]["n_steps"][:i].sum()
        want = f["lws"].copy()
        want["step_base"] = got["lws"][i]["step_base"]
        assert got["lws"][i: i + 1].tobytes() == want.tobytes(), i
        b, k = int(got["lws"][i]["step_base"]), int(got["lws"][i]["n_steps"])
        assert got["steps"][b: b + k].tobytes() == f["steps"].tobytes(), i
    # the reference sweeps proposal 2, on the owner of the foreign rows in proposal 0's range, apart from it
    lay = layers(rows, foreign_owners(t.lws, t.groups, rows))
    assert not any(0 in idx and 2 in idx for idx in lay)


def _raw(engine, rows, recs, now, fc, n=None, steps=None, cap=0):
    q = R.RolloutWhatIf(rows, recs, len(fc) if n is None else n, 0, now,
                        R.LwsForecastOut(R.ptr(fc) if fc is not None else None, steps, cap, 0, 0))
    from lws_b200.engine import lib

    return lib().lwse_resident_rollout_whatif(engine._h, C.byref(q)), q


def test_arguments(engine):
    from lws_b200.engine import LwseError

    t = synth.make(synth.profile("fuzz", 0.2), seed=5)
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    with pytest.raises(LwseError) as e:  # loaded, not swept
        engine.resident_rollout_whatif([0], t.lws[:1])
    assert e.value.status == ERR_NOT_READY
    engine.resident_sweep(t.flags)
    empty = engine.resident_rollout_whatif(np.zeros(0, np.uint32), t.lws[:0])
    assert len(empty["now"]) == 0 and empty["n_steps_needed"] == 0 and len(empty["steps"]) == 0
    rows = np.array([0, 1], np.uint32)
    recs = R.aligned_empty(2, R.LWS_REC)
    recs[:] = t.lws[:2]
    now, fc = R.aligned_empty(2, R.LWS_OUT), R.aligned_empty(2, R.LWS_FORECAST)
    assert _raw(engine, R.ptr(rows), R.ptr(recs), R.ptr(now), fc)[0] == 0
    assert _raw(engine, None, R.ptr(recs), R.ptr(now), fc)[0] == ERR_INVALID_ARG
    assert _raw(engine, R.ptr(rows), None, R.ptr(now), fc)[0] == ERR_INVALID_ARG
    assert _raw(engine, R.ptr(rows), R.ptr(recs), None, fc)[0] == ERR_INVALID_ARG
    assert _raw(engine, R.ptr(rows), R.ptr(recs), R.ptr(now), None, n=2)[0] == ERR_INVALID_ARG
    raw = np.zeros(2 * 64 + 32, np.uint8)
    mis = raw[(-raw.ctypes.data) % 16 + 8:][: 2 * 64]
    mis[:] = recs.view(np.uint8)
    assert _raw(engine, R.ptr(rows), mis.ctypes.data, R.ptr(now), fc)[0] == ERR_INVALID_ARG
    bad = np.array([0, len(t.lws)], np.uint32)
    assert _raw(engine, R.ptr(bad), R.ptr(recs), R.ptr(now), fc)[0] == ERR_INVALID_ARG
    # a pod patch without a sweep: the group results no longer belong to the rows
    engine.resident_tick(engine.make_tick([(R.TABLE_POD_STATE, np.array([0], np.uint32), t.pod_state[:1].copy())],
                                          t.flags | R.TICK_NO_SWEEP))
    with pytest.raises(LwseError) as e:
        engine.resident_rollout_whatif(rows, recs)
    assert e.value.status == ERR_NOT_READY
    engine.resident_sweep(t.flags)
    _same(engine.resident_rollout_whatif(rows, recs), rollout_whatif(t, rows, recs), "after the sweep")


def test_slot_sum_2gib_refused(engine):
    """2048 proposals of 2^20 slots each: a slot sum of exactly 2^31 is refused, writes nothing, and the
    next call is right."""
    t = synth.make(synth.profile("fuzz", 0.2), seed=6)
    _load(engine, t)
    n = 2048
    rows = np.zeros(n, np.uint32)
    recs = R.aligned_empty(n, R.LWS_REC)
    recs[:] = t.lws[0]
    recs["replicas"] = R.LWS_FORECAST_MAX_SLOTS
    recs["max_surge"] = 0
    recs["flags"] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT)
    now, fc = R.aligned_empty(n, R.LWS_OUT), R.aligned_empty(n, R.LWS_FORECAST)
    now.view(np.uint8)[:] = 0xA5
    fc.view(np.uint8)[:] = 0xA5
    rc, q = _raw(engine, R.ptr(rows), R.ptr(recs), R.ptr(now), fc)
    assert rc == ERR_UNSUPPORTED
    assert (now.view(np.uint8) == 0xA5).all() and (fc.view(np.uint8) == 0xA5).all()
    assert q.fc.n_steps_written == 0 and q.fc.n_steps_needed == 0
    rows2, recs2 = proposals(t.lws, 200, 6)
    _same(engine.resident_rollout_whatif(rows2, recs2), rollout_whatif(t, rows2, recs2), "after the refusal")


def test_gathered_rows_4gib_refused(engine):
    """Proposals whose gathered group rows reach 2^32 (4096 proposals of a 2^20-group object) are refused
    before the gathered table is allocated; the next call is right."""
    from lws_b200.engine import LwseError

    ng = 1 << 20
    lws = R.aligned_empty(2, R.LWS_REC)
    lws["replicas"] = lws["sts_replicas"] = lws["sts_replicas_annotation"] = [4, 1]
    lws["size"] = 1
    lws["flags"] = R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID
    lws["group_base"], lws["group_count"] = [0, ng - 1], [ng - 1, 1]
    groups = R.aligned_empty(ng, R.GROUP_REC)
    groups["lws_index"][: ng - 1] = 0
    groups["lws_index"][ng - 1] = 1
    groups["leader_node"] = R.NONE
    pst, pid = R.aligned_empty(0, R.POD_STATE), R.aligned_empty(0, R.POD_IDENT)
    nodes = R.aligned_empty(1, R.NODE_REC)
    engine.upload_nodes(nodes, 1)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_sweep(0)
    n = -(-(1 << 32) // (ng - 1))
    with pytest.raises(LwseError) as e:
        engine.resident_rollout_whatif(np.zeros(n, np.uint32), np.repeat(lws[:1], n), steps=False)
    assert e.value.status == ERR_UNSUPPORTED
    w = type("W", (), dict(lws=lws, groups=groups, pod_state=pst, pod_ident=pid, nodes=nodes, flags=0))
    rows = np.array([1, 1], np.uint32)
    recs = R.aligned_empty(2, R.LWS_REC)
    recs[:] = lws[[1, 1]]
    recs["flags"][0] |= np.uint32(R.LWS_UPDATED)
    recs["replicas"][1] = 3
    _same(engine.resident_rollout_whatif(rows, recs), rollout_whatif(w, rows, recs), "after the refusal")


def test_whatifs_between_pipelined_ticks_change_no_tick(engine):
    """Two ticks in flight, a what-if after every submit: every tick's change lists and the final outputs
    are those of the same ticks without what-ifs, and each what-if is the reference's over the oracle's
    state after the ticks submitted so far."""
    runs = []
    for with_whatifs in (False, True):
        t, reqs, plan, flags = _resident_world(engine, 33)
        engine.resident_tick(engine.make_tick((), flags))
        ticks = churn.ArenaPlan(engine, plan, flags).ticks
        pst, grp, rq = t.pod_state.copy(), t.groups.copy(), reqs.copy()
        states = []
        for k in range(8):
            churn.apply_to_mirror(plan[k % len(plan)], pst, grp, rq)
            states.append((grp.copy(), pst.copy()))
        rows, recs = proposals(t.lws, 400, 33)
        lists, wis = [], []
        engine.resident_tick_submit(ticks[0])
        for k in range(1, 8):
            engine.resident_tick_submit(ticks[k % len(ticks)])
            if with_whatifs:
                wis.append(engine.resident_rollout_whatif(rows, recs))
            lists.append(_tick_lists(engine.resident_tick_wait()))
        lists.append(_tick_lists(engine.resident_tick_wait()))
        runs.append((lists, wis, engine.resident_outputs()))
    (a, _, out_a), (b, wis, out_b) = runs
    assert a == b
    assert out_a[0].tobytes() == out_b[0].tobytes() and out_a[1].tobytes() == out_b[1].tobytes()
    for k, got in enumerate(wis, start=1):
        g, p = states[k]
        w = type("W", (), dict(lws=t.lws, groups=g, pod_state=p, pod_ident=t.pod_ident, nodes=t.nodes, flags=t.flags))
        _same(got, rollout_whatif(w, rows, recs), f"what-if after submitting tick {k}")
