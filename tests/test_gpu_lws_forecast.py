"""The LeaderWorkerSet rolling-update forecast on the device (lwse_lws_forecast_host /
lwse_resident_forecast) against the CPU reference of tests/lws_forecast_ref.py, byte for byte: the trace
checkpoints, full-size C5 and C3, fuzzed tables (percent surge / unavailable, spec partitions, irregular,
rollingUpdateParameters-error and bad-table rows, objects wide enough for multi-lane tiles), truncated
trajectories, and the resident tables after patched ticks, with forecasts between pipelined ticks."""
import numpy as np
import pytest

import oracle
from lws_b200 import churn, synth
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast
from test_lws_forecast import checkpoints, sim_at, sim_tables

pytestmark = pytest.mark.gpu

ERR_NOT_READY = -6  # lwse_status


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def _same(got, want, where=""):
    assert got["lws"].tobytes() == want["lws"].tobytes(), f"{where}: per-object forecast differs"
    assert got["n_steps_needed"] == want["n_steps_needed"] and got["n_steps_written"] == want["n_steps_written"]
    if want["steps"] is None:
        assert got["steps"] is None
    else:
        assert got["steps"].tobytes() == want["steps"].tobytes(), f"{where}: trajectory rows differ"


# flag bytes a group pass can give (COND_* only with COUNTED; with COUNTED, STATE_* are 0 or equal COND_*)
_BYTES = np.array([0, 1, 2, 3, 4, 4 | 8, 4 | 16, 4 | 8 | 16, 1 | 4 | 8, 2 | 4 | 16, 31], np.uint32)


def fuzzed(n_lws, lo, hi, seed):
    """Object rows with random rollout state over random flag bytes: percent and integer surge /
    unavailable, spec partitions, pending template changes, missing StatefulSets, stale annotations, and a
    few irregular, intstr-invalid, label-invalid and bad-table rows.  Every 37th object has a pending
    template change and a negative integer maxUnavailable (which the webhook rejects) with maxSurge at
    replicas: its first pass (Case 2) asks for 2 * replicas + 20 groups, more than its slots hold, and the
    replay stops UNFINISHED before any cycle.  (Such a spec must not reach Case 5: a negative rolling step
    can put the walk's rolling-step partition past the StatefulSet's replicas, where the reference indexes
    past its replica states and the C oracle reads past its array.)  Every 101st object (from the 5th) has
    more replicas than LWSE_LWS_FORECAST_MAX_SLOTS and is not forecast."""
    rng = np.random.default_rng(seed)
    lws = R.aligned_empty(n_lws, R.LWS_REC)
    reps = rng.integers(lo, hi + 1, n_lws)
    gc = np.maximum(reps + rng.integers(-3, 4, n_lws), 0)
    lws["group_count"] = gc
    lws["group_base"] = np.cumsum(gc) - gc
    lws["replicas"] = reps
    lws["size"] = rng.choice([1, 2, 8], n_lws)
    lws["rev_hash"] = rng.integers(1, 2**63, n_lws, dtype=np.uint64)
    pct_s, pct_u = rng.random(n_lws) < 0.3, rng.random(n_lws) < 0.3
    lws["max_surge"] = np.where(pct_s, rng.integers(0, 60, n_lws), rng.integers(0, 4, n_lws))
    lws["max_unavailable"] = np.where(pct_u, rng.integers(0, 60, n_lws), rng.integers(0, 4, n_lws))
    lws["partition"] = np.where(rng.random(n_lws) < 0.2, rng.integers(0, hi + 1, n_lws), 0)
    lws["sts_replicas"] = np.maximum(reps + rng.integers(-2, 4, n_lws), 0)
    lws["sts_partition"] = rng.integers(0, hi + 1, n_lws)
    lws["sts_replicas_annotation"] = np.where(rng.random(n_lws) < 0.8, reps, reps + 1)
    lws["uid_hash"] = rng.integers(1, 2**63, n_lws, dtype=np.uint64)
    f = np.uint32(R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID) * (rng.random(n_lws) < 0.9)
    f |= np.where(pct_s, R.LWS_SURGE_IS_PERCENT, 0).astype(np.uint32)
    f |= np.where(pct_u, R.LWS_UNAVAIL_IS_PERCENT, 0).astype(np.uint32)
    f |= np.where(rng.random(n_lws) < 0.2, R.LWS_UPDATED, 0).astype(np.uint32)
    odd = rng.random(n_lws)
    f |= np.where(odd < 0.01, R.LWS_IRREGULAR, 0).astype(np.uint32)
    f |= np.where((odd >= 0.01) & (odd < 0.02), R.LWS_INTSTR_INVALID, 0).astype(np.uint32)
    f |= np.where((odd >= 0.02) & (odd < 0.03), R.LWS_GROUP_LABEL_INVALID, 0).astype(np.uint32)
    neg, huge = np.arange(0, n_lws, 37), np.arange(5, n_lws, 101)
    lws["max_unavailable"][neg] = -20
    lws["max_surge"][neg] = reps[neg]
    lws["sts_replicas"][neg] = reps[neg]
    f[neg] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT | R.LWS_UNAVAIL_IS_PERCENT | R.LWS_IRREGULAR | R.LWS_INTSTR_INVALID
                         | R.LWS_GROUP_LABEL_INVALID)
    f[neg] |= np.uint32(R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID | R.LWS_UPDATED)
    lws["replicas"][huge] = R.LWS_FORECAST_MAX_SLOTS + 1
    lws["flags"] = f
    n_groups = int(gc.sum())
    plain = np.setdiff1d(np.arange(n_lws), np.concatenate([neg, huge]))
    bad = rng.choice(plain, size=max(n_lws // 200, 2), replace=False)
    lws["group_base"][bad] = n_groups  # past the table
    lws["group_count"][bad] = 1 + bad % 3
    go = R.aligned_empty(n_groups, R.GROUP_OUT)
    go["flags"] = rng.choice(_BYTES, n_groups) | (rng.integers(0, 1 << 9, n_groups, dtype=np.uint32) << 5)
    return lws, go


def test_trace_checkpoints_through_the_kernel(engine):
    rows, outs = [], []
    base = 0
    for name, k in checkpoints():
        lws, _, go = sim_tables(sim_at(name, k))
        lws["group_base"] += base
        base += len(go)
        rows.append(lws)
        outs.append(go)
    lws = np.concatenate(rows)
    go = np.concatenate(outs)
    want = lws_forecast(lws, go)
    _same(engine.lws_forecast(lws, go), want, "traces")
    assert want["n_steps_needed"] > 50


@pytest.mark.parametrize("name", ["C5", "C3"])
def test_full_size_equals_reference(engine, name):
    t = synth.make(name)
    lo, go, _ = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, flags=t.flags, threads=8)
    want = lws_forecast(t.lws, go)
    got = engine.lws_forecast(t.lws, go)
    _same(got, want, name)
    if name == "C5":
        assert (got["lws"]["n_steps"] > 0).sum() > 1000
    summ = engine.lws_forecast(t.lws, go, steps=False)
    assert summ["lws"].tobytes() == got["lws"].tobytes() and summ["steps"] is None


@pytest.mark.parametrize("lo,hi,seed", [(0, 12, 1), (1, 40, 2), (100, 400, 3), (600, 1500, 4)])
def test_fuzzed_equals_reference(engine, lo, hi, seed):
    """Narrow objects run one lane each; the last two tables average more than 64 groups per object and
    run multi-lane tiles."""
    lws, go = fuzzed(3000 if hi < 100 else 300, lo, hi, seed)
    want = lws_forecast(lws, go)
    _same(engine.lws_forecast(lws, go), want, f"fuzz {seed}")
    f = want["lws"]["flags"]
    for bit in (R.LWSF_ROLLING, R.LWSF_WAITING, R.LWSF_DONE, R.LWSF_HELD, R.LWSF_UNFINISHED, R.LWSF_NOT_FORECAST,
                R.LWSF_BAD_TABLE):
        assert (f & bit).any(), bit
    huge = np.arange(5, len(lws), 101)
    neg = np.setdiff1d(np.arange(0, len(lws), 37), huge)
    assert (want["lws"]["flags"][huge] == R.LWSF_NOT_FORECAST).all()
    fn = want["lws"][neg]
    assert ((fn["flags"] & R.LWSF_UNFINISHED) != 0).all() and (fn["n_steps"] == 0).all()


def test_truncated_trajectory_writes_only_what_fits(engine):
    lws, go = fuzzed(2000, 1, 30, 7)
    full = lws_forecast(lws, go)
    need = full["n_steps_needed"]
    for cap in (0, 1, need // 3, need - 1, need, need + 5):
        want = lws_forecast(lws, go, step_capacity=cap)
        got = engine.lws_forecast(lws, go, step_capacity=cap)
        _same(got, want, f"capacity {cap}")
        assert got["n_steps_written"] <= cap
        trunc = (got["lws"]["flags"] & R.LWSF_TRUNCATED) != 0
        assert trunc.any() == (cap < need)
    none = engine.lws_forecast(lws, go, steps=False)
    assert none["steps"] is None and none["n_steps_written"] == 0 and none["n_steps_needed"] == need
    assert none["lws"].tobytes() == full["lws"].tobytes()


def _resident_world(engine, seed):
    p = synth.profile("fuzz", 0.5)
    p.n_namespaces = 3
    t = synth.make(p, seed=seed)
    reqs = t.place_requests()
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    occ = R.occupancy_of(t.pod_ident, len(t.nodes))
    plan = churn.make_plan(t, reqs, oracle.place(t.nodes, occ, t.n_domains, t.n_namespaces, reqs), 0.03, 0.05,
                           n_sets=6, seed=seed)
    return t, reqs, plan, t.flags | R.TICK_PLACE


def test_resident_forecast_after_patched_ticks(engine):
    from lws_b200.engine import LwseError

    t, reqs, plan, flags = _resident_world(engine, 21)
    with pytest.raises(LwseError) as e:
        engine.resident_forecast()
    assert e.value.status == ERR_NOT_READY
    engine.resident_tick(engine.make_tick((), flags))
    ticks = churn.ArenaPlan(engine, plan, flags).ticks
    pst, grp, rq = t.pod_state.copy(), t.groups.copy(), reqs.copy()
    for k in range(len(plan)):
        churn.apply_to_mirror(plan[k], pst, grp, rq)
        engine.resident_tick(ticks[k])
        lo, go = engine.resident_outputs()
        want = lws_forecast(t.lws, go)
        _same(engine.resident_forecast(), want, f"tick {k}")
    # a pod patch without a sweep: the group results no longer belong to the rows
    engine.resident_tick(engine.make_tick([(R.TABLE_POD_STATE, np.array([0], np.uint32), pst[:1].copy())],
                                          flags | R.TICK_NO_SWEEP))
    with pytest.raises(LwseError) as e:
        engine.resident_forecast()
    assert e.value.status == ERR_NOT_READY
    engine.resident_tick(engine.make_tick((), flags))
    _same(engine.resident_forecast(), lws_forecast(t.lws, engine.resident_outputs()[1]), "after the sweep")


def _tick_lists(res):
    out = []
    for key in ("lws", "group", "place"):
        if f"{key}_rows" not in res:
            continue
        rows = res[f"{key}_rows"]
        vals = res[f"{key}_out"]
        order = np.argsort(rows, kind="stable")
        out.append((rows[order].tobytes(), vals[order].tobytes()))
    return out


def test_forecasts_between_pipelined_ticks_change_no_tick(engine):
    """Two ticks in flight, a resident forecast after every submit: every tick's change lists are the
    ones of the same ticks without forecasts, and each forecast is the reference's forecast of the group
    results of the most recently submitted tick (the oracle's sweep after the patches of every tick
    submitted so far)."""
    runs = []
    for with_forecasts in (False, True):
        t, reqs, plan, flags = _resident_world(engine, 33)
        engine.resident_tick(engine.make_tick((), flags))
        ticks = churn.ArenaPlan(engine, plan, flags).ticks
        pst, grp, rq = t.pod_state.copy(), t.groups.copy(), reqs.copy()
        after = []  # the oracle's group results after each submitted tick
        for k in range(8):
            churn.apply_to_mirror(plan[k % len(plan)], pst, grp, rq)
            after.append(oracle.sweep_lws(t.lws, grp, pst, t.pod_ident, t.nodes, flags=t.flags)[1])
        lists, fcs = [], []
        engine.resident_tick_submit(ticks[0])
        for k in range(1, 8):
            engine.resident_tick_submit(ticks[k % len(ticks)])
            if with_forecasts:
                fcs.append(engine.resident_forecast())
            lists.append(_tick_lists(engine.resident_tick_wait()))
        lists.append(_tick_lists(engine.resident_tick_wait()))
        runs.append((lists, fcs, engine.resident_outputs()))
    (a, _, out_a), (b, fcs, out_b) = runs
    assert a == b
    assert out_a[0].tobytes() == out_b[0].tobytes() and out_a[1].tobytes() == out_b[1].tobytes()
    assert out_b[1].tobytes() == after[-1].tobytes()
    for k, fc in enumerate(fcs, start=1):
        _same(fc, lws_forecast(t.lws, after[k]), f"forecast after submitting tick {k}")
    assert fcs[-1]["n_steps_needed"] > 0
