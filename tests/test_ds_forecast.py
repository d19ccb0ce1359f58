"""The rollout forecast's CPU reference (tests/ds_forecast_ref.py) against the ground truth it replays:

  - the 22 exact ComputeAllSteps sequences (planner_test.go:106-505, tests/golden/planner_sequences.json),
    each built as a DS with one annotated old revision and no new revision yet;
  - the reference's multi-cycle executor flows (executor_test.go:1244-1298, and the newest-first drain
    cases of executor_test.go:486-556), and seeded random DS, replayed object by object with DsSim
    (child LWS created, scaled and deleted the way the reference's LWSManager would) over
    oracle.sweep_ds, cycle for cycle;
  - the summaries against the trajectory they came from.
"""
import copy
import json
import os
import random

import numpy as np
import pytest

import oracle
from ds_forecast_ref import ds_forecast, trajectory
from ds_sim import DsSim
from lws_b200 import api, encoder, synth
from lws_b200 import records as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "planner_sequences.json")))["cases"]


def golden_item(case):
    roles = [api.DisaggregatedRoleSpec(f"r{i}", case["target"][i],
                                       api.RollingUpdateConfiguration(maxSurge=ms, maxUnavailable=mu))
             for i, (ms, mu) in enumerate(case["config"])]
    ds = api.DisaggregatedSet("g", roles=roles)
    children = [api.ChildLWS(f"r{i}", "old", s, s, 1.0, {api.DSInitialReplicasAnnotationKey: str(s)})
                for i, s in enumerate(case["source"])]
    return encoder.DsItem(ds, "new", children)


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden_sequences(case):
    t = encoder.encode_ds([golden_item(case)])
    res = ds_forecast(t.ds, t.roles, t.revroles)
    fc = res["ds"][0]
    if not any(case["source"]):  # reconcileSimple scales to target in one reconcile: no rollout
        assert fc["flags"] == 0 and fc["cycles"] == 0 and fc["n_steps"] == 0
        return
    want = [[(o[i], nw[i]) for i in range(len(o))] for o, nw in case["steps"][1:]]
    assert trajectory(res, t.ds, 0) == want
    assert fc["flags"] == R.DSF_ROLLING | R.DSF_DONE
    seq = case["steps"]  # peak / floor exactly, from the golden sequence itself
    for i in range(len(case["source"])):
        now = seq[0][0][i] + seq[0][1][i]
        peak = max([now] + [a[0][i] + b[1][i] for a, b in zip(seq, seq[1:])])
        floor = min([now] + [b[0][i] + a[1][i] for a, b in zip(seq, seq[1:])])
        assert (int(res["roles"][i]["peak_replicas"]), int(res["roles"][i]["floor_available"])) == (peak, floor)
    _check_summaries(res, t.ds, 0)


def _check_summaries(res, ds, d):
    """Finals from the trajectory, and peak / floor bounding every transition in it.  (The exact values
    are compared with an independent replay in check_against_sim.)"""
    n, base = int(ds["n_roles"][d]), int(ds["role_base"][d])
    fr = res["roles"][base: base + n]
    steps = trajectory(res, ds, d)
    start = [(int(fr[i]["peak_replicas"]), int(fr[i]["floor_available"])) for i in range(n)]
    if not steps:
        for i in range(n):
            assert fr[i]["peak_replicas"] == fr[i]["floor_available"] == fr[i]["final_old"] + fr[i]["final_new"]
        return
    assert [(int(fr[i]["final_old"]), int(fr[i]["final_new"])) for i in range(n)] == list(steps[-1])
    for i, (peak, floor) in enumerate(start):
        seq = [s[i] for s in steps]
        # the state before the first step is not in the trajectory: the bounds include every transition
        for (o0, n0), (o1, n1) in zip(seq, seq[1:]):
            assert peak >= o0 + n1 and floor <= o1 + n0


# ---------------------------------------------------------------------------- DsSim replays
def sim_replay(item, cap=400):
    """The contract's cycles played on the objects: every child ready, reconcile (oracle sweep + DsSim's
    LWSManager), until a cycle changes nothing.  → (steps, cycles, final totals, stopped, peak, floor):
    per role, peak = max of old + new now and of old_k + new_{k+1}, floor = min of old + new now and of
    old_{k+1} + new_k."""
    names = encoder.encode_ds([item]).role_names[0]
    sim = DsSim(item.ds, item.revision, copy.deepcopy(item.children),
                lambda t: oracle.sweep_ds(t.ds, t.roles, t.revroles))

    def state():
        return sorted((c.revision, c.role, c.replicas) for c in sim.children)

    def totals():
        out = []
        for name in names:
            old = sum((1 if c.replicas is None else c.replicas) for c in sim.children
                      if c.role == name and c.revision != item.revision)
            new = sum((1 if c.replicas is None else c.replicas) for c in sim.children
                      if c.role == name and c.revision == item.revision)
            out.append((old, new))
        return out

    steps, cycles, cur = [], 0, totals()
    peak = [o + nw for o, nw in cur]
    floor = list(peak)
    for _ in range(cap):
        before = state()
        for c in sim.children:
            c.readyReplicas = 1 if c.replicas is None else c.replicas
        flags = sim.reconcile()
        if state() == before and not flags & R.DOUT_INIT:
            return steps, cycles, cur, True, peak, floor
        cycles += 1
        nxt = totals()
        for i, ((o0, n0), (o1, n1)) in enumerate(zip(cur, nxt)):
            peak[i] = max(peak[i], o0 + n1)
            floor[i] = min(floor[i], o1 + n0)
        if nxt != cur:
            steps.append(nxt)
        cur = nxt
    return steps, cycles, cur, False, peak, floor


def check_against_sim(item):
    t = encoder.encode_ds([item])
    res = ds_forecast(t.ds, t.roles, t.revroles)
    fc = res["ds"][0]
    if not fc["flags"] & R.DSF_ROLLING:
        assert fc["cycles"] == 0 and fc["n_steps"] == 0
        now = [(int(x["final_old"]), int(x["final_new"])) for x in res["roles"]]
        assert [int(x["peak_replicas"]) for x in res["roles"]] == [o + nw for o, nw in now]
        assert [int(x["floor_available"]) for x in res["roles"]] == [o + nw for o, nw in now]
        return res
    steps, cycles, final, stopped, peak, floor = sim_replay(item)
    assert stopped
    assert trajectory(res, t.ds, 0) == steps
    assert int(fc["cycles"]) == cycles
    n = len(final)
    fr = res["roles"][:n]
    assert [(int(x["final_old"]), int(x["final_new"])) for x in fr] == final
    assert [int(x["peak_replicas"]) for x in fr] == peak
    assert [int(x["floor_available"]) for x in fr] == floor
    S = int(t.ds[0]["n_spec_roles"])
    done = all(o == 0 for o, _ in final) and all(final[i][1] == int(t.roles[i]["target_replicas"]) for i in range(S))
    assert bool(fc["flags"] & R.DSF_DONE) == done and bool(fc["flags"] & R.DSF_UNFINISHED) == (not done)
    _check_summaries(res, t.ds, 0)
    return res


def abc_item(target, a, b, surge, order):
    cfg = [api.RollingUpdateConfiguration(maxSurge=surge[i], maxUnavailable=0) for i in range(2)]
    ds = api.DisaggregatedSet("test", roles=[api.DisaggregatedRoleSpec("prefill", target[0], cfg[0]),
                                             api.DisaggregatedRoleSpec("decode", target[1], cfg[1])])
    kids = {"A": [api.ChildLWS("prefill", "A", a[0], a[0], 0.0), api.ChildLWS("decode", "A", a[1], a[1], 0.0)],
            "B": [api.ChildLWS("prefill", "B", b[0], b[0], 0.0), api.ChildLWS("decode", "B", b[1], b[1], 0.0)]}
    return encoder.DsItem(ds, "C", [c for rev in order for c in kids[rev]])


FLOWS = [((2, 4), (1, 2), (1, 2), (1, 1)), ((4, 3), (1, 2), (3, 1), (1, 2))]  # executor_test.go:1244-1298


@pytest.mark.parametrize("order", [("A", "B"), ("B", "A")])
@pytest.mark.parametrize("flow", FLOWS)
def test_reference_flows_match_sim(flow, order):
    res = check_against_sim(abc_item(*flow, order))
    assert res["ds"][0]["flags"] & R.DSF_DONE


SORT_REVISIONS = [  # executor_test.go:506-511, :536-555
    [("hash1", 0, 0)],
    [("newest", 120, 120), ("oldest", 0, 0), ("middle", 60, 60)],
    [("d", 30, 30), ("a", 0, 0), ("c", 20, 20), ("b", 10, 10)],
    [("A", 0, 20), ("B", 10, 10)],
    [("B", 10, 10), ("A", 0, 20)],
]


@pytest.mark.parametrize("revisions", SORT_REVISIONS)
def test_sort_flows_match_sim(revisions):
    cfg = api.RollingUpdateConfiguration(maxSurge=1, maxUnavailable=0)
    n = len(revisions)
    ds = api.DisaggregatedSet("test", roles=[api.DisaggregatedRoleSpec("prefill", n, cfg),
                                             api.DisaggregatedRoleSpec("decode", n, cfg)])
    children = []
    for h, tp, td in revisions:
        children += [api.ChildLWS("prefill", h, 1, 1, float(tp)), api.ChildLWS("decode", h, 1, 1, float(td))]
    res = check_against_sim(encoder.DsItem(ds, "new", children))
    assert res["ds"][0]["flags"] & R.DSF_DONE


def random_item(rng: random.Random):
    n_spec = rng.randint(2, 10)
    cfgs = [None, (1, 0), (2, 0), ("25%", 0), (0, 1), (1, 1), ("50%", "50%"), ("x%", 1), (1, "bad"), (0, 0)]
    roles = []
    for i in range(n_spec):
        c = rng.choice(cfgs)
        ru = None if c is None else api.RollingUpdateConfiguration(maxSurge=c[0], maxUnavailable=c[1])
        roles.append(api.DisaggregatedRoleSpec(f"r{i}", rng.choice([None, 0, 1, 2, 3, 5, 8]), ru))
    ds = api.DisaggregatedSet(f"ds{rng.random()}", roles=roles)
    names = [r.name for r in roles] + (["gone"] if n_spec < 10 and rng.random() < 0.3 else [])
    children, clock = [], 0.0
    for v in range(rng.randint(1, 3)):
        clock += rng.choice([0.0, 1.0, 2.0])
        for name in names:
            if rng.random() < 0.1:
                continue
            rep = None if rng.random() < 0.05 else rng.randint(0, 8)
            ann = {}
            if rng.random() < 0.7:
                ann[api.DSInitialReplicasAnnotationKey] = str(rng.choice([rep or 0, rng.randint(0, 8)]))
            children.append(api.ChildLWS(name, f"old{v}", rep, rng.randint(0, rep or 1), clock, ann))
    if rng.random() < 0.5:
        clock += 1.0
        for r in roles:
            if rng.random() < 0.9:
                tgt = 1 if r.replicas is None else r.replicas
                rep = rng.randint(0, tgt)
                children.append(api.ChildLWS(r.name, "new", rep, rng.randint(0, rep), clock))
    rng.shuffle(children)
    return encoder.DsItem(ds, "new", children)


@pytest.mark.parametrize("seed", range(6))
def test_random_ds_match_sim(seed):
    rng = random.Random(seed)
    rolling = 0
    for _ in range(60):
        res = check_against_sim(random_item(rng))
        rolling += bool(res["ds"][0]["flags"] & R.DSF_ROLLING)
    assert rolling > 20


def test_batched_replay_equals_one_ds_at_a_time():
    """DS that stop early keep their state while the others replay: the batch equals each DS alone."""
    rng = random.Random(77)
    items = [random_item(rng) for _ in range(40)] + [abc_item(*FLOWS[1], ("B", "A"))]
    t = encoder.encode_ds(items)
    res = ds_forecast(t.ds, t.roles, t.revroles)
    for d, item in enumerate(items):
        one = encoder.encode_ds([item])
        r1 = ds_forecast(one.ds, one.roles, one.revroles)
        got, want = res["ds"][d].copy(), r1["ds"][0].copy()
        got["step_base"] = want["step_base"] = 0
        assert got.tobytes() == want.tobytes()
        base, n = int(t.ds[d]["role_base"]), int(t.ds[d]["n_roles"])
        assert res["roles"][base: base + n].tobytes() == r1["roles"].tobytes()
        assert trajectory(res, t.ds, d) == trajectory(r1, one.ds, 0)


def test_synth_tables_summaries_and_truncation():
    t = synth.make_ds(3000, (2, 3, 5, 10), fuzz=0.05, seed=4)
    ds = t.ds.copy()
    ds["n_roles"][5] = 11  # BAD_TABLE rows
    ds["rev_base"][7] = len(t.revroles)
    res = ds_forecast(ds, t.roles, t.revroles)
    assert res["ds"]["flags"][5] == R.DSF_BAD_TABLE and res["ds"]["flags"][7] == R.DSF_BAD_TABLE
    rolling = (res["ds"]["flags"] & R.DSF_ROLLING) != 0
    assert rolling.sum() > 1000 and (res["ds"]["n_steps"] > 0).sum() > 1000
    for d in np.nonzero(rolling)[0][:300]:
        _check_summaries(res, ds, int(d))
    cap = res["n_steps_needed"] // 2
    part = ds_forecast(ds, t.roles, t.revroles, step_capacity=cap)
    trunc = (part["ds"]["flags"] & R.DSF_TRUNCATED) != 0
    rows = part["ds"]["n_steps"].astype(np.int64) * ds["n_roles"]
    end = part["ds"]["step_base"].astype(np.int64) + rows
    assert np.array_equal(trunc, (rows > 0) & (end > cap))
    assert part["steps"].tobytes() == res["steps"][: part["n_steps_written"]].tobytes()
    flags_off = part["ds"].copy()
    flags_off["flags"] &= ~np.uint32(R.DSF_TRUNCATED)
    assert flags_off.tobytes() == res["ds"].tobytes() and part["roles"].tobytes() == res["roles"].tobytes()
    summ = ds_forecast(ds, t.roles, t.revroles, steps=False)
    assert summ["steps"] is None and summ["ds"].tobytes() == res["ds"].tobytes()
    assert summ["roles"].tobytes() == res["roles"].tobytes()


def test_informer_names_a_forecast():
    """DsIncrementalEncoder.forecast_of: one DS's forecast by name, with role names and per-role steps."""
    from lws_b200 import ds_informer

    items = [abc_item(*FLOWS[1], ("A", "B"))] + [random_item(random.Random(s)) for s in range(5)]
    enc = ds_informer.DsIncrementalEncoder(items)
    ds, roles, rr = enc.tables()
    res = ds_forecast(ds, roles, rr)
    named = enc.forecast_of(res, "default", "test")
    row = enc.ds_row("default", "test")
    assert named["flags"] == int(res["ds"][row]["flags"]) and set(named["roles"]) == {"prefill", "decode"}
    steps = trajectory(res, ds, row)
    assert named["roles"]["prefill"]["trajectory"] == [s[0] for s in steps]
    assert named["roles"]["decode"]["trajectory"] == [s[1] for s in steps]
    assert named["roles"]["decode"]["final_new"] == 3 and named["roles"]["prefill"]["final_old"] == 0
    summaries = ds_forecast(ds, roles, rr, steps=False)
    assert enc.forecast_of(summaries, "default", "test")["roles"]["prefill"]["trajectory"] == []
