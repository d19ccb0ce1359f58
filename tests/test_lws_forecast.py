"""The LeaderWorkerSet forecast's CPU reference (tests/lws_forecast_ref.py) against the ground truth:

  - from every checkpoint of the integration traces (tests/traces.py), an LwsSim replay in which an ideal
    StatefulSet controller and kubelet act after every reconcile (groups at or past the new replicas
    deleted, missing ones created, every group made ready, those below the partition keeping their
    revision), cycle for cycle;
  - T7 (leaderworkerset_test.go:1088-1205), whose trace is the replay's own sequence;
  - the availability floor against maxUnavailable for updates that start at rest;
  - the layout of the new records against lwse.h.
"""
import copy
import ctypes as C
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from lws_b200 import api
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast, trajectory
from sim import LwsSim
from traces import TRACES, make_lws

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_sweep(tables, flags=0):
    lo, go, _ = oracle.sweep_lws(tables.lws, tables.groups, tables.pod_state, tables.pod_ident, tables.nodes,
                                 flags=flags)
    return lo, go


def sim_tables(s):
    """The sim's current tables and their sweep.  LwsSim's leader pods are owned by the leader
    StatefulSet (named after the LWS, not the group), which the encoder marks LWS_IRREGULAR for the
    pod-restart path; the rollout arithmetic does not read those pods, so the flag is dropped here."""
    t = s.last_tables
    lws = t.lws.copy()
    lws["flags"] &= ~np.uint32(R.LWS_IRREGULAR)
    lo, go, _ = oracle.sweep_lws(lws, t.groups, t.pod_state, t.pod_ident, t.nodes)
    return lws, lo, go


def sts_step(s):
    """The ideal StatefulSet controller and kubelet after one reconcile, as one change: groups at or past
    the StatefulSet's replicas deleted, missing ones created, every group running and ready, those at or
    past its partition at its revision (SetPodGroupToReady, test/testutils/util.go:386-401, without the
    intermediate settles that would let the controller see a group below the partition at the new
    revision)."""
    n, p = s.leader_sts.replicas, s.leader_sts.partition
    for name in list(s.pods):
        if int(name.rsplit("-", 1)[1]) >= n:
            del s.pods[name]
            s.stss.pop(name, None)
    for i in range(n):
        if f"{s.lws.name}-{i}" not in s.pods:
            s.create_leader_pods(i, i + 1)
    for i in range(n):
        name = f"{s.lws.name}-{i}"
        pod = s.pods[name]
        if i >= p:
            pod.labels[api.RevisionKey] = s.leader_sts.labels[api.RevisionKey]
        pod.phase = "Running"
        pod.readyCondition = True
        if s.lws.size > 1:
            s.stss.pop(name, None)  # recreated by the pod controller with the pod's revision
    if s.lws.size > 1:
        s.reconcile_pods()
        for i in range(n):
            sts = s.stss[f"{s.lws.name}-{i}"]
            sts.availableReplicas = sts.statusReplicas = sts.replicas
            sts.currentRevision = sts.updateRevision = ""
    s.settle()


def snapshot(s):
    return s.state(), sorted((k, v.labels.get(api.RevisionKey), v.phase, v.readyCondition) for k, v in s.pods.items())


def sim_replay(s, cap=64):
    """The states after every cycle that changed something, as the forecast's trajectory rows."""
    rows = []
    for _ in range(cap):
        before = snapshot(s)
        sts_step(s)
        if snapshot(s) == before:
            break
        rows.append(tuple(int(v) for v in s.state()))
    return rows


def checkpoints():
    for name, (cfg, steps) in TRACES.items():
        for k in range(len(steps)):
            yield name, k


def sim_at(name, k):
    cfg, steps = TRACES[name]
    s = LwsSim(make_lws(cfg), oracle_sweep)
    s.settle()
    s.create_leader_pods(0, cfg["replicas"])
    for act, _ in steps[: k + 1]:
        act(s)
    return s


@pytest.mark.parametrize("name,k", list(checkpoints()))
def test_reference_matches_sim_replay(name, k):
    s = sim_at(name, k)
    lws, lo, go = sim_tables(s)
    assert (int(lo[0]["sts_partition"]), int(lo[0]["sts_replicas"])) == s.state()[:2]
    res = lws_forecast(lws, go)
    fc = res["lws"][0]
    want = sim_replay(copy.deepcopy(s))
    assert trajectory(res, 0) == want
    assert fc["cycles"] == fc["n_steps"] == len(want)
    assert not fc["flags"] & (R.LWSF_UNFINISHED | R.LWSF_NOT_FORECAST | R.LWSF_BAD_TABLE | R.LWSF_TRUNCATED)
    final = want[-1] if want else s.state()
    assert (int(fc["final_partition"]), int(fc["final_replicas"])) == final[:2]
    assert bool(fc["flags"] & R.LWSF_ROLLING) == (int(lo[0]["flags"] & R.LOUT_COND_MASK) >> R.LOUT_COND_SHIFT
                                                  == R.COND_UPDATE_IN_PROGRESS)
    assert fc["peak_sts_replicas"] >= max([s.leader_sts.replicas] + [r[1] for r in want])
    assert fc["floor_ready"] <= min([int(lo[0]["ready_replicas"])] + [r[2] for r in want])


def test_t7_reproduces_the_trace():
    """From the state right after the template update, the replay is the trace, step for step: the
    (partition, replicas) pairs with consecutive repeats dropped, and the final row in full.  (The row
    before the last still counts the surge group, which the last apply removes.)"""
    cfg, steps = TRACES["T7"]
    s = sim_at("T7", 1)
    lws, lo, go = sim_tables(s)
    res = lws_forecast(lws, go)
    rows = trajectory(res, 0)
    pairs = [s.state()[:2]]
    for r in rows:
        if r[:2] != pairs[-1]:
            pairs.append(r[:2])
    trace = [w for _, w in steps[1:]]
    assert pairs == [w[:2] for w in trace]
    assert rows[-1] == trace[-1][:4] == (0, 4, 4, 4)
    assert rows == [(3, 5, 5, 1), (2, 5, 5, 2), (1, 5, 5, 3), (0, 5, 5, 4), (0, 4, 5, 5), (0, 4, 4, 4)]
    fc = res["lws"][0]
    assert fc["flags"] == R.LWSF_ROLLING | R.LWSF_WAITING | R.LWSF_DONE
    assert (fc["peak_sts_replicas"], fc["floor_ready"]) == (5, 4)


def at_rest_update(replicas, mu, ms):
    cfg = dict(replicas=replicas, maxUnavailable=mu, maxSurge=ms, partition=0, size=2)
    s = LwsSim(make_lws(cfg), oracle_sweep)
    s.bootstrap()
    s.update_template()
    lws, _, go = sim_tables(s)
    return lws_forecast(lws, go)["lws"][0]


@pytest.mark.parametrize("replicas,mu,ms", [c for c in itertools.product(range(1, 7), range(4), range(4))
                                            if c[1] or c[2]])
def test_floor_respects_max_unavailable(replicas, mu, ms):
    """An update that starts at rest never has fewer than replicas - maxUnavailable ready groups, and
    finishes."""
    fc = at_rest_update(replicas, mu, ms)
    assert fc["flags"] & R.LWSF_DONE and not fc["flags"] & R.LWSF_UNFINISHED
    assert (fc["final_partition"], fc["final_replicas"]) == (0, replicas)
    assert fc["floor_ready"] >= replicas - min(mu, replicas)


@pytest.mark.parametrize("ms", [1, 2, 3])
def test_single_replica_surge_update(ms):
    """replicas 1, maxUnavailable 0: once the surge group is ready the controller keeps it (replicas 2)
    while group 0 rolls, and only then scales back, so a ready group is always left.  (A sim that lets the
    controller reconcile while group 0 is momentarily at the new revision sees (partition 0, replicas 1)
    in one write instead, and a floor of 0; the ideal StatefulSet never shows that state.)"""
    cfg = dict(replicas=1, maxUnavailable=0, maxSurge=ms, partition=0, size=2)
    s = LwsSim(make_lws(cfg), oracle_sweep)
    s.bootstrap()
    s.update_template()
    lws, _, go = sim_tables(s)
    res = lws_forecast(lws, go)
    assert trajectory(res, 0) == [(0, 2, 2, 1), (0, 1, 2, 2), (0, 1, 1, 1)] == sim_replay(copy.deepcopy(s))
    assert (res["lws"][0]["peak_sts_replicas"], res["lws"][0]["floor_ready"]) == (2, 1)


def test_forecast_of_steady_objects_is_empty():
    s = sim_at("T1", 0)
    lws, _, go = sim_tables(s)
    fc = lws_forecast(lws, go)["lws"][0]
    assert fc["flags"] == R.LWSF_DONE and fc["n_steps"] == 0 and fc["cycles"] == 0
    assert (fc["final_partition"], fc["final_replicas"], fc["peak_sts_replicas"], fc["floor_ready"]) == (0, 4, 4, 4)


def test_forecast_layout_matches_header():
    """sizeof / offsetof of the forecast records via a gcc-compiled probe, and the flag values."""
    recs = {"lwse_lws_forecast": R.LWS_FORECAST, "lwse_lws_forecast_step": R.LWS_FORECAST_STEP}
    outf = [f for f, _ in R.LwsForecastOut._fields_]
    flags = ["ROLLING", "WAITING", "DONE", "UNFINISHED", "TRUNCATED", "HELD", "BAD_TABLE", "NOT_FORECAST"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("out_size %zu\\n", sizeof(lwse_lws_forecast_out));',
             'printf("max_cycles %u\\n", LWSE_LWS_FORECAST_MAX_CYCLES);',
             'printf("max_slots %u\\n", LWSE_LWS_FORECAST_MAX_SLOTS);']
    for name, dt in recs.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in dt.names]
    lines += [f'printf("out.{f} %zu\\n", offsetof(lwse_lws_forecast_out, {f}));' for f in outf]
    lines += [f'printf("f.{f} %u\\n", LWSE_LWSF_{f});' for f in flags]
    lines += ["return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = dict(l.split(" ", 1) for l in out.strip().splitlines())
    for name, dt in recs.items():
        assert int(got[name]) == dt.itemsize
        for f in dt.names:
            assert int(got[f"{name}.{f}"]) == dt.fields[f][1], (name, f)
    assert int(got["out_size"]) == C.sizeof(R.LwsForecastOut) == 32
    for f in outf:
        assert int(got[f"out.{f}"]) == getattr(R.LwsForecastOut, f).offset, f
    for f in flags:
        assert int(got[f"f.{f}"]) == getattr(R, f"LWSF_{f}"), f
    assert int(got["max_cycles"]) == R.LWS_FORECAST_MAX_CYCLES
    assert int(got["max_slots"]) == R.LWS_FORECAST_MAX_SLOTS
