"""The rollout what-if's CPU reference (tests/rollout_whatif_ref.py) against the ground truth, without a GPU:

  - T7 (leaderworkerset_test.go:1088-1205) from the checkpoint before its template update;
  - every trace checkpoint whose next action is a spec edit (template, replicas, partition): the what-if of
    that edit against an LwsSim replay from the edited, not yet reconciled state, with the ideal
    StatefulSet of test_lws_forecast.sim_replay (each of its steps landing whole);
  - the availability floor of 16 rollout settings proposed for one at-rest object in one query;
  - IncrementalEncoder.whatif_rollout against what lws_event + flush() then patches;
  - the layout of lwse_rollout_whatif against lwse.h.
"""
import copy
import ctypes as C
import inspect
import itertools
import os
import subprocess
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest

from informer_world import make_world
from lws_b200 import api, encoder, informer
from lws_b200 import records as R
from lws_forecast_ref import trajectory
from rollout_whatif_ref import rollout_whatif
from sim import LwsSim
from test_lws_forecast import checkpoints, oracle_sweep, sim_at, snapshot, sts_step
from traces import TRACES, make_lws

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def world_of(s):
    """The sim's current tables as a resident world (LWS_IRREGULAR dropped, as test_lws_forecast.sim_tables)."""
    t = s.last_tables
    lws = t.lws.copy()
    lws["flags"] &= ~np.uint32(R.LWS_IRREGULAR)
    return SimpleNamespace(lws=lws, groups=t.groups.copy(), pod_state=t.pod_state.copy(), pod_ident=t.pod_ident.copy(),
                           nodes=t.nodes, flags=0)


def proposal_of(s):
    """The row the sim's object encodes to now (what its next sweep would read), LWS_IRREGULAR dropped."""
    updated = s.leader_sts is not None and s.leader_sts.labels.get(api.RevisionKey) != s.rev_key
    item = encoder.LwsItem(lws=s.lws, revision_key=s.rev_key, lws_updated=updated, leader_sts=s.leader_sts)
    rec = encoder.encode_lws([item], s._cluster(), s.topology_key).lws.copy()
    rec["flags"] &= ~np.uint32(R.LWS_IRREGULAR)
    return rec


def edit_of(act):
    """The spec edit an action of tests/traces.py starts with: ("template",), ("replicas", n),
    ("partition", p), ("template+replicas", n), or None."""
    name = act.__qualname__
    free = inspect.getclosurevars(act).nonlocals
    if name == "update":
        return ("template",)
    if name.startswith("replicas.") or name.startswith("replicas_then."):
        return ("replicas", free["n"])
    if name.startswith("partition."):
        return ("partition", free["p"])
    if name.startswith("update_and_replicas."):
        return ("template+replicas", free["n"])
    if name.startswith("seq."):
        return edit_of(free["fns"][0])
    return None


def apply_edit(s, edit):
    """The edit as the API server would hold it, before any controller has reconciled it."""
    if edit[0] in ("template", "template+replicas"):
        s.template_rev += 1
    if edit[0] in ("replicas", "template+replicas"):
        s.lws.replicas = edit[1]
    if edit[0] == "partition":
        s.lws.rollingUpdate.partition = edit[1]


def atomic_replay(s, cap=64):
    """test_lws_forecast.sim_replay with each StatefulSet step landing whole before the controller reconciles.
    (sts_step creates missing groups through create_leader_pods, which settles after every group: after an
    edit that adds groups the controller would reconcile halfway through the step, at a state the ideal
    StatefulSet never shows.)"""
    def step(s):
        s.settle = lambda limit=50: None
        try:
            sts_step(s)
        finally:
            del s.settle
        s.settle()

    rows = []
    for _ in range(cap):
        before = snapshot(s)
        step(s)
        if snapshot(s) == before:
            break
        rows.append(tuple(int(v) for v in s.state()))
    return rows


def spec_edits():
    for name, k in checkpoints():
        steps = TRACES[name][1]
        if k + 1 < len(steps) and edit_of(steps[k + 1][0]) is not None:
            yield name, k


def test_t7_from_before_the_template_update():
    """T7's rollout from the checkpoint before the update: the six rows test_t7_reproduces_the_trace pins,
    derived by hand from Case 2 → Case 5.  The proposal's first pass is Case 2: (partition, replicas) =
    (min(replicas, sts replicas), replicas + maxSurge) = (4, 5), and the first apply creates surge group 4."""
    s = sim_at("T7", 0)
    w = world_of(s)
    s.template_rev += 1
    res = rollout_whatif(w, [0], proposal_of(s))
    assert (int(res["now"][0]["sts_partition"]), int(res["now"][0]["sts_replicas"])) == (4, 5)
    assert trajectory(res, 0) == [(3, 5, 5, 1), (2, 5, 5, 2), (1, 5, 5, 3), (0, 5, 5, 4), (0, 4, 5, 5), (0, 4, 4, 4)]
    fc = res["lws"][0]
    assert fc["flags"] == R.LWSF_ROLLING | R.LWSF_WAITING | R.LWSF_DONE
    assert (fc["peak_sts_replicas"], fc["floor_ready"]) == (5, 4)


def test_the_traces_have_spec_edits():
    kinds = {edit_of(TRACES[n][1][k + 1][0])[0] for n, k in spec_edits()}
    assert kinds == {"template", "replicas", "partition", "template+replicas"}


@pytest.mark.parametrize("name,k", list(spec_edits()))
def test_trace_edit_matches_sim_replay(name, k):
    """now is the controller's first write for the edit; the trajectory is the sim's replay after it."""
    s = sim_at(name, k)
    w = world_of(s)
    apply_edit(s, edit_of(TRACES[name][1][k + 1][0]))
    res = rollout_whatif(w, [0], proposal_of(s))
    now = res["now"][0]
    assert not now["flags"] & R.LOUT_RUP_ERROR
    s.reconcile_lws()
    assert (int(now["sts_partition"]), int(now["sts_replicas"])) == s.state()[:2]
    want = atomic_replay(copy.deepcopy(s))
    assert trajectory(res, 0) == want
    fc = res["lws"][0]
    assert fc["cycles"] == fc["n_steps"] == len(want)
    assert not fc["flags"] & (R.LWSF_UNFINISHED | R.LWSF_NOT_FORECAST | R.LWSF_BAD_TABLE | R.LWSF_TRUNCATED)
    final = want[-1] if want else s.state()
    assert (int(fc["final_partition"]), int(fc["final_replicas"])) == final[:2]
    assert fc["peak_sts_replicas"] >= max([int(now["sts_replicas"])] + [r[1] for r in want])


@pytest.mark.parametrize("replicas", range(1, 7))
def test_settings_grid_respects_max_unavailable(replicas):
    """All 16 (maxUnavailable, maxSurge) pairs in 0..3 as template edits of one at-rest object, one query:
    each proposal with either above 0 finishes with at least replicas - maxUnavailable ready groups
    throughout (test_floor_respects_max_unavailable, reached through proposals)."""
    s = LwsSim(make_lws(dict(replicas=replicas, maxUnavailable=1, maxSurge=0, partition=0, size=2)), oracle_sweep)
    s.bootstrap()
    w = world_of(s)
    s.template_rev += 1
    pairs = list(itertools.product(range(4), range(4)))
    recs = R.aligned_empty(len(pairs), R.LWS_REC)
    for j, (mu, ms) in enumerate(pairs):
        s.lws.rollingUpdate.maxUnavailable, s.lws.rollingUpdate.maxSurge = mu, ms
        recs[j] = proposal_of(s)[0]
    res = rollout_whatif(w, np.zeros(len(pairs), np.uint32), recs)
    for j, (mu, ms) in enumerate(pairs):
        fc = res["lws"][j]
        assert int(fc["step_base"]) == int(res["lws"]["n_steps"][:j].sum())
        if mu or ms:
            assert fc["flags"] & R.LWSF_DONE and not fc["flags"] & R.LWSF_UNFINISHED, (mu, ms)
            assert (fc["final_partition"], fc["final_replicas"]) == (0, replicas)
            assert fc["floor_ready"] >= replicas - min(mu, replicas), (mu, ms)


def test_informer_proposal_is_the_next_patch():
    """whatif_rollout(item) is the LWS row lws_event(item) + flush() then patches, and changes nothing in the
    encoder until then."""
    items, cluster = make_world(5)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    checked = 0
    for key in sorted(enc.slots)[:6]:
        it = enc.items[key]
        lws = copy.deepcopy(it.lws)
        lws.replicas += 1
        lws.rollingUpdate.maxSurge = 2
        item = encoder.LwsItem(lws=lws, revision_key="rev-2", lws_updated=True)
        before = [a.copy() for a in enc.full_tables()]
        dirty = set(enc.dirty)
        row, rec = enc.whatif_rollout(item)
        assert [a.tobytes() for a in enc.full_tables()] == [a.tobytes() for a in before]
        assert enc.dirty == dirty and item.leader_sts is None
        enc.lws_event("MODIFIED", item)
        patches = enc.flush()
        segs = [(rows, vals) for t, rows, vals in patches.segments if t == R.TABLE_LWS]
        assert len(segs) == 1 and segs[0][0].tolist() == [row]
        assert segs[0][1][0].tobytes() == rec.tobytes()
        assert rec["flags"] & R.LWS_UPDATED and rec["replicas"] == lws.replicas
        checked += 1
    assert checked == 6
    with pytest.raises(KeyError):
        enc.whatif_rollout(encoder.LwsItem(lws=api.LeaderWorkerSet(name="absent", namespace="ns-0"), revision_key="r"))


def test_rollout_whatif_layout_matches_header():
    """sizeof / offsetof of lwse_rollout_whatif via a gcc-compiled probe."""
    fields = [f for f, _ in R.RolloutWhatIf._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("size %zu\\n", sizeof(lwse_rollout_whatif));']
    lines += [f'printf("{f} %zu\\n", offsetof(lwse_rollout_whatif, {f}));' for f in fields]
    lines += ["return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = dict(l.split(" ", 1) for l in out.strip().splitlines())
    assert int(got["size"]) == C.sizeof(R.RolloutWhatIf) == 64
    for f in fields:
        assert int(got[f]) == getattr(R.RolloutWhatIf, f).offset, f
