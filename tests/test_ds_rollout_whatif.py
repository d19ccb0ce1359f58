"""The DS rollout what-if's CPU reference (tests/ds_rollout_whatif_ref.py) and the DS encoder's proposals, without
a GPU:

  - a hand-derived template bump of a steady two-role DS;
  - the 22 exact ComputeAllSteps sequences (tests/golden/planner_sequences.json), each proposed as a template
    edit with the case's targets and rollout settings on a DS steady at the case's source;
  - ``DsIncrementalEncoder.whatif_rollout`` on seeded watch-event worlds: the proposed rows equal ``encode_ds`` of
    the edited object with the retired revision's children last, the encoder does not change, and an edit of the
    role set is refused;
  - DsSim replays of the edited objects, which agree with the what-if trajectory;
  - the ctypes record against the header.
"""
import copy
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ds_rollout_whatif_ref import M, ds_rollout_whatif, proposed, trajectory_of
from ds_world import DsWorld
from lws_b200 import api, ds_informer, encoder
from lws_b200 import records as R
from test_ds_forecast import sim_replay

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "planner_sequences.json")))["cases"]


def answer(enc, props, q_roles=None, **kw):
    ds, roles, revroles = enc.tables()
    return ds_rollout_whatif(ds, roles, revroles, enc.links, props, q_roles, **kw)


def one(enc, ds, revision):
    p, roles = enc.whatif_rollout(ds, revision)
    return np.array([p], R.DS_PROPOSAL), roles.copy()


def steady(targets, cfgs, rev="A"):
    """DS "svc" steady at revision ``rev``: prefill and decode at ``targets`` replicas, every child ready."""
    roles = [api.DisaggregatedRoleSpec(n, t, c) for n, t, c in zip(["prefill", "decode"], targets, cfgs)]
    kids = [api.ChildLWS(r.name, rev, t, t, 1.0) for r, t in zip(roles, targets)]
    return encoder.DsItem(api.DisaggregatedSet("svc", roles=roles), rev, kids)


def test_hand_derived_template_bump():
    """prefill 3 and decode 2, maxSurge 1, maxUnavailable 0, steady at A: a new template."""
    cfg = api.RollingUpdateConfiguration(maxSurge=1, maxUnavailable=0)
    item = steady([3, 2], [cfg, cfg])
    enc = ds_informer.DsIncrementalEncoder([item])
    props, roles = one(enc, item.ds, "B")
    assert int(props[0]["flags"]) == R.DSP_NEW_REVISION
    res = answer(enc, props, roles)
    now = res["now"][0]
    assert int(now["flags"]) == R.DOUT_ROLLING | R.DOUT_INIT and int(now["ready_revs"]) == 1
    fc = res["ds"][0]
    assert int(fc["flags"]) == R.DSF_ROLLING | R.DSF_DONE and int(fc["cycles"]) == 9 and int(fc["n_steps"]) == 7
    fr = res["roles"]
    assert [tuple(int(fr[j][k]) for k in ("peak_replicas", "floor_available", "final_old", "final_new"))
            for j in range(2)] == [(4, 3, 0, 3), (3, 2, 0, 2)]
    assert trajectory_of(res, 0, 2) == [[(3, 1), (2, 1)], [(2, 1), (2, 1)], [(2, 1), (1, 1)], [(2, 2), (1, 2)],
                                         [(1, 2), (1, 2)], [(1, 3), (1, 2)], [(0, 3), (0, 2)]]
    assert (fr[2:] == np.zeros(M - 2, R.DS_FORECAST_ROLE)).all() and (res["now_roles"][2:].view(np.int64) == 0).all()
    # the same tables are encode_ds of the object with target B, byte for byte
    t = encoder.encode_ds([encoder.DsItem(item.ds, "B", item.children)])
    P, Pr, Prr, _, bad = proposed(*enc.tables(), _none(enc), props, roles)
    assert not bad[0] and P.tobytes() == t.ds.tobytes() and Prr.tobytes() == t.revroles.tobytes()
    assert Pr[:2].tobytes() == t.roles.tobytes()
    named = enc.whatif_of(res, 0, "default", "svc")
    assert named["roles"]["decode"]["trajectory"][-1] == (0, 2) and named["roles"]["prefill"]["next"] == (-1, -1)  # INIT: no planner step yet


def _none(enc):
    links = R.aligned_empty(len(enc.revroles), R.DS_LINK)
    links["lws_row"] = R.NONE
    return links


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden_sequences(case):
    """Steady at the case's source (every child ready), then the case's targets and settings with a new template."""
    n = len(case["source"])
    old = [api.DisaggregatedRoleSpec(f"r{i}", s) for i, s in enumerate(case["source"])]
    item = encoder.DsItem(api.DisaggregatedSet("g", roles=old), "A",
                          [api.ChildLWS(f"r{i}", "A", s, s, 1.0) for i, s in enumerate(case["source"])])
    enc = ds_informer.DsIncrementalEncoder([item])
    edit = api.DisaggregatedSet("g", roles=[
        api.DisaggregatedRoleSpec(f"r{i}", case["target"][i], api.RollingUpdateConfiguration(maxSurge=ms, maxUnavailable=mu))
        for i, (ms, mu) in enumerate(case["config"])])
    props, roles = one(enc, edit, "B")
    assert int(props[0]["flags"]) == R.DSP_NEW_REVISION | R.DSP_ROLES
    res = answer(enc, props, roles)
    fc = res["ds"][0]
    if not any(case["source"]):  # reconcileSimple scales to target in one reconcile: no rollout
        assert fc["flags"] == 0 and fc["cycles"] == 0 and fc["n_steps"] == 0
        return
    want = [[(o[i], nw[i]) for i in range(n)] for o, nw in case["steps"][1:]]
    assert trajectory_of(res, 0, n) == want
    assert fc["flags"] == R.DSF_ROLLING | R.DSF_DONE


def _edits(rng, ds):
    """Edits of one DS object that keep its roles: new replicas and new rollout settings per role."""
    out = copy.deepcopy(ds)
    for r in out.roles:
        if rng.random() < 0.5:
            r.replicas = None if rng.random() < 0.1 else int(rng.integers(0, 7))
        if rng.random() < 0.5:
            r.rollingUpdate = (None if rng.random() < 0.2 else
                               api.RollingUpdateConfiguration(maxSurge=[0, 1, 3, "50%"][int(rng.integers(0, 4))],
                                                              maxUnavailable=[0, 1, "25%"][int(rng.integers(0, 3))]))
    return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_encoder_proposals_equal_encode_ds(seed):
    """Every DS of a watch-event world after some events, with a template edit, a scale / settings edit, or both:
    the proposed rows are encode_ds of the edited object (retired revision's children last), up to role_base and
    rev_base; whatif_rollout changes nothing in the encoder."""
    w = DsWorld(seed)
    enc = ds_informer.DsIncrementalEncoder(w.initial_items(), spare=1.0)
    for _ in range(25):
        w.step(enc)
    enc.flush()
    rng = np.random.default_rng(seed)
    before = ({k: copy.deepcopy(v) for k, v in enc.slots.items()}, set(enc.dirty),
              [t.copy() for t in enc.tables()])
    props, q, wants = [], [], []
    for key in sorted(enc.slots):
        ds, rev = enc.items[key]
        for kind in range(3):
            edit = ds if kind == 0 else _edits(rng, ds)
            new_rev = rev if kind == 1 else f"{rev}-next"
            try:
                p, roles = enc.whatif_rollout(edit, new_rev)
            except ValueError:
                continue
            kids = list(enc.children.get(key, {}).values())
            kids = [c for c in kids if c.revision != rev] + [c for c in kids if c.revision == rev]
            wants.append(encoder.encode_ds([encoder.DsItem(edit, new_rev, kids)]))
            props.append(p)
            q.append(roles)
    assert len(props) >= 12
    props, q = np.array(props, R.DS_PROPOSAL), np.concatenate(q)
    assert ((props["flags"] & R.DSP_NEW_REVISION) != 0).any() and ((props["flags"] & R.DSP_ROLES) != 0).any()
    P, Pr, Prr, _, bad = proposed(*enc.tables(), _none(enc), props, q)
    for i, t in enumerate(wants):
        n = len(t.roles)
        assert not bad[i]
        a, b = P[i].copy(), t.ds[0].copy()
        a["role_base"] = a["rev_base"] = b["role_base"] = b["rev_base"] = 0
        assert a.tobytes() == b.tobytes(), i
        assert Pr[i * M: i * M + n].tobytes() == t.roles.tobytes(), i
        vb = int(P[i]["rev_base"])
        assert Prr[vb: vb + len(t.revroles)].tobytes() == t.revroles.tobytes(), i
    slots, dirty, tables = before
    assert enc.slots == slots and enc.dirty == dirty
    assert all(a.tobytes() == b.tobytes() for a, b in zip(enc.tables(), tables))


def test_role_set_change_is_refused():
    cfg = api.RollingUpdateConfiguration(maxSurge=1, maxUnavailable=0)
    item = steady([3, 2], [cfg, cfg])
    enc = ds_informer.DsIncrementalEncoder([item])
    renamed = copy.deepcopy(item.ds)
    renamed.roles[1].name = "decoder"
    added = copy.deepcopy(item.ds)
    added.roles.append(api.DisaggregatedRoleSpec("router", 1))
    # the last spec role dropped while its children remain: allRoleNames is still [prefill, decode], decode now a
    # removed role
    dropped = copy.deepcopy(item.ds)
    dropped.roles = dropped.roles[:1]
    assert encoder.encode_ds([encoder.DsItem(dropped, "B", item.children)]).role_names[0] == ["prefill", "decode"]
    for edit in (renamed, added, dropped):
        for rev in ("A", "B"):
            with pytest.raises(ValueError):
                enc.whatif_rollout(edit, rev)
    with pytest.raises(KeyError):
        enc.whatif_rollout(api.DisaggregatedSet("other", roles=item.ds.roles), "B")
    # a removed role taken back into the spec: decode has children only in old revision A, the target is B
    kids = [api.ChildLWS("prefill", "A", 3, 3, 1.0), api.ChildLWS("decode", "A", 2, 2, 1.0),
            api.ChildLWS("prefill", "B", 3, 3, 2.0)]
    enc = ds_informer.DsIncrementalEncoder([encoder.DsItem(dropped, "B", kids)])
    assert enc.role_names(enc.ds_row("default", "svc")) == ["prefill", "decode"]
    assert int(enc.ds[enc.ds_row("default", "svc")]["n_spec_roles"]) == 1
    for rev in ("B", "C"):
        with pytest.raises(ValueError):
            enc.whatif_rollout(item.ds, rev)
    enc.whatif_rollout(dropped, "C")  # the same split: accepted


def _sim_items(seed):
    """Mid-rollout DS objects with distinct creation stamps per revision, and edits of them."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(12):
        n = int(rng.integers(1, 4))
        roles = [api.DisaggregatedRoleSpec(f"r{i}", int(rng.integers(1, 6)),
                                           api.RollingUpdateConfiguration(maxSurge=int(rng.integers(1, 3)),
                                                                          maxUnavailable=int(rng.integers(0, 2))))
                 for i in range(n)]
        ds = api.DisaggregatedSet(f"d{k}", roles=roles)
        kids, stamp = [], 1.0
        revs = ["v0", "v1", "v2"][: int(rng.integers(1, 4))]
        for j, rev in enumerate(revs):
            stamp += 1.0
            for r in roles:
                rep = int(rng.integers(0, 5)) if j < len(revs) - 1 else int(r.replicas)
                kids.append(api.ChildLWS(r.name, rev, rep, rep, stamp))
        out.append((encoder.DsItem(ds, revs[-1], kids), _edits(rng, ds)))
    return out


@pytest.mark.parametrize("seed", [5, 6])
def test_sim_replay_agrees(seed):
    """DsSim plays the edited object (every child ready before each reconcile); its steps are the what-if
    trajectory, and its finals, peaks and floors the forecast's."""
    for item, edit in _sim_items(seed):
        enc = ds_informer.DsIncrementalEncoder([item])
        props, roles = one(enc, edit, "next")
        res = answer(enc, props, roles)
        fc = res["ds"][0]
        n = len(item.ds.roles)
        kids = copy.deepcopy(item.children)
        kids = [c for c in kids if c.revision != item.revision] + [c for c in kids if c.revision == item.revision]
        steps, cycles, final, stopped, peak, floor = sim_replay(encoder.DsItem(edit, "next", kids))
        assert fc["flags"] & R.DSF_ROLLING and stopped
        assert trajectory_of(res, 0, n) == steps and int(fc["cycles"]) == cycles
        fr = res["roles"][:n]
        assert [(int(x["final_old"]), int(x["final_new"])) for x in fr] == final
        assert [int(x["peak_replicas"]) for x in fr] == peak and [int(x["floor_available"]) for x in fr] == floor


def test_limits_and_bad_rows():
    """V = 31 is valid after a bump and V = 32 is BAD; a DS without a target revision's children keeps V; a row
    past the limits is BAD whatever the flags; the offsets run over the proposals in order."""
    from ds_limits_world import _empty, _put, assemble

    items = []
    for V, has_new in ((31, True), (32, True), (32, False), (2, True)):
        x = _empty(2, 0, V, has_new)
        for r in range(V + 1):
            for i in range(2):
                if r < V or has_new:
                    _put(x, r, i, 1 if r == V else 0, stamp=r + 1)
        items.append(x)
    ds, roles, rr = assemble(items)
    ds["n_spec_roles"][3] = 3  # past the limits
    props = np.zeros(8, R.DS_PROPOSAL)
    props["ds"] = [0, 0, 1, 1, 2, 2, 3, 3]
    props["flags"] = [0, R.DSP_NEW_REVISION] * 4
    res = ds_rollout_whatif(ds, roles, rr, None, props)
    assert res["bad"].tolist() == [False, False, False, True, False, False, True, True]
    P = proposed(ds, roles, rr, _none_n(len(rr)), props)[0]
    assert P["n_old_revs"].tolist()[:6] == [31, 32, 32, 32, 32, 32]
    assert (res["now"]["flags"][res["bad"]] == R.DOUT_BAD_TABLE).all()
    assert (res["ds"]["flags"][res["bad"]] == R.DSF_BAD_TABLE).all()
    assert (res["ds"]["flags"][~res["bad"]] & R.DSF_BAD_TABLE == 0).all()
    rows = res["ds"]["n_steps"].astype(np.int64) * np.where(res["bad"], 0, 2)
    assert res["ds"]["step_base"].tolist() == (np.cumsum(rows) - rows).tolist()


def _none_n(n):
    links = R.aligned_empty(n, R.DS_LINK)
    links["lws_row"] = R.NONE
    return links


def test_record_matches_header():
    """sizeof and offsets of lwse_ds_proposal and lwse_ds_rollout_whatif against the ctypes mirrors, and the cap."""
    src = "\n".join([
        "#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/lwse.h"', "int main(){",
        'printf("%zu %zu %zu\\n", sizeof(lwse_ds_proposal), offsetof(lwse_ds_proposal, flags), sizeof(lwse_ds_rollout_whatif));',
        'printf("%zu %zu %zu %zu\\n", offsetof(lwse_ds_rollout_whatif, n), offsetof(lwse_ds_rollout_whatif, now),'
        ' offsetof(lwse_ds_rollout_whatif, now_roles), offsetof(lwse_ds_rollout_whatif, fc));',
        'printf("%u %u %u\\n", LWSE_DSP_NEW_REVISION, LWSE_DSP_ROLES, LWSE_DS_WHATIF_MAX_PROPOSALS);', "return 0;}"])
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "p.c"), "w").write(src)
        subprocess.run(["gcc", "-o", os.path.join(d, "p"), os.path.join(d, "p.c")], check=True)
        out = subprocess.run([os.path.join(d, "p")], check=True, capture_output=True, text=True).stdout.split()
    W = R.DsRolloutWhatIf
    assert [int(x) for x in out] == [R.DS_PROPOSAL.itemsize, R.DS_PROPOSAL.fields["flags"][1], C.sizeof(W),
                                     W.n.offset, W.now.offset, W.now_roles.offset, W.fc.offset,
                                     R.DSP_NEW_REVISION, R.DSP_ROLES, R.DS_WHATIF_MAX_PROPOSALS]
    assert R.DS_WHATIF_MAX_PROPOSALS == 13_015_052
