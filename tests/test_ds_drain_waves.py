"""DS drain waves without a GPU: the plan from restart pairs and per-row caps (``ds_drain_waves_ref.plan_fast``)
equals the plan by its definition (``plan_literal``, every probe the two set-form references) on seeded worlds with
slack, for both scopes, four key orders, caps 1, 2 and 64 and each constraint mask; the LWS-floor-only plan keeps
the drain waves plan; and the two mutations the exactness argument rules out give wrong plans."""
import functools

import numpy as np
import pytest

from drain_budget_ref import drain_budget_cost_ref
from drain_waves_ref import plan_fast as lws_plan_fast
from ds_drain_waves_ref import (CONSTRAINTS, DEFAULT, ds_cost_per_ds, ds_waves_edges_world, orders, plan_fast, plan_literal,
                                slack_world)
from ds_drain_ref import ds_drain_cost_ref, overlap_worlds
from lws_b200 import records as R

WORLDS = {"mixed": dict(n_ds=30, n_nodes=96, seed=3), "pct100": dict(n_ds=30, n_nodes=96, seed=5, mu=(100, True)),
          "mu1": dict(n_ds=20, n_nodes=128, seed=7, mu=(1, False)), "mu2": dict(n_ds=24, n_nodes=96, seed=9, mu=(2, False)),
          "pct50": dict(n_ds=24, n_nodes=96, seed=13, mu=(50, True))}


@functools.lru_cache(maxsize=None)
def world(name):
    return slack_world(**WORLDS[name])


def key_orders(w, by_domain):
    lws_out, base_out = w.base
    bcost = drain_budget_cost_ref(w.lws, lws_out, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, base_out,
                                  by_domain)
    return orders(np.arange(len(bcost)), bcost)


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2]


@pytest.mark.parametrize("name", sorted(WORLDS))
@pytest.mark.parametrize("by_domain", [False, True])
def test_fast_equals_literal(name, by_domain):
    w = world(name)
    for oname, ids in key_orders(w, by_domain).items():
        for c in CONSTRAINTS:
            for mw in (1, 2, 64):
                if not by_domain and oname != "by_cost" and mw != 64:
                    continue  # (the literal plan probes the oracle per key and wave: node scope at one cap per order)
                got = plan_fast(w, ids, by_domain, mw, c)
                assert same(got, plan_literal(w, ids, by_domain, mw, c)), (name, oname, c, mw)


def test_worlds_exercise_the_plan():
    """The seeded worlds plan keys into several waves, hit the cap, and the DS verdicts decide where the LWS floors
    leave room."""
    seen = {"waves": 0, "no_wave": 0, "ds_only": 0, "service_unkept": 0}
    for name in WORLDS:
        w = world(name)
        for by_domain in (False, True):
            ids = key_orders(w, by_domain)["by_cost"]
            lws_only = plan_fast(w, ids, by_domain, 64, R.DSW_LWS_FLOOR)
            dflt = plan_fast(w, ids, by_domain, 64, DEFAULT)
            seen["waves"] = max(seen["waves"], dflt[2]["n_waves"])
            seen["no_wave"] += plan_fast(w, ids, by_domain, 1, DEFAULT)[2]["n_no_wave"]
            a = dflt[0]["alone"].astype(np.int64)
            seen["ds_only"] += int((((a & DEFAULT) != 0) & ((a & R.DSW_LWS_FLOOR) == 0)).sum())
            seen["service_unkept"] += int(lws_only[1]["ds_service_lost"].sum())
            assert not dflt[1]["ds_service_lost"].any() and not dflt[1]["ds_old_service_lost"].any()
            assert not dflt[1]["lws_breached"].any()
    assert seen["waves"] >= 2 and seen["no_wave"] > 0 and seen["ds_only"] > 0 and seen["service_unkept"] > 0, seen


@pytest.mark.parametrize("name", sorted(WORLDS))
def test_lws_floor_only_is_the_drain_waves_plan(name):
    """With LWS_FLOOR alone the plan is lwse_resident_drain_waves': same wave, status and shared wave columns."""
    w = world(name)
    lws_out, base_out = w.base
    for by_domain in (False, True):
        ids = key_orders(w, by_domain)["random"]
        for mw in (2, 64):
            k, v, t = plan_fast(w, ids, by_domain, mw, R.DSW_LWS_FLOOR)
            lk, lv, lt = lws_plan_fast(w.lws, lws_out, w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains,
                                       base_out, ids, by_domain, mw)
            assert t == lt
            for f in ("id", "wave", "status", "groups_restarted", "ready_restarted", "lws_touched", "lws_breached"):
                assert np.array_equal(k[f], lk[f]), f
            for f in lv.dtype.names:
                if f != "reserved":
                    assert np.array_equal(v[f], lv[f]), f


def test_alone_bits_decide_breaches_alone():
    for name in WORLDS:
        w = world(name)
        for c in CONSTRAINTS:
            k, _, _ = plan_fast(w, np.arange(len(w.nodes)), False, 64, c)
            assert np.array_equal(k["status"] == R.DRAINW_BREACHES_ALONE, (k["alone"] & c) != 0), (name, c)


@functools.lru_cache(maxsize=None)
def edges():
    return ds_waves_edges_world()


def at(ids, keys, k):
    return keys[list(ids).index(k)]


@pytest.mark.parametrize("by_domain", [False, True])
def test_edges_fast_equals_literal(by_domain):
    w, ids, _ = edges()
    for c in CONSTRAINTS:
        for mw in (2, 64):
            assert same(plan_fast(w, ids, by_domain, mw, c), plan_literal(w, ids, by_domain, mw, c)), (c, mw)


def test_edges_each_case_on_its_side():
    w, ids, notes = edges()
    ch = notes["children"]
    L = ready_targets(w)
    assert ch["unevaluated"] in L and ch["fb_excluded"] not in L
    alone = {lab: [int(at(ids, plan_fast(w, ids, False, 64, R.DSW_ALL)[0], k)["alone"]) for k in notes[lab]]
             for lab in notes if lab not in ("children", "cap")}
    assert alone["service_ready1"] == [R.DSW_DS_SERVICE] and alone["unevaluated"] == [R.DSW_DS_SERVICE]
    assert alone["stable"] == [R.DSW_DS_STALL] and alone["old_rev"] == [R.DSW_DS_OLD_SERVICE]
    assert alone["below"] == [R.DSW_LWS_FLOOR] and alone["ready2"] == [0, 0] and alone["shared"] == [0, 0]
    for lab in ("removed", "bad_table", "fb_unlinked", "fb_stale_uid", "fb_past_table", "fb_excluded", "fb_not_exists"):
        assert alone[lab] == [0], lab
    keys = plan_fast(w, ids, False, 64, R.DSW_ALL)[0]
    cost = ds_cost_per_ds(w)
    assert cost["rows_zeroed"][notes["removed"][0]] == 1 and cost["ds_touched"][notes["removed"][0]] == 1
    for lab in ("bad_table", "fb_unlinked", "fb_stale_uid", "fb_past_table", "fb_excluded", "fb_not_exists"):
        assert cost["ds_touched"][notes[lab][0]] == 0, lab
    assert cost["ds_touched"][notes["shared"][0]] == 2
    # ready 2 (and the shared child): the second key opens a wave of its own under a service cap of 1
    for lab in ("ready2", "shared"):
        a, b = (at(ids, keys, k) for k in notes[lab])
        assert a["status"] == b["status"] == R.DRAINW_PLANNED and a["wave"] != b["wave"], lab
    # below its floor: the LWS floor breaches alone, a DS-only plan places the key
    k_svc = plan_fast(w, ids, False, 64, R.DSW_DS_SERVICE)[0]
    assert at(ids, k_svc, notes["below"][0])["status"] == R.DRAINW_PLANNED
    assert at(ids, k_svc, notes["unevaluated"][0])["status"] == R.DRAINW_BREACHES_ALONE
    # 65 keys on a child of slack 1: waves 0-63, then NO_WAVE
    st = [(int(at(ids, keys, k)["status"]), int(at(ids, keys, k)["wave"])) for k in notes["cap"]]
    assert st[:64] == [(R.DRAINW_PLANNED, v) for v in range(64)] and st[64] == (R.DRAINW_NO_WAVE, R.NONE)


def ready_targets(w):
    from ds_drain_ref import ready_columns

    L = ready_columns(w, np.zeros(len(w.lws), np.int64))[0]
    return set(L[L >= 0].tolist())


def test_edges_overlapping_ranges():
    """Two more DS over the range of the first linked DS (shared) plan as two more DS with copies of those rows
    (copied), whose ranges are disjoint and where the literal plan applies; the per-DS restatement of the per-key
    form counts a shared row once per DS."""
    w, ids, notes = edges()
    shared, copied = overlap_worlds(w, 2)  # (copies of the DS of `ready2`)
    assert ds_cost_per_ds(copied).tobytes() == ds_drain_cost_ref(copied).tobytes()
    assert ds_cost_per_ds(shared).tobytes() == ds_cost_per_ds(copied).tobytes()
    for c in (R.DSW_LWS_FLOOR, R.DSW_DS_SERVICE, R.DSW_ALL):
        got = plan_fast(shared, ids, False, 64, c)
        assert same(got, plan_fast(copied, ids, False, 64, c)), c
        assert same(got, plan_literal(copied, ids, False, 64, c)), c
        assert int(at(ids, got[0], notes["ready2"][0])["ds_touched"]) == 3


@pytest.mark.parametrize("mutation", ["evaluated_only", "no_gates"])
def test_mutations_give_wrong_plans(mutation):
    """Binding only the pairs of EVALUATED rows (the LWS plan's rule), or capping every linked spec row whatever
    its DS's flags, gives a plan the definition refutes on the edges world (re-swept and consistent)."""
    w, ids, notes = edges()
    kw = {"linked_bind": False} if mutation == "evaluated_only" else {"gates": False}
    wrong = 0
    for c in (R.DSW_DS_SERVICE, R.DSW_DS_STALL, R.DSW_ALL):
        good = plan_fast(w, ids, False, 64, c)
        assert same(good, plan_literal(w, ids, False, 64, c)), c
        wrong += not same(good, plan_fast(w, ids, False, 64, c, **kw))
    assert wrong > 0
    if mutation == "evaluated_only":
        k = plan_fast(w, ids, False, 64, R.DSW_DS_SERVICE, linked_bind=False)[0]
        assert at(ids, k, notes["unevaluated"][0])["status"] == R.DRAINW_PLANNED


def test_ds_drain_waves_report():
    """The informer's names: waves of node names, unplanned keys with their status and alone verdicts."""
    from lws_b200 import informer

    enc = informer.IncrementalEncoder.__new__(informer.IncrementalEncoder)
    enc.node_index = {"n0": 0, "n1": 1, "n2": 2, "n3": 3}
    keys = np.zeros(4, R.DS_DRAIN_WAVE_KEY)
    keys["id"] = [3, 0, 2, 1]
    keys["status"] = [R.DRAINW_PLANNED, R.DRAINW_BREACHES_ALONE, R.DRAINW_PLANNED, R.DRAINW_NO_WAVE]
    keys["wave"] = [1, R.NONE, 0, R.NONE]
    keys["alone"] = [0, R.DSW_DS_SERVICE | R.DSW_LWS_FLOOR, 0, 0]
    rep = enc.ds_drain_waves_report({"keys": keys, "waves": np.zeros(2, R.DS_DRAIN_WAVE)}, "nodes")
    assert rep == {"waves": [["n2"], ["n3"]],
                   "unplanned": [("n0", "breaches_alone", ["lws_floor", "ds_service"]), ("n1", "no_wave", [])]}
