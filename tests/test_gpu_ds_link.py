"""Linked DS ticks (LWSE_TABLE_DS_LINKS): revision-role rows linked to resident child LeaderWorkerSets take
their ready counts from the LWS tick on the device.  Every check compares bit for bit with
``oracle.sweep_ds`` over revision-role rows whose ready values are substituted by the rule
(``ds_link_world.linked_revroles``), computed from the test's host copy of the resident LWS tables and
``oracle.sweep_lws`` over them; ``ds_resident_tick_info`` shows which rows took the LWS value."""
import numpy as np
import pytest

import oracle
from ds_link_world import child_lws_tables, flip_ready, linked_revroles, none_links
from lws_b200 import api, churn, synth
from lws_b200 import records as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def _same_mirrors(res, want, where=""):
    for k, name in enumerate(("ds_out", "role_out", "revrole_out")):
        assert res[name].tobytes() == want[k].tobytes(), f"{where}: {name} differs from the oracle"


def _changed_ds(before, after, ds):
    n = ds["n_roles"].astype(np.int64)
    role_owner = np.repeat(np.arange(len(ds)), n)
    rr_owner = np.repeat(np.arange(len(ds)), (ds["n_old_revs"].astype(np.int64) + 1) * n)
    ch = (before[0].view(np.uint8).reshape(len(ds), -1) != after[0].view(np.uint8).reshape(len(ds), -1)).any(1)
    ch[role_owner[before[1].view(np.uint64) != after[1].view(np.uint64)]] = True
    ch[rr_owner[before[2] != after[2]]] = True
    return np.flatnonzero(ch).astype(np.uint32)


def _expect(ds, roles, rr, links, lws=None, lws_out=None):
    sub, took, fell = linked_revroles(rr, links, lws, lws_out)
    return oracle.sweep_ds(ds, roles, sub), took, fell


def test_c4_linked_ticks_follow_leader_readiness(engine):
    """50 000 DS, every existing revision-role row linked to a resident size-1 child; LWS ticks flip
    leader-pod readiness of 1 % of the groups, each followed by a DS tick with no patches at all."""
    d = synth.make_ds(50_000, (2,), seed=21)
    rng = np.random.default_rng(8)
    lws, groups, pst, pid, links = child_lws_tables(d.revroles, rng)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick(()))
    engine.ds_resident_load(d.ds, d.roles, d.revroles)
    assert not engine.ds_resident_tick_info()["linked"]
    res = engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)])
    lo = oracle.sweep_lws(lws, groups, pst, pid)[0]
    want, took, fell = _expect(d.ds, d.roles, d.revroles, links, lws, lo)
    _same_mirrors(res, want, "first linked tick")
    info = engine.ds_resident_tick_info()
    n_exist = int((d.revroles["flags"] & R.RR_EXISTS != 0).sum())
    assert info["linked"] and (info["rows_from_lws"], info["rows_fallback"]) == (took, fell) == (n_exist, 0)
    assert info["lws_ticks"] >= 1
    moved = 0
    for k in range(12):
        rows, v = flip_ready(groups, rng, 0.01)
        groups[rows] = v
        engine.resident_tick(engine.make_tick([(R.TABLE_GROUPS, rows, v)]))
        lo = oracle.sweep_lws(lws, groups, pst, pid)[0]
        got = engine.ds_resident_tick()
        now, took, fell = _expect(d.ds, d.roles, d.revroles, links, lws, lo)
        assert np.array_equal(np.sort(got["rows"]), _changed_ds(want, now, d.ds)), f"tick {k}: changed DS"
        _same_mirrors(got, now, f"tick {k}")
        info = engine.ds_resident_tick_info()
        assert (info["rows_from_lws"], info["rows_fallback"]) == (took, fell), k
        moved += len(got["rows"])
        want = now
    assert moved > 0


def test_ds_tick_between_submit_and_wait_sees_the_submitted_lws_tick(engine):
    """C3 pipelined LWS ticks with a linked C4 DS tick between each submit(k) and wait(k-1): the DS tick
    reads tick k's results; the LWS changed rows are those of a run without DS ticks, and steady LWS
    ticks still replay their graph."""
    t = synth.make("C3-steady", seed=41)
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    d = synth.make_ds(50_000, (2,), seed=3)
    rng = np.random.default_rng(6)
    links = none_links(len(d.revroles))
    ex = np.flatnonzero(d.revroles["flags"] & R.RR_EXISTS)
    at = rng.integers(0, len(t.lws), size=len(ex))
    links["lws_row"][ex] = at
    links["lws_uid_hash"][ex] = t.lws["uid_hash"][at]

    def run(with_ds):
        engine.upload_nodes(t.nodes, t.n_domains)
        engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        engine.resident_place_load(reqs, t.n_namespaces)
        engine.resident_tick(engine.make_tick((), flags))
        plan = churn.make_plan(t, reqs, engine.resident_place_outputs(), 0.01, 0.01, n_sets=6, seed=4)
        ticks = churn.ArenaPlan(engine, plan, flags).ticks
        pst, grp, rq = t.pod_state.copy(), t.groups.copy(), reqs.copy()
        if with_ds:
            engine.ds_resident_load(d.ds, d.roles, d.revroles)
            engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)])
        out, graphs = [], []
        n = 16
        engine.resident_tick_submit(ticks[0])
        churn.apply_to_mirror(plan[0], pst, grp, rq)
        for k in range(1, n + 1):
            if k < n:
                engine.resident_tick_submit(ticks[k % len(ticks)])
                churn.apply_to_mirror(plan[k % len(plan)], pst, grp, rq)
                graphs.append(engine.resident_tick_info()["graph"])
            if with_ds:
                res = engine.ds_resident_tick()
                lo = oracle.sweep_lws(t.lws, grp, pst, t.pod_ident, t.nodes, flags=t.flags)[0]
                want, took, fell = _expect(d.ds, d.roles, d.revroles, links, t.lws, lo)
                _same_mirrors(res, want, f"step {k}")
                info = engine.ds_resident_tick_info()
                assert (info["rows_from_lws"], info["rows_fallback"]) == (took, fell), k
                assert took > 0
            r = engine.resident_tick_wait()
            out.append(tuple(np.sort(r[name].copy()).tobytes() for name in ("lws_rows", "group_rows", "place_rows")))
        return out, graphs

    base, base_graphs = run(False)
    mixed, graphs = run(True)
    assert mixed == base
    assert graphs == base_graphs and all(graphs[6:]), (base_graphs, graphs)


def test_each_fallback_path(engine):
    """Every condition of the rule fails once, and ds_resident_tick_info shows the rows that fell back."""
    from lws_b200.engine import Engine

    d = synth.make_ds(3000, (2, 3), seed=12)
    ds, roles, rr = d.ds, d.roles, d.revroles
    rng = np.random.default_rng(4)
    lws, groups, pst, pid, links = child_lws_tables(rr, rng)
    n_linked = int((links["lws_row"] != R.NONE).sum())

    def tick(eng, segs=(), lws_tables=None, where=""):
        res = eng.ds_resident_tick(list(segs))
        lo = oracle.sweep_lws(*lws_tables)[0] if lws_tables is not None else None
        want, took, fell = _expect(ds, roles, rr, links, lws_tables[0] if lws_tables else None, lo)
        _same_mirrors(res, want, where)
        info = eng.ds_resident_tick_info()
        assert info["linked"] and (info["rows_from_lws"], info["rows_fallback"]) == (took, fell), where
        return took, fell

    # no LWS tables at all
    fresh = Engine(0)
    try:
        fresh.ds_resident_load(ds, roles, rr)
        assert tick(fresh, [(R.TABLE_DS_LINKS, 0, links, True)], None, "no LWS tables") == (0, n_linked)
        # LWS tables loaded, no sweep yet: the output rows are all-ones
        fresh.resident_load(lws, groups, pst, pid)
        assert tick(fresh, (), None, "after load, before a sweep") == (0, n_linked)
        fresh.resident_tick(fresh.make_tick(()))
        took, fell = tick(fresh, (), (lws, groups, pst, pid), "after a sweep")
        assert (took, fell) == (n_linked, 0)
    finally:
        fresh.close()

    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick(()))
    engine.ds_resident_load(ds, roles, rr)
    tables = (lws, groups, pst, pid)
    assert tick(engine, [(R.TABLE_DS_LINKS, 0, links, True)], tables, "linked") == (n_linked, 0)
    # LWS rows changed under the links: a row reused for another object (uid), an irregular object,
    # rollingUpdateParameters and updateConditions errors
    ex = np.flatnonzero(links["lws_row"] != R.NONE)
    pick = links["lws_row"][ex[rng.choice(len(ex), size=8, replace=False)]].astype(np.uint32)
    cases = [("uid", "uid_hash", None), ("irregular", "flags", R.LWS_IRREGULAR),
             ("rup", "flags", R.LWS_INTSTR_INVALID), ("status", "flags", R.LWS_GROUP_LABEL_INVALID)]
    for j, (what, field, bit) in enumerate(cases):
        rows = np.sort(pick[2 * j: 2 * j + 2])
        v = lws[rows].copy()
        if bit is None:
            v[field] = v[field] ^ np.uint64(0x5555)
        else:
            v[field] |= np.uint32(bit)
        lws[rows] = v
        engine.resident_tick(engine.make_tick([(R.TABLE_LWS, rows, v)]))
        lo = oracle.sweep_lws(*tables)[0]
        if what != "uid":
            want_bit = {"irregular": R.LOUT_IRREGULAR, "rup": R.LOUT_RUP_ERROR, "status": R.LOUT_STATUS_ERROR}[what]
            assert (lo["flags"][rows] & want_bit).all(), what
        took, fell = tick(engine, (), tables, what)
        users = int(np.isin(links["lws_row"], pick[: 2 * j + 2]).sum())
        assert fell == users > 0, what
    # a link to a row at or beyond n_lws, and a link on a row without RR_EXISTS
    absent = np.flatnonzero((rr["flags"] & R.RR_EXISTS) == 0)[:3].astype(np.uint32)
    far = ex[~np.isin(links["lws_row"][ex], pick)][:2].astype(np.uint32)
    v = links[far].copy()
    v["lws_row"] = [len(lws), len(lws) + 7]
    links[far] = v
    w = links[absent].copy()
    w["lws_row"], w["lws_uid_hash"] = 0, lws["uid_hash"][0]
    links[absent] = w
    before = fell
    took, fell = tick(engine, [(R.TABLE_DS_LINKS, far, v), (R.TABLE_DS_LINKS, absent, w)], tables, "far / absent")
    assert fell == before + len(far) + len(absent)
    # an LWS row given to another object by a patch without a sweep (lwse_resident_patch): the results
    # still belong to the previous object, so no linked row takes them until the next sweep
    q = int(ex[~np.isin(links["lws_row"][ex], pick) & ~np.isin(ex, far)][0])
    L = np.array([links["lws_row"][q]], np.uint32)
    v = lws[L].copy()
    v["uid_hash"] ^= np.uint64(0xABC)
    lws[L] = v
    engine.resident_patch(R.TABLE_LWS, L, v)
    u = links[q: q + 1].copy()
    u["lws_uid_hash"] = v["uid_hash"]
    links[q: q + 1] = u
    took, fell = tick(engine, [(R.TABLE_DS_LINKS, np.array([q], np.uint32), u)], None, "patched, not swept")
    assert took == 0 and fell == int((links["lws_row"] != R.NONE).sum())
    engine.resident_tick(engine.make_tick(()))
    took2, _ = tick(engine, (), tables, "swept again")
    assert took2 > 0


def test_rejected_link_patches_change_nothing(engine):
    """Rejected link segments, each behind a valid one in the same call, on a linked engine: the link
    table, the mirrors and the row counts stay what they were."""
    from lws_b200.engine import Engine, LwseError

    d = synth.make_ds(2000, (2,), seed=5)
    fresh = Engine(0)
    try:
        with pytest.raises(LwseError) as ei:  # a link segment before the DS load
            fresh.ds_resident_tick([(R.TABLE_DS_LINKS, 0, none_links(4), True)])
        assert ei.value.status == -6
    finally:
        fresh.close()
    rng = np.random.default_rng(3)
    lws, groups, pst, pid, links = child_lws_tables(d.revroles, rng)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick(()))
    engine.ds_resident_load(d.ds, d.roles, d.revroles)
    res = engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)])
    lo = oracle.sweep_lws(lws, groups, pst, pid)[0]
    want, took, fell = _expect(d.ds, d.roles, d.revroles, links, lws, lo)
    _same_mirrors(res, want, "linked")
    info = engine.ds_resident_tick_info()
    assert (info["rows_from_lws"], info["rows_fallback"]) == (took, fell) and took > 0
    assert want[2].tobytes() != oracle.sweep_ds(d.ds, d.roles, d.revroles)[2].tobytes()  # links change results
    n = len(d.revroles)
    ex = np.flatnonzero(links["lws_row"] != R.NONE).astype(np.uint32)
    unlink = none_links(8)  # would unlink eight rows if anything of the call were applied
    reserved = links[ex[8]: ex[8] + 1].copy()
    reserved["reserved"] = 1
    bad = [
        [(R.TABLE_DS_LINKS, np.array([ex[9], n], np.uint32), none_links(2))],  # row == n_revroles
        [(R.TABLE_DS_LINKS, n - 1, none_links(2), True)],                      # range past the end
        [(R.TABLE_DS_LINKS, np.array([ex[8]], np.uint32), reserved)],           # a reserved word set
    ]
    for segs in bad:
        with pytest.raises(LwseError) as ei:
            engine.ds_resident_tick([(R.TABLE_DS_LINKS, ex[:8], unlink)] + segs)
        assert ei.value.status == -1
        res = engine.ds_resident_tick()
        assert res["n_changed"] == 0
        _same_mirrors(res, want, "after a rejected link patch")
        info = engine.ds_resident_tick_info()
        assert info["linked"] and (info["rows_from_lws"], info["rows_fallback"]) == (took, fell)


def test_reference_flows_with_readiness_from_linked_children(engine, capsys):
    """The executor flows of tests/test_gpu_ds_tick.py (executor_test.go:1244-1298 both child orders,
    :486-556 drain order), every child a resident size-1 LeaderWorkerSet whose leader pods carry the
    readiness; no revision-role row ever holds a ready count.  One loop iteration is one LWS tick and one
    DS tick.  Linked: the same per-cycle results as the oracle replay (and the unlinked replay of
    test_gpu_ds_tick), one iteration per rollout step.  Against it the unlinked loop in which the ready
    count reaches the DS tick only through the status the LWS tick computed, written back and delivered
    one iteration later: the same final state, more iterations."""
    from ds_link_world import FlowLoop, steps_of
    from ds_sim import DsSim
    from test_oracle_ds_flows import abc
    import test_oracle_ds_order_stability as V

    def make(sweep):
        sims = []
        for order in (("A", "B"), ("B", "A")):
            for args in (((2, 4), (1, 2), (1, 2), (1, 1)), ((4, 3), (1, 2), (3, 1), (1, 2))):
                ds, children = abc(*args, order)
                sims.append(DsSim(ds, "C", children, sweep))
        for revisions, _ in V.SORT_CASES:
            children = []
            for h, tp, td in revisions:
                children += [api.ChildLWS("prefill", h, 1, 1, float(tp)), api.ChildLWS("decode", h, 1, 1, float(td))]
            sims.append(DsSim(V._ds(len(revisions)), "new", children, sweep))
        for i, s in enumerate(sims):  # one table: distinct names
            s.ds = api.DisaggregatedSet(f"flow-{i}", s.ds.namespace, roles=s.ds.roles)
        return sims

    def run(sims, loop, cycles):
        for s in sims:
            s.sweep_ds = loop.sweep_for(s)
        for step in range(cycles):
            if step:
                loop.tick()
                if loop.linked:
                    info = engine.ds_resident_tick_info()
                    assert info["rows_fallback"] == 0 and info["rows_from_lws"] > 0, step
                    assert not loop.ds_enc.revroles["ready_replicas"].any()  # no status ever reached a row
            for s in sims:
                s.reconcile()
                s.simulate_all_ready()

    ref = make(lambda t: oracle.sweep_ds(t.ds, t.roles, t.revroles))
    for s in ref:
        for _ in range(40):
            s.reconcile()
            s.simulate_all_ready()
    linked = make(None)
    run(linked, FlowLoop(engine, linked, True), 40)
    for a, b in zip(ref, linked):
        assert b.history == a.history, b.ds.name
    trip = make(None)
    run(trip, FlowLoop(engine, trip, False), 80)
    for a, b in zip(ref, trip):
        assert b.history[-1] == a.history[-1], b.ds.name  # the same end state, later
    n_ref, it_ref = (sum(x) for x in zip(*(steps_of(s.history) for s in ref)))
    n_link, it_link = (sum(x) for x in zip(*(steps_of(s.history) for s in linked)))
    n_trip, it_trip = (sum(x) for x in zip(*(steps_of(s.history) for s in trip)))
    assert (n_link, it_link) == (n_ref, it_ref) and it_trip > it_link
    with capsys.disabled():
        print(f"\nreference flows: {len(ref)} flows; linked {n_link} rollout steps in {it_link} loop iterations "
              f"({it_link / n_link:.2f} per step); status round trip {n_trip} steps in {it_trip} iterations "
              f"({it_trip / n_trip:.2f} per step)")
