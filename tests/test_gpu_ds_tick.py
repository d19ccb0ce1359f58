"""The DS tick (lwse_ds_resident_load / lwse_ds_resident_tick): resident DisaggregatedSet tables patched
row by row, every DS swept each tick, and exactly the DS whose results changed (or whose own row was
patched) reported — against ``oracle.sweep_ds`` over the same tables.  Also the reference flows replayed
through the DS encoder and the DS tick, DS ticks between the submit and the wait of pipelined
LeaderWorkerSet ticks, and the error paths."""
import numpy as np
import pytest

import oracle
from lws_b200 import api, churn, ds_informer, encoder, synth
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


def _owners(ds):
    """DS row of every role row and every revision-role row of a contiguous synth layout."""
    n = ds["n_roles"].astype(np.int64)
    nrr = (ds["n_old_revs"].astype(np.int64) + 1) * n
    assert np.array_equal(ds["role_base"], np.concatenate([[0], np.cumsum(n)[:-1]]))
    return np.repeat(np.arange(len(ds)), n), np.repeat(np.arange(len(ds)), nrr)


def _changed_ds(before, after, role_owner, rr_owner, n_ds):
    ch = np.zeros(n_ds, bool)
    ch |= (before[0].view(np.uint8).reshape(n_ds, -1) != after[0].view(np.uint8).reshape(n_ds, -1)).any(1)
    ch[role_owner[(before[1].view(np.uint64) != after[1].view(np.uint64))]] = True
    ch[rr_owner[before[2] != after[2]]] = True
    return ch


def test_c4_first_tick_lists_every_ds(engine):
    t = synth.make_ds(50_000, (2,))
    engine.ds_resident_load(t.ds, t.roles, t.revroles)
    res = engine.ds_resident_tick()
    assert res["n_changed"] == len(t.ds)
    assert np.array_equal(np.sort(res["rows"]), np.arange(len(t.ds), dtype=np.uint32))
    _same_mirrors(res, oracle.sweep_ds(t.ds, t.roles, t.revroles), "first tick")
    again = engine.ds_resident_tick()  # nothing patched: nothing listed, mirrors unchanged
    assert again["n_changed"] == 0
    _same_mirrors(again, oracle.sweep_ds(t.ds, t.roles, t.revroles), "idle tick")


def test_seeded_row_patches_report_exactly_the_changed_ds(engine):
    """200 ticks of ~1 % revision-role rows plus some role and DS rows, scattered and as ranges: each
    tick lists exactly the DS whose oracle results changed or whose DS row was patched."""
    t = synth.make_ds(50_000, (2,), seed=11)
    ds, roles, rr = t.ds.copy(), t.roles.copy(), t.revroles.copy()
    role_owner, rr_owner = _owners(ds)
    n_ds = len(ds)
    engine.ds_resident_load(ds, roles, rr)
    prev = oracle.sweep_ds(ds, roles, rr)
    res = engine.ds_resident_tick()
    assert res["n_changed"] == n_ds
    rng = np.random.default_rng(5)
    for k in range(200):
        segs = []
        # revision-role rows: status updates (ready), scale changes, sometimes nil replicas
        rows = np.unique(rng.choice(len(rr), size=len(rr) // 100, replace=False)).astype(np.uint32)
        v = rr[rows].copy()
        v["ready_replicas"] = rng.integers(0, 33, size=len(rows))
        scale = rng.random(len(rows)) < 0.3
        v["replicas"] = np.where(scale, rng.integers(0, 33, size=len(rows)), v["replicas"])
        nil = rng.random(len(rows)) < 0.02
        v["flags"] = np.where(nil, v["flags"] | R.RR_REPLICAS_NIL, v["flags"] & ~np.uint32(R.RR_REPLICAS_NIL))
        segs.append((R.TABLE_DS_REVROLES, rows, v))
        # role rows: a new target; every fourth tick a contiguous block as a range
        if k % 4 == 0:
            first = int(rng.integers(0, len(roles) - 16))
            v = roles[first: first + 16].copy()
            v["target_replicas"] = np.where(v["flags"] & R.ROLE_IN_SPEC, rng.integers(0, 33, size=16), 0)
            segs.append((R.TABLE_DS_ROLES, first, v, True))
            roles[first: first + 16] = v
        else:
            r = np.unique(rng.choice(len(roles), size=20, replace=False)).astype(np.uint32)
            v = roles[r].copy()
            v["target_replicas"] = np.where(v["flags"] & R.ROLE_IN_SPEC, rng.integers(0, 33, size=len(r)), 0)
            segs.append((R.TABLE_DS_ROLES, r, v))
            roles[r] = v
        # DS rows: HAS_NEW_REVISION toggled, or re-written unchanged (still listed); ranges on odd ticks
        if k % 2:
            first = int(rng.integers(0, n_ds - 4))
            patched = np.arange(first, first + 4)
            v = ds[patched].copy()
            v["flags"] ^= np.where(rng.random(4) < 0.5, R.DS_HAS_NEW_REVISION, 0).astype(np.uint32)
            segs.append((R.TABLE_DS, first, v, True))
        else:
            patched = np.unique(rng.choice(n_ds, size=6, replace=False))
            v = ds[patched].copy()
            v["flags"] ^= np.where(rng.random(len(patched)) < 0.5, R.DS_HAS_NEW_REVISION, 0).astype(np.uint32)
            segs.append((R.TABLE_DS, patched.astype(np.uint32), v))
        ds[patched] = v
        rr[rows] = segs[0][2]
        res = engine.ds_resident_tick(segs)
        want = oracle.sweep_ds(ds, roles, rr)
        expect = _changed_ds(prev, want, role_owner, rr_owner, n_ds)
        expect[patched] = True
        got = np.sort(res["rows"])
        assert res["n_changed"] == len(got) == len(np.unique(got)), k
        assert np.array_equal(got, np.flatnonzero(expect).astype(np.uint32)), f"tick {k}: changed set"
        _same_mirrors(res, want, f"tick {k}")
        prev = want


class ResidentDsPath:
    """Many DsSim flows in ONE resident table: between reconciles the child-list changes of every sim
    become watch events of the DS encoder, one DS tick applies them, and each sim reads its DS's
    results from the tick's mirrors."""

    def __init__(self, engine, sims):
        self.engine, self.sims = engine, sims
        items = [encoder.DsItem(s.ds, s.revision, [self._copy(c) for c in s.children]) for s in sims]
        self.enc = ds_informer.DsIncrementalEncoder(items, spare=1.0)
        engine.ds_resident_load(*self.enc.tables())
        self.snap = [self._snapshot(s) for s in sims]
        self.res = engine.ds_resident_tick()

    @staticmethod
    def _copy(c):
        return api.ChildLWS(c.role, c.revision, c.replicas, c.readyReplicas, c.creationTimestamp, dict(c.annotations))

    def _snapshot(self, sim):
        return {(c.role, c.revision): (c.replicas, c.readyReplicas, c.creationTimestamp, dict(c.annotations))
                for c in sim.children}

    def tick(self):
        for i, s in enumerate(self.sims):
            now = self._snapshot(s)
            ns, name = s.ds.namespace, s.ds.name
            for key in self.snap[i]:
                if key not in now:
                    self.enc.child_event("DELETED", ns, name, api.ChildLWS(key[0], key[1]))
            for c in s.children:
                key = (c.role, c.revision)
                if key not in self.snap[i]:
                    self.enc.child_event("ADDED", ns, name, self._copy(c))
                elif self.snap[i][key] != now[key]:
                    self.enc.child_event("MODIFIED", ns, name, self._copy(c))
            self.snap[i] = now
        p = self.enc.flush()
        assert not self.enc.needs_reload
        self.res = self.engine.ds_resident_tick(p.segments)

    def sweep_for(self, sim):
        def sweep(t):
            d = self.enc.ds_row(sim.ds.namespace, sim.ds.name)
            assert self.enc.role_names(d) == t.role_names[0] and self.enc.old_revisions(d) == t.old_revisions[0]
            row = self.enc.ds[d]
            rb, n, vb = int(row["role_base"]), int(row["n_roles"]), int(row["rev_base"])
            nrr = (int(row["n_old_revs"]) + 1) * n
            return (self.res["ds_out"][d: d + 1].copy(), self.res["role_out"][rb: rb + n].copy(),
                    self.res["revrole_out"][vb: vb + nrr].copy())
        return sweep


def test_reference_flows_through_the_resident_path(engine):
    """executor_test.go:1244-1298 (both child orders) and :486-556 (drain order), every flow a DS of one
    shared table, against the same flows decided by the oracle."""
    from ds_sim import DsSim
    from test_oracle_ds_flows import abc
    import test_oracle_ds_order_stability as V

    def oracle_sweep(t):
        return oracle.sweep_ds(t.ds, t.roles, t.revroles)

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

    ref = make(oracle_sweep)
    sims = make(None)
    path = ResidentDsPath(engine, sims)
    for s in sims:
        s.sweep_ds = path.sweep_for(s)
    for step in range(40):
        if step:
            path.tick()
        for a, b in zip(ref, sims):
            a.reconcile()
            b.reconcile()
            a.simulate_all_ready()
            b.simulate_all_ready()
    for a, b in zip(ref, sims):
        assert b.history == a.history, b.ds.name


def test_stability_and_readiness_vectors_in_one_table(engine):
    """executor_test.go:558-588 and the service readiness rule: every vector a DS of one resident table."""
    import test_oracle_ds_order_stability as V

    items = []
    for case, _ in V.STABLE_CASES:
        pr, prd, dr, drd = case
        ds = api.DisaggregatedSet(f"s{len(items)}", roles=[api.DisaggregatedRoleSpec("prefill", 4), api.DisaggregatedRoleSpec("decode", 4)])
        items.append(encoder.DsItem(ds, "hash1", [
            api.ChildLWS("prefill", "old", 2, 2, 1.0), api.ChildLWS("decode", "old", 2, 2, 1.0),
            api.ChildLWS("prefill", "hash1", pr, prd, 2.0), api.ChildLWS("decode", "hash1", dr, drd, 2.0)]))
    for ready, _ in V.READY_CASES:
        ds = api.DisaggregatedSet(f"s{len(items)}", roles=[api.DisaggregatedRoleSpec("prefill", 2), api.DisaggregatedRoleSpec("decode", 2)])
        items.append(encoder.DsItem(ds, "new", [
            api.ChildLWS("prefill", "old", 2, 2, 1.0), api.ChildLWS("decode", "old", 2, 2, 1.0),
            api.ChildLWS("prefill", "new", 3, ready[0], 2.0), api.ChildLWS("decode", "new", 3, ready[1], 2.0)]))
    enc = ds_informer.DsIncrementalEncoder(items)
    engine.ds_resident_load(*enc.tables())
    res = engine.ds_resident_tick()
    want = (V.STABLE_CASES, R.DOUT_STABLE), (V.READY_CASES, R.DOUT_NEW_READY)
    i = 0
    for cases, bit in want:
        for _, expect in cases:
            d = enc.ds_row("default", f"s{i}")
            assert bool(res["ds_out"][d]["flags"] & bit) == expect, i
            i += 1


def test_ds_ticks_between_submit_and_wait_leave_lws_ticks_alone(engine):
    """C3 pipelined LeaderWorkerSet ticks, with and without a C4 DS tick between each submit and wait: the
    same changed LWS / group / placement rows, and the steady LWS ticks still replay their graph."""
    t = synth.make("C3-steady", seed=41)
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    d = synth.make_ds(50_000, (2,), seed=3)
    rng = np.random.default_rng(2)

    def run(with_ds):
        engine.upload_nodes(t.nodes, t.n_domains)
        engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        engine.resident_place_load(reqs, t.n_namespaces)
        engine.resident_tick(engine.make_tick((), flags))
        plan = churn.make_plan(t, reqs, engine.resident_place_outputs(), 0.01, 0.01, n_sets=6, seed=4)
        ticks = churn.ArenaPlan(engine, plan, flags).ticks
        if with_ds:
            engine.ds_resident_load(d.ds, d.roles, d.revroles)
            engine.ds_resident_tick()
        out, graphs = [], []
        n = 24
        engine.resident_tick_submit(ticks[0])
        for k in range(1, n + 1):
            if k < n:
                engine.resident_tick_submit(ticks[k % len(ticks)])
                graphs.append(engine.resident_tick_info()["graph"])
            if with_ds:
                rows = np.unique(rng.choice(len(d.revroles), size=len(d.revroles) // 100, replace=False)).astype(np.uint32)
                v = d.revroles[rows].copy()
                v["ready_replicas"] = rng.integers(0, 33, size=len(rows))
                engine.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
            r = engine.resident_tick_wait()
            out.append(tuple(np.sort(r[name].copy()).tobytes() for name in ("lws_rows", "group_rows", "place_rows")))
        return out, graphs

    base, base_graphs = run(False)
    mixed, graphs = run(True)
    assert mixed == base
    assert graphs == base_graphs and all(graphs[6:]), (base_graphs, graphs)  # steady ticks are graph replays


def test_error_paths_leave_tables_and_outputs_alone(engine):
    from lws_b200.engine import Engine, LwseError

    fresh = Engine(0)
    try:
        with pytest.raises(LwseError) as ei:  # a DS tick before a DS load
            fresh.ds_resident_tick()
        assert ei.value.status == -6
    finally:
        fresh.close()
    t = synth.make_ds(2000, (2, 3), seed=9)
    ds, roles, rr = t.ds.copy(), t.roles.copy(), t.revroles.copy()
    engine.ds_resident_load(ds, roles, rr)
    engine.ds_resident_tick()
    good_rows = np.array([1, 2], np.uint32)
    bad = [
        [(R.TABLE_DS_REVROLES, np.array([len(rr)], np.uint32), rr[:1].copy())],          # row == table size
        [(R.TABLE_DS_ROLES, len(roles) - 1, roles[:2].copy(), True)],                     # range past the end
        [(R.TABLE_DS, np.array([0, len(ds) + 5], np.uint32), ds[:2].copy())],             # one bad row of two
        [(R.TABLE_LWS, good_rows, np.zeros(2, R.LWS_REC))],                               # not a DS table
        [(R.TABLE_DS_REVROLES, good_rows, rr[:2].copy()), (9, good_rows, rr[:2].copy())],  # unknown table
    ]
    for segs in bad:
        v = rr[:2].copy()
        v["ready_replicas"] += 7  # would change results if it were applied
        segs = [(R.TABLE_DS_REVROLES, good_rows, v)] + segs
        with pytest.raises(LwseError) as ei:
            engine.ds_resident_tick(segs)
        assert ei.value.status == -1
        res = engine.ds_resident_tick()
        assert res["n_changed"] == 0
        _same_mirrors(res, oracle.sweep_ds(ds, roles, rr), "after a rejected tick")
    # NULL values
    import ctypes as C
    from lws_b200.engine import lib

    seg = (R.PatchSeg * 1)(R.PatchSeg(R.TABLE_DS_REVROLES, 0, 1, 0, good_rows.ctypes.data, None))
    ch = R.DsChanges()
    assert lib().lwse_ds_resident_tick(engine._h, seg, 1, C.byref(ch)) == -1
    assert lib().lwse_ds_resident_tick(engine._h, None, 0, None) == -1
    # the LWS calls still refuse the DS tables
    vals = ds[:2].copy()
    assert lib().lwse_resident_patch(engine._h, R.TABLE_DS, good_rows.ctypes.data, vals.ctypes.data, 2) < 0
    res = engine.ds_resident_tick()
    assert res["n_changed"] == 0
    _same_mirrors(res, oracle.sweep_ds(ds, roles, rr), "end")
