"""The resident tick on request tables that are not grouped by namespace: LeaderWorkerSets created and
deleted through the incremental encoder, a full-size C3 table made ungrouped, and the edge cases of
the namespace index — every placement row against the spec oracle on the same rows."""
import numpy as np
import pytest

from lws_b200 import churn, encoder, informer, synth
from lws_b200 import records as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def grouped(reqs):
    return bool(np.all(np.diff(reqs["ns"].astype(np.int64)) >= 0))


def ungroup(reqs, frac=0.01, seed=3):
    """Move `frac` of the live requests to new tail rows (the old rows become inert) and interleave the
    rows of the two largest namespaces."""
    rng = np.random.default_rng(seed)
    live = np.flatnonzero(reqs["size"] >= 1)
    moved = np.sort(rng.choice(live, size=max(1, int(len(live) * frac)), replace=False))
    out = R.aligned_empty(len(reqs) + len(moved), R.PLACE_REQ)
    out[: len(reqs)] = reqs
    out[len(reqs):] = reqs[moved]
    out["size"][moved] = 0
    out["leader_node"][moved] = R.NONE
    ns = out["ns"].astype(np.int64)
    a, b = np.argsort(np.bincount(ns))[-2:]
    pa, pb = np.flatnonzero(ns == a), np.flatnonzero(ns == b)
    pos = np.sort(np.concatenate([pa, pb]))
    k = min(len(pa), len(pb))
    order = np.concatenate([np.stack([pa[:k], pb[:k]], 1).reshape(-1), pa[k:], pb[k:]])
    rows = out[order].copy()
    out[pos] = rows
    assert not grouped(out)
    return out


def test_informer_stream_with_creates_and_deletes(engine):
    """Creates and deletes (new namespaces, names re-used) through the arena with two ticks in flight:
    after each tick the engine's changed rows, applied to the previous results, equal the oracle on a fresh
    encode by name (sweep) and on the same rows (placement); the occupancy at every drain."""
    import oracle
    from informer_world import make_world, outputs_by_name
    from lifecycle_world import LifecycleWorld

    items, cluster = make_world(5, n_lws=24, n_nodes=40)
    world = LifecycleWorld(items, cluster, 6, p_create=0.2, p_delete=0.12)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=2.0)
    lws, groups, pst, pid, reqs = enc.full_tables()
    engine.upload_nodes(enc.node_rec, len(enc.domain_values))
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, enc.n_namespaces)
    flags = R.SWEEP_GANG | R.TICK_PLACE
    engine.resident_tick(engine.make_tick((), flags))
    m_lo, m_go = (a.copy() for a in engine.resident_outputs())
    m_po = engine.resident_place_outputs().copy()
    half = 1 << 20
    arena = engine.resident_arena(2 * half)

    def in_arena(segments, which):
        cursor, out = which * half, []
        for table, rows, vals in segments:
            views = []
            for a in (np.ascontiguousarray(rows, dtype=np.uint32), np.ascontiguousarray(vals)):
                cursor = (cursor + 255) // 256 * 256
                v = arena[cursor: cursor + a.nbytes].view(a.dtype)
                v[...] = a
                cursor += a.nbytes
                views.append(v)
            out.append((table, views[0], views[1]))
        assert cursor <= (which + 1) * half
        return out

    def expected():
        fresh_items = list(world.items.values())
        ft = encoder.encode_lws(fresh_items, world.cluster(), "zone")
        w_lo, w_go, w_occ = oracle.sweep_lws(ft.lws, ft.groups, ft.pod_state, ft.pod_ident, ft.nodes, flags=R.SWEEP_GANG,
                                             want_occupancy=True)
        want = outputs_by_name(ft.lws, ft.groups, w_lo, w_go, {i: (it.lws.namespace, it.lws.name) for i, it in enumerate(fresh_items)})
        want_p = oracle.place(enc.node_rec, w_occ, len(enc.domain_values), enc.n_namespaces, enc.reqs)
        return want, want_p, w_occ, enc.lws.copy(), enc.groups.copy(), {sl.lws_row: key for key, sl in enc.slots.items()}

    def check(res, exp, where):
        (want_l, want_g), want_p, _, t_lws, t_grp, names = exp
        m_lo[res["lws_rows"]] = res["lws_out"]
        m_go[res["group_rows"]] = res["group_out"]
        m_po[res["place_rows"]] = res["place_out"]
        got_l, got_g = outputs_by_name(t_lws, t_grp, m_lo, m_go, names)
        assert got_l == want_l, where
        assert got_g == want_g, where
        assert m_po.tobytes() == want_p.tobytes(), where

    pending, infos, was_ungrouped = [], [], False
    for tick in range(40):
        for _ in range(int(world.rng.integers(1, 6))):
            world.step(enc)
        patches = enc.flush()
        assert not enc.needs_reload
        exp = expected()
        t = engine.make_tick(in_arena(patches.segments, tick & 1), flags)
        if len(pending) == 2:
            check(engine.resident_tick_wait(), pending.pop(0), f"tick {tick - 2}")
        engine.resident_tick_submit(t)
        info = engine.resident_tick_info()
        was_ungrouped = was_ungrouped or not grouped(enc.reqs)
        infos.append((was_ungrouped, info))
        pending.append(exp)
        if tick % 10 == 9:  # drain: the occupancy the engine counts from the patched identity rows
            while pending:
                check(engine.resident_tick_wait(), pending.pop(0), f"drain {tick}")
            assert np.array_equal(engine.resident_occupancy(), exp[2]), f"tick {tick}"
    while pending:
        check(engine.resident_tick_wait(), pending.pop(0), "end")
    assert any(u for u, _ in infos), "the stream never ungrouped the request table"
    for u, info in infos:
        assert info["form"] == "namespace"
        if u:
            assert info["indexed"]
    assert any(u and i["graph"] for u, i in infos), infos


@pytest.mark.parametrize("scan", [False, True], ids=["two_level", "scan"])
def test_c3_full_size_ungrouped(engine, scan):
    """synth C3 at scale 1.0 with 1 % of the requests moved to the tail and two namespaces interleaved:
    resident ticks with scheduling churn, one of them moving a request to another namespace — every
    tick's placement rows and change list equal the oracle's."""
    import oracle

    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = ungroup(t.place_requests())
    n_ns = t.n_namespaces
    occ = R.occupancy_of(t.pod_ident, len(t.nodes))
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, n_ns)
    flags = t.flags | R.TICK_PLACE | (R.SWEEP_PLACE_SCAN if scan else 0)
    first = engine.resident_tick(engine.make_tick((), flags))
    info = engine.resident_tick_info()
    assert info["form"] == ("scan" if scan else "namespace") and info["indexed"] and info["index_built"]
    prev = oracle.place(t.nodes, occ, t.n_domains, n_ns, reqs, threads=16)
    assert engine.resident_place_outputs().tobytes() == prev.tobytes()
    assert first["n_place"] == len(reqs)
    # the churn plan's scheduling events, plus one tick that moves a live request to another namespace
    plan = churn.make_plan(t, reqs, prev, 0.01, 0.002, n_sets=4)
    mirror = reqs.copy()
    rng = np.random.default_rng(9)
    for k in range(6):
        ps = plan[k % len(plan)]
        rows, vals = ps.req_rows, ps.req_vals
        moves = k == 3
        if moves:
            planned = np.concatenate([p.req_rows for p in plan])  # (no later set may move it back)
            r = int(rng.choice(np.setdiff1d(np.flatnonzero(mirror["size"] >= 1), planned)))
            v = R.aligned_empty(1, R.PLACE_REQ)
            v[:] = mirror[r]
            v["ns"] = (int(v["ns"][0]) + 1) % n_ns
            order = np.argsort(np.concatenate([rows, [r]]))
            rows = np.concatenate([rows, [r]]).astype(np.uint32)[order]
            vals = np.concatenate([vals, v])[order]
        mirror[rows] = vals
        segs = [(R.TABLE_POD_STATE, ps.pod_rows, ps.pod_vals), (R.TABLE_PLACE_REQS, rows, vals)]
        if len(ps.grp_rows):
            segs.append((R.TABLE_GROUPS, ps.grp_rows, ps.grp_vals))
        res = engine.resident_tick(engine.make_tick(segs, flags))
        info = engine.resident_tick_info()
        assert info["indexed"] and info["index_built"] == moves, (k, info)
        want = oracle.place(t.nodes, occ, t.n_domains, n_ns, mirror, threads=16)
        got = engine.resident_place_outputs()
        assert got.tobytes() == want.tobytes(), f"tick {k}"
        changed = np.flatnonzero((want.view(np.uint8).reshape(len(want), -1) != prev.view(np.uint8).reshape(len(prev), -1)).any(axis=1))
        assert res["n_place"] == len(changed), f"tick {k}"
        order = np.argsort(res["place_rows"])
        assert np.array_equal(res["place_rows"][order], changed), f"tick {k}"
        assert res["place_out"][order].tobytes() == want[changed].tobytes(), f"tick {k}"
        prev = want


def _edge_world(n_nodes=400):
    from informer_world import make_world

    items, cluster = make_world(0, n_lws=4, n_nodes=n_nodes)
    return informer.IncrementalEncoder(items, cluster, "zone")


@pytest.mark.parametrize("scan", [False, True], ids=["two_level", "scan"])
def test_index_edge_cases(engine, scan):
    """One namespace scattered over > 1 024 rows with > 256 unpinned requests, priority ties the row
    decides, namespaces that do not exist, empty namespaces in the headroom."""
    import oracle

    enc = _edge_world()
    n_nodes, n_dom = len(enc.node_rec), len(enc.domain_values)
    rng = np.random.default_rng(4)
    n = 3000
    reqs = R.aligned_empty(n, R.PLACE_REQ)
    reqs["ns"] = rng.choice([0, 0, 0, 1, 2, 5, 9], size=n)  # namespace 0 everywhere; 9 >= n_namespaces
    reqs["priority"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    ties = rng.choice(n, size=200, replace=False)
    reqs["priority"][ties] = np.uint64(12345) << np.uint64(30)  # equal keys but for the row
    reqs["group_key"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    reqs["group"] = np.arange(n)
    reqs["size"] = rng.integers(0, 12, size=n)
    pinned = rng.random(n) < 0.2
    reqs["leader_node"] = np.where(pinned, rng.integers(0, n_nodes, size=n), R.NONE).astype(np.uint32)
    n_ns = 8  # namespaces 3, 4, 6, 7 are empty; 9 does not exist
    assert ((reqs["ns"] == 0) & (reqs["size"] >= 1) & ~pinned).sum() > 256
    lws, groups, pst, pid, _ = enc.full_tables()
    engine.upload_nodes(enc.node_rec, n_dom)
    engine.resident_load(lws, groups, pst, pid)
    occ = R.occupancy_of(pid, n_nodes)
    engine.resident_place_load(reqs, n_ns)
    flags = R.TICK_PLACE | R.TICK_NO_SWEEP | (R.SWEEP_PLACE_SCAN if scan else 0)
    engine.resident_tick(engine.make_tick((), flags))
    assert engine.resident_tick_info()["indexed"]
    want = oracle.place(enc.node_rec, occ, n_dom, n_ns, reqs)
    got = engine.resident_place_outputs()
    assert got.tobytes() == want.tobytes()
    assert (got["flags"][reqs["ns"] >= n_ns] & R.PLACE_UNSCHEDULABLE).all()
    # the same rows in another order: the index differs, the rows' results do not
    shuffled = R.aligned_empty(n, R.PLACE_REQ)
    shuffled[:] = reqs[rng.permutation(n)]
    engine.resident_place_load(shuffled, n_ns)
    engine.resident_tick(engine.make_tick((), flags))
    want_p = oracle.place(enc.node_rec, occ, n_dom, n_ns, shuffled)
    assert engine.resident_place_outputs().tobytes() == want_p.tobytes()
