"""Node watch events as row patches in the resident tick (LWSE_TABLE_NODES): capacity changes, cordons,
relabels, deletions and additions, through the informer and on a full-size C3 table, in every placement
form — every placement row and group row against the oracle on the same rows, and the node index rebuilt
exactly by the ticks that change which nodes are usable or their domains."""
import numpy as np
import pytest

from lws_b200 import informer, synth
from lws_b200 import records as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def usable_mask(nodes, n_domains):
    f = nodes["flags"]
    return ((f & R.NODE_SCHEDULABLE) != 0) & ((f & R.NODE_HAS_TOPOLOGY) != 0) & (nodes["domain_id"] < n_domains)


def usable_count(nodes, n_domains):
    return int(usable_mask(nodes, n_domains).sum())


class Arena:
    """Two halves of the engine's patch arena, one per tick in flight."""

    def __init__(self, engine, half=4 << 20):
        self.half = half
        self.buf = engine.resident_arena(2 * half)

    def put(self, segments, which):
        cursor, out = which * self.half, []
        for table, rows, vals in segments:
            views = []
            for a in (np.ascontiguousarray(rows, dtype=np.uint32), np.ascontiguousarray(vals)):
                cursor = (cursor + 255) // 256 * 256
                v = self.buf[cursor: cursor + a.nbytes].view(a.dtype)
                v[...] = a
                cursor += a.nbytes
                views.append(v)
            out.append((table, views[0], views[1]))
        assert cursor <= (which + 1) * self.half
        return out


def by_name(t_lws, t_grp, lo, go, names, domain_values):
    """{object: lws_out bytes}, {(object, group index): group_out bytes with the domain as its label value}."""
    l, g = {}, {}
    for row, name in names.items():
        l[name] = lo[row].tobytes()
        base, count = int(t_lws["group_base"][row]), int(t_lws["group_count"][row])
        for gi in range(count):
            o = go[base + gi].copy()
            d = int(o["domain_id"])
            o["domain_id"] = 0
            g[(name, gi)] = (o.tobytes(), domain_values[d] if d != R.NONE else None)
    return l, g


def test_informer_stream_with_node_events(engine):
    """Node, pod and LeaderWorkerSet events through the arena with two ticks in flight: after each tick the
    changed rows applied to the previous results equal the oracle on a fresh encode by name (sweep) and on
    the informer's own node table and occupancy (placement); the occupancy at every drain."""
    import oracle
    from lws_b200 import encoder
    from informer_world import make_world
    from node_world import NodeWorld

    items, cluster = make_world(5, n_lws=24, n_nodes=40)
    world = NodeWorld(items, cluster, 6, p_node=0.3, p_create=0.1, p_delete=0.06)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=2.0, node_spare=64)
    lws, groups, pst, pid, reqs = enc.full_tables()
    engine.upload_nodes(enc.node_rec, enc.n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(reqs, enc.n_namespaces)
    flags = R.SWEEP_GANG | R.TICK_PLACE
    engine.resident_tick(engine.make_tick((), flags))
    m_lo, m_go = (a.copy() for a in engine.resident_outputs())
    m_po = engine.resident_place_outputs().copy()
    arena = Arena(engine, 1 << 20)

    def expected():
        fresh_items = list(world.items.values())
        ft = encoder.encode_lws(fresh_items, world.cluster(), "zone")
        w_lo, w_go, _ = oracle.sweep_lws(ft.lws, ft.groups, ft.pod_state, ft.pod_ident, ft.nodes, flags=R.SWEEP_GANG)
        want = by_name(ft.lws, ft.groups, w_lo, w_go, {i: (it.lws.namespace, it.lws.name) for i, it in enumerate(fresh_items)},
                       ft.domain_values)
        occ = R.occupancy_of(enc.pod_ident, len(enc.node_rec))
        want_p = oracle.place(enc.node_rec, occ, enc.n_domains, enc.n_namespaces, enc.reqs)
        return (want, want_p, occ, enc.lws.copy(), enc.groups.copy(), {sl.lws_row: key for key, sl in enc.slots.items()},
                list(enc.domain_values), usable_count(enc.node_rec, enc.n_domains))

    def check(res, exp, where):
        (want_l, want_g), want_p, _, t_lws, t_grp, names, dvals, _ = exp
        m_lo[res["lws_rows"]] = res["lws_out"]
        m_go[res["group_rows"]] = res["group_out"]
        m_po[res["place_rows"]] = res["place_out"]
        got_l, got_g = by_name(t_lws, t_grp, m_lo, m_go, names, dvals)
        assert got_l == want_l, where
        assert got_g == want_g, where
        assert m_po.tobytes() == want_p.tobytes(), where

    pending, infos = [], []
    for tick in range(48):
        for _ in range(int(world.rng.integers(1, 7))):
            world.step(enc)
        if tick % 6 == 1:
            world.node_event(enc, "MODIFIED")
        patches = enc.flush()
        assert not enc.needs_reload
        exp = expected()
        t = engine.make_tick(arena.put(patches.segments, tick & 1), flags)
        if len(pending) == 2:
            check(engine.resident_tick_wait(), pending.pop(0), f"tick {tick - 2}")
        engine.resident_tick_submit(t)
        ni, ti = engine.resident_node_info(), engine.resident_tick_info()
        n_node_rows = sum(len(s[1]) for s in patches.segments if s[0] == R.TABLE_NODES)
        assert ni["rows_patched"] == n_node_rows and ni["n_usable"] == exp[7], (tick, ni)
        infos.append((ni, ti))
        pending.append(exp)
        if tick % 8 == 7:
            while pending:
                check(engine.resident_tick_wait(), pending.pop(0), f"drain {tick}")
            assert np.array_equal(engine.resident_occupancy(), exp[2]), f"tick {tick}"
    while pending:
        check(engine.resident_tick_wait(), pending.pop(0), "end")
    assert any(ni["index_built"] for ni, _ in infos)
    assert any(ni["rows_patched"] and not ni["index_built"] for ni, _ in infos)
    assert any(ni["rows_patched"] and ti["graph"] for ni, ti in infos), infos


def _c3_node_ticks(t, reqs, rng, n_ticks):
    """Node-row patch sets over a C3 table: 1 % capacity changes every tick; every other pair of ticks also
    cordons / uncordons, relabels, deletes (zeroes) and re-adds nodes — the node of a pinned leader among
    them — and empties one domain completely.  → [(rows, values, changes usability)], the node table after each."""
    nodes = t.nodes.copy()
    n = len(nodes)
    pinned = np.unique(reqs["leader_node"][reqs["leader_node"] < n]).astype(np.int64)
    out, tables = [], []
    saved = {}
    for k in range(n_ticks):
        rows = set(rng.choice(n, size=max(1, n // 100), replace=False).tolist())
        vals = {r: nodes[r].copy() for r in rows}
        for r in rows:
            vals[r]["capacity"] = int(rng.integers(0, 16))
        rebuild = (k // 2) % 2 == 1
        if rebuild:
            ev = [int(rng.choice(pinned)), *rng.choice(n, size=4, replace=False).tolist()]
            for j, r in enumerate(ev):
                v = vals.setdefault(r, nodes[r].copy())
                if j % 4 == 0:
                    v["flags"] ^= R.NODE_SCHEDULABLE  # cordon / uncordon (the first one: a pinned leader's node)
                elif j % 4 == 1:
                    v["domain_id"] = int(rng.integers(0, t.n_domains))  # relabel
                elif j % 4 == 2:
                    if r in saved:
                        vals[r] = saved.pop(r)  # the node comes back
                    else:
                        saved[r] = nodes[r].copy()
                        vals[r] = np.zeros(1, R.NODE_REC)[0]  # deleted
                else:
                    v["flags"] |= R.NODE_SCHEDULABLE
            d = int(rng.integers(0, t.n_domains))  # a domain emptied completely
            for r in np.flatnonzero(nodes["domain_id"] == d):
                v = vals.setdefault(int(r), nodes[int(r)].copy())
                v["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
        order = sorted(vals)
        rr = np.array(order, dtype=np.uint32)
        vv = R.aligned_empty(len(order), R.NODE_REC)
        for i, r in enumerate(order):
            vv[i] = vals[r]
        before = nodes.copy()
        nodes[rr] = vv
        changes = not np.array_equal(usable_mask(before, t.n_domains) * (before["domain_id"] + 1),
                                     usable_mask(nodes, t.n_domains) * (nodes["domain_id"] + 1))
        out.append((rr, vv, changes))
        tables.append(nodes.copy())
    return out, tables


@pytest.mark.parametrize("form", ["two_level", "scan", "indexed", "general"])
def test_c3_full_size_node_events(engine, form):
    """synth C3 at scale 1.0, ticks pipelined two deep from the arena with node-row patches: every placement
    row and every group row equal the oracle on the same rows; the node index is rebuilt exactly on the
    ticks that change usability or domains; steady and rebuild ticks both replay as graphs.  The general form:
    the same table uploaded with a domain capacity of 8 192 (spare ids no node uses), more domains than the
    namespace kernel's shared memory holds, so the tick runs the general placement kernel."""
    import oracle
    from test_gpu_lifecycle import ungroup

    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests() if form != "indexed" else ungroup(t.place_requests())
    n_ns = t.n_namespaces
    occ = R.occupancy_of(t.pod_ident, len(t.nodes))
    n_dom = 8192 if form == "general" else t.n_domains
    engine.upload_nodes(t.nodes, n_dom)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, n_ns)
    flags = t.flags | R.TICK_PLACE | (R.SWEEP_PLACE_SCAN if form == "scan" else 0)
    engine.resident_tick(engine.make_tick((), flags))
    assert engine.resident_tick_info()["form"] == {"two_level": "namespace", "indexed": "namespace"}.get(form, form)
    m_go = engine.resident_outputs()[1].copy()
    m_po = engine.resident_place_outputs().copy()
    rng = np.random.default_rng(21)
    sets, tables = _c3_node_ticks(t, reqs, rng, 12)
    arena = Arena(engine)
    pending, infos = [], []

    def check(res, k):
        nodes = tables[k]
        m_go[res["group_rows"]] = res["group_out"]
        m_po[res["place_rows"]] = res["place_out"]
        _, w_go, _ = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, nodes, flags=t.flags, threads=16)
        assert m_go.tobytes() == w_go.tobytes(), f"tick {k}: group rows"
        want = oracle.place(nodes, occ, n_dom, n_ns, reqs, threads=16)
        assert m_po.tobytes() == want.tobytes(), f"tick {k}: placement rows"

    for k, (rows, vals, changes) in enumerate(sets):
        seg = arena.put([(R.TABLE_NODES, rows, vals)], k & 1)
        if len(pending) == 2:
            check(engine.resident_tick_wait(), pending.pop(0))
        engine.resident_tick_submit(engine.make_tick(seg, flags))
        ni, ti = engine.resident_node_info(), engine.resident_tick_info()
        assert ni["rows_patched"] == len(rows), k
        assert ni["index_built"] == changes, (k, ni)
        assert ni["n_usable"] == int(usable_mask(tables[k], n_dom).sum()), k
        assert ti["indexed"] == (form == "indexed"), k
        infos.append((changes, ti["graph"]))
        pending.append(k)
    while pending:
        check(engine.resident_tick_wait(), pending.pop(0))
    if form == "general":  # (the general form is never replayed as a graph)
        assert not any(g for _, g in infos)
    else:
        assert any(c and g for c, g in infos) and any(not c and g for c, g in infos), infos


def test_round_after_a_node_tick_without_one():
    """A tick with node patches and no placement round, then at once a tick with a round and no patches, one
    tick at a time and two in flight, kernel by kernel (LWSE_TICK_GRAPH=0): the round (and the index it
    rebuilds) reads the node rows the first tick's scatter wrote."""
    import os

    import oracle
    from lws_b200.engine import Engine

    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    occ = R.occupancy_of(t.pod_ident, len(t.nodes))
    before = os.environ.get("LWSE_TICK_GRAPH")
    os.environ["LWSE_TICK_GRAPH"] = "0"  # read when an engine is created
    try:
        eng = Engine(0)
    finally:
        if before is None:
            del os.environ["LWSE_TICK_GRAPH"]
        else:
            os.environ["LWSE_TICK_GRAPH"] = before
    try:
        eng.upload_nodes(t.nodes, t.n_domains)
        eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        eng.resident_place_load(reqs, t.n_namespaces)
        place = t.flags | R.TICK_PLACE
        eng.resident_tick(eng.make_tick((), place))
        nodes = t.nodes.copy()
        rng = np.random.default_rng(31)
        arena = Arena(eng)
        for k in range(8):
            # cordon (or uncordon) whole domains, so that the next round's index differs a lot
            doms = rng.choice(t.n_domains, size=40, replace=False)
            rows = np.flatnonzero(np.isin(nodes["domain_id"], doms)).astype(np.uint32)
            vals = R.aligned_empty(len(rows), R.NODE_REC)
            vals[:] = nodes[rows]
            vals["flags"] ^= np.uint16(R.NODE_SCHEDULABLE)
            nodes[rows] = vals
            a = eng.make_tick(arena.put([(R.TABLE_NODES, rows, vals)], 0), t.flags)  # sweep only, no round
            b = eng.make_tick((), place)
            if k % 2 == 0:
                eng.resident_tick_submit(a)
                eng.resident_tick_submit(b)  # while the first one is still in flight
                eng.resident_tick_wait()
                eng.resident_tick_wait()
            else:
                eng.resident_tick(a)
                eng.resident_tick(b)
            assert eng.resident_node_info()["index_built"], k
            want = oracle.place(nodes, occ, t.n_domains, t.n_namespaces, reqs, threads=16)
            assert eng.resident_place_outputs().tobytes() == want.tobytes(), k
    finally:
        eng.close()


def _edge_setup(engine, n_nodes=400, spare=0):
    import oracle  # noqa: F401  (built by the session)
    from informer_world import make_world

    items, cluster = make_world(0, n_lws=6, n_nodes=n_nodes)
    enc = informer.IncrementalEncoder(items, cluster, "zone", node_spare=spare)
    lws, groups, pst, pid, reqs = enc.full_tables()
    rng = np.random.default_rng(4)
    n = 2000
    big = R.aligned_empty(n, R.PLACE_REQ)
    big["ns"] = rng.choice([0, 0, 1, 2], size=n)
    big["priority"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    big["group_key"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    big["group"] = np.arange(n)
    big["size"] = rng.integers(0, 6, size=n)
    big["leader_node"] = np.where(rng.random(n) < 0.2, rng.integers(0, len(enc.node_rec), size=n), R.NONE).astype(np.uint32)
    big = big[np.argsort(big["ns"], kind="stable")].copy()
    engine.upload_nodes(enc.node_rec, enc.n_domains)
    engine.resident_load(lws, groups, pst, pid)
    engine.resident_place_load(big, 3)
    return enc, big, R.occupancy_of(pid, len(enc.node_rec))


@pytest.mark.parametrize("scan", [False, True], ids=["two_level", "scan"])
def test_node_patch_edge_cases(engine, scan):
    """Every node unusable (a LWSE_PATCH_RANGE segment), a domain id >= n_domains, lwse_resident_patch of node
    rows, and the general form (lwse_place_host on an ungrouped table) reading the rebuilt index."""
    import oracle

    enc, reqs, occ = _edge_setup(engine)
    nodes = enc.node_rec.copy()
    n_dom = enc.n_domains
    flags = R.TICK_PLACE | (R.SWEEP_PLACE_SCAN if scan else 0)

    def tick_and_check(segs, where):
        engine.resident_tick(engine.make_tick(segs, flags))
        want = oracle.place(nodes, occ, n_dom, 3, reqs)
        assert engine.resident_place_outputs().tobytes() == want.tobytes(), where
        return engine.resident_node_info()

    # every node unusable: one range segment over the whole table
    off = nodes.copy()
    off["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
    saved, nodes[:] = nodes.copy(), off
    ni = tick_and_check([(R.TABLE_NODES, 0, off, True)], "all cordoned")
    assert ni["index_built"] and ni["n_usable"] == 0
    assert (engine.resident_place_outputs()["flags"][(reqs["size"] >= 1) & (reqs["leader_node"] == R.NONE)]
            & R.PLACE_UNSCHEDULABLE).all()
    nodes[:] = saved
    ni = tick_and_check([(R.TABLE_NODES, 0, saved, True)], "all back")
    assert ni["index_built"] and ni["n_usable"] == usable_count(saved, n_dom)
    # a domain id beyond n_domains: the node is not usable (nor a pinned leader's domain)
    rows = np.flatnonzero(usable_mask(nodes, n_dom))[:5].astype(np.uint32)
    vals = R.aligned_empty(len(rows), R.NODE_REC)
    vals[:] = nodes[rows]
    vals["domain_id"] = n_dom + 3
    nodes[rows] = vals
    ni = tick_and_check([(R.TABLE_NODES, rows, vals)], "domain out of range")
    assert ni["index_built"] and ni["n_usable"] == usable_count(nodes, n_dom)
    # the synchronous patch: the next round rebuilds the index
    rows2 = np.flatnonzero(~usable_mask(nodes, n_dom) & ((nodes["flags"] & R.NODE_HAS_TOPOLOGY) != 0))[:3].astype(np.uint32)
    vals2 = R.aligned_empty(len(rows2), R.NODE_REC)
    vals2[:] = nodes[rows2]
    vals2["flags"] |= R.NODE_SCHEDULABLE
    vals2["domain_id"] = np.minimum(vals2["domain_id"], n_dom - 1)
    engine.resident_patch(R.TABLE_NODES, rows2, vals2)
    nodes[rows2] = vals2
    ni = tick_and_check([], "after lwse_resident_patch")
    assert ni["index_built"] and ni["rows_patched"] == 0
    ni = tick_and_check([], "steady")
    assert not ni["index_built"]
    # the general form (an ungrouped table through lwse_place_host) on the rebuilt index
    rows3 = rows[:2]
    vals3 = R.aligned_empty(len(rows3), R.NODE_REC)
    vals3[:] = saved[rows3]
    engine.resident_patch(R.TABLE_NODES, rows3, vals3)
    nodes[rows3] = vals3
    shuffled = reqs[np.random.default_rng(1).permutation(len(reqs))].copy()
    got, _ = engine.place_host(shuffled, occ, 3)
    assert got.tobytes() == oracle.place(nodes, occ, n_dom, 3, shuffled).tobytes()


def test_upload_more_nodes_after_resident_load(engine):
    """lwse_upload_nodes with more nodes after lwse_resident_load: the occupancy is recounted for the new
    table, and the following ticks are exact."""
    import oracle

    enc, reqs, _ = _edge_setup(engine, n_nodes=300)
    grown = R.aligned_empty(len(enc.node_rec) + 700, R.NODE_REC)
    grown[: len(enc.node_rec)] = enc.node_rec
    rng = np.random.default_rng(8)
    grown["capacity"][len(enc.node_rec):] = rng.integers(1, 12, size=700)
    grown["flags"][len(enc.node_rec):] = R.NODE_SCHEDULABLE | R.NODE_HAS_TOPOLOGY
    grown["domain_id"][len(enc.node_rec):] = rng.integers(0, enc.n_domains, size=700)
    engine.upload_nodes(grown, enc.n_domains)
    occ = R.occupancy_of(enc.pod_ident, len(grown))
    assert np.array_equal(engine.resident_occupancy(), occ)
    flags = R.SWEEP_GANG | R.TICK_PLACE
    for k in range(3):
        rows = rng.choice(len(grown), size=20, replace=False).astype(np.uint32)
        rows.sort()
        vals = R.aligned_empty(len(rows), R.NODE_REC)
        vals[:] = grown[rows]
        vals["capacity"] = rng.integers(0, 12, size=len(rows))
        grown[rows] = vals
        engine.resident_tick(engine.make_tick([(R.TABLE_NODES, rows, vals)], flags))
        want = oracle.place(grown, occ, enc.n_domains, 3, reqs)
        assert engine.resident_place_outputs().tobytes() == want.tobytes(), k
        assert np.array_equal(engine.resident_occupancy(), occ), k
    _, w_go, _ = oracle.sweep_lws(enc.lws, enc.groups, enc.pod_state, enc.pod_ident, grown, flags=R.SWEEP_GANG)
    assert engine.resident_outputs()[1].tobytes() == w_go.tobytes()
