"""Placement what-if on the device (lwse_resident_place_whatif) at C3 (10 000 nodes, 625 domains, 98 072
requests): every query against the spec reference of tests/test_place_whatif.py byte for byte, the same rows
and change list as a real tick with the same patches, the namespace subset, isolation from ticks in flight,
the general form, the error returns and a change buffer smaller than the change."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import synth
from lws_b200 import records as R
from test_gpu_lifecycle import ungroup
from test_gpu_node_events import Arena
from test_place_whatif import whatif_ref

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def c3():
    t = synth.make("C3", 1.0, seed=synth.SEED)
    return t, R.occupancy_of(t.pod_ident, len(t.nodes))


def load(engine, t, reqs, n_domains=None):
    engine.upload_nodes(t.nodes, n_domains or t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(reqs, t.n_namespaces)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))


def node_seg(nodes, rows, edit):
    rows = np.asarray(sorted(set(int(r) for r in rows)), dtype=np.uint32)
    vals = R.aligned_empty(len(rows), R.NODE_REC)
    vals[:] = nodes[rows]
    edit(vals)
    return (R.TABLE_NODES, rows, vals)


def req_seg(reqs, rows, edit):
    rows = np.asarray(rows, dtype=np.uint32)
    vals = R.aligned_empty(len(rows), R.PLACE_REQ)
    vals[:] = reqs[rows]
    edit(vals, rows)
    return (R.TABLE_PLACE_REQS, rows, vals)


def extra_rows(rng, n, ns, n_nodes, pinned=0.0):
    x = R.aligned_empty(n, R.PLACE_REQ)
    x["priority"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    x["group_key"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
    x["group"] = np.arange(n)
    x["ns"] = ns
    x["size"] = rng.integers(1, 5, size=n)
    x["leader_node"] = np.where(rng.random(n) < pinned, rng.integers(0, n_nodes, size=n), R.NONE).astype(np.uint32)
    return x


def queries(t, reqs, seed=5):
    """(name, segments, extra rows or None, n_namespaces or 0)."""
    rng = np.random.default_rng(seed)
    nodes, n_ns = t.nodes, t.n_namespaces
    big_ns = int(np.argmax(np.bincount(reqs["ns"].astype(np.int64), minlength=n_ns)))
    d = int(nodes["domain_id"][int(np.flatnonzero(nodes["flags"] & R.NODE_SCHEDULABLE)[0])])

    def cordon(v):
        v["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)

    def capacity(v):
        v["capacity"] = rng.integers(0, 16, size=len(v))

    def relabel(v):
        v["domain_id"] = (v["domain_id"] + 7) % t.n_domains

    pinned = np.flatnonzero((reqs["leader_node"] != R.NONE) & (reqs["size"] >= 1))
    live = np.flatnonzero(reqs["size"] >= 1)

    def unpin(v, rows):
        v["leader_node"] = R.NONE

    def move(v, rows):
        v["ns"] = (v["ns"] + 3) % n_ns

    def zero(v, rows):
        v[:] = np.zeros(len(v), R.PLACE_REQ)

    usable = np.flatnonzero((nodes["flags"] & R.NODE_SCHEDULABLE) != 0)
    q = [
        ("extra_one_ns", [], extra_rows(rng, 16, big_ns, len(nodes)), 0),
        ("extra_several_ns", [], extra_rows(rng, 40, rng.choice([1, 5, 9, big_ns], size=40), len(nodes), pinned=0.2), 0),
        ("extra_new_ns", [], extra_rows(rng, 24, n_ns, len(nodes)), n_ns + 1),
        ("cordon_domain", [node_seg(nodes, np.flatnonzero(nodes["domain_id"] == d), cordon)], None, 0),
        ("capacity_only", [node_seg(nodes, rng.choice(len(nodes), size=len(nodes) // 100, replace=False), capacity)], None, 0),
        ("relabel", [node_seg(nodes, usable[:1], relabel)], None, 0),
        ("unpin", [req_seg(reqs, pinned[:5], unpin)], None, 0),
        ("move_ns", [req_seg(reqs, live[10:13], move)], None, 0),
        ("zero_row", [req_seg(reqs, live[20:22], zero)], None, 0),
        ("requests_1pct", [req_seg(reqs, rng.choice(live, size=len(reqs) // 100, replace=False), unpin)], None, 0),
        ("combined", [node_seg(nodes, np.flatnonzero(nodes["domain_id"] == (d + 1) % t.n_domains), cordon),
                      req_seg(reqs, np.concatenate([pinned[5:8], live[30:32]]), move)],
         extra_rows(rng, 16, big_ns, len(nodes)), 0),
        ("combined_requests", [req_seg(reqs, pinned[8:12], unpin), req_seg(reqs, live[40:42], zero)],
         extra_rows(rng, 8, 2, len(nodes)), 0),
    ]
    return q


def touched_namespaces(reqs, segs, extra, n_ns, base_n_ns):
    ns = set(range(base_n_ns, n_ns))
    for sg in segs:
        if sg[0] == R.TABLE_PLACE_REQS:
            ns |= set(reqs["ns"][np.asarray(sg[1], dtype=np.int64)].tolist()) | set(sg[2]["ns"].tolist())
    if extra is not None:
        ns |= set(extra["ns"].tolist())
    return {v for v in ns if v < n_ns}


def check(got, ref, where):
    order = np.argsort(got["rows"], kind="stable")
    assert np.array_equal(got["rows"][order], ref["rows"]), f"{where}: changed rows"
    assert got["before"][order].tobytes() == ref["before"].tobytes(), f"{where}: before rows"
    assert got["after"][order].tobytes() == ref["after"].tobytes(), f"{where}: after rows"
    assert got["extra_out"].tobytes() == ref["extra_out"].tobytes(), f"{where}: extra rows"
    for k in R.PLACE_WHATIF[:-1]:
        assert got[k] == ref[k], f"{where}: {k} {got[k]} != {ref[k]}"


@pytest.mark.parametrize("table", ["grouped", "indexed"])
def test_queries_match_the_reference_and_the_tick(engine, c3, table):
    """Every query against the reference; each query without extra rows then runs as a real tick with the
    same segments, whose place rows equal ``after`` and whose change list equals ``rows``; a tick with the
    old values restores the tables before the next query."""
    t, occ = c3
    reqs = t.place_requests() if table == "grouped" else ungroup(t.place_requests())
    n_ns = t.n_namespaces
    load(engine, t, reqs)
    base = engine.resident_place_outputs().copy()
    flags = t.flags | R.TICK_PLACE
    for name, segs, extra, q_ns in queries(t, reqs):
        got = engine.resident_place_whatif(segs, extra, q_ns)
        ref = whatif_ref(t.nodes, occ, t.n_domains, reqs, segs, extra, n_ns=q_ns or n_ns, base_n_ns=n_ns)
        check(got, ref, name)
        assert got["form"] == "namespace", name
        nodes_patched = any(sg[0] == R.TABLE_NODES for sg in segs)
        want_solved = n_ns if nodes_patched else len(touched_namespaces(reqs, segs, extra, q_ns or n_ns, n_ns))
        assert got["namespaces_solved"] == want_solved, name
        assert engine.resident_place_outputs().tobytes() == base.tobytes(), name
        if extra is not None or q_ns:
            continue
        res = engine.resident_tick(engine.make_tick(segs, flags))
        assert sorted(res["place_rows"].tolist()) == ref["rows"].tolist(), f"{name}: tick change list"
        tick_rows = engine.resident_place_outputs()
        assert tick_rows.tobytes() == ref["after_all"].tobytes(), f"{name}: tick rows"
        undo = []
        for sg in segs:
            src = t.nodes if sg[0] == R.TABLE_NODES else reqs
            vals = R.aligned_empty(len(sg[1]), src.dtype)
            vals[:] = src[np.asarray(sg[1], dtype=np.int64)]
            undo.append((sg[0], sg[1], vals))
        engine.resident_tick(engine.make_tick(undo, flags))
        assert engine.resident_place_outputs().tobytes() == base.tobytes(), f"{name}: restored"


def test_namespace_subset_and_a_no_op_node_patch(engine, c3):
    """Without node patches only the touched namespaces are solved; with a node row rewritten with its own
    value every namespace is, and the rows are the same."""
    t, occ = c3
    reqs = t.place_requests()
    load(engine, t, reqs)
    rng = np.random.default_rng(9)
    extra = extra_rows(rng, 16, 3, len(t.nodes))
    live = np.flatnonzero(reqs["size"] >= 1)
    segs = [req_seg(reqs, live[100:104], lambda v, rows: v.__setitem__("size", v["size"] + 1))]
    got = engine.resident_place_whatif(segs, extra)
    ref = whatif_ref(t.nodes, occ, t.n_domains, reqs, segs, extra, n_ns=t.n_namespaces)
    check(got, ref, "subset")
    touched = touched_namespaces(reqs, segs, extra, t.n_namespaces, t.n_namespaces)
    assert got["namespaces_solved"] == len(touched) < t.n_namespaces
    noop = node_seg(t.nodes, [17], lambda v: None)
    got2 = engine.resident_place_whatif(segs + [noop], extra)
    check(got2, ref, "no-op node patch")
    assert got2["namespaces_solved"] == t.n_namespaces


def test_isolation_from_ticks_in_flight(engine, c3):
    """What-ifs between the submit and wait of two ticks in flight, and between graph-replayed ticks: every
    tick's change lists, the final rows, occupancy and node / tick info equal a run without what-ifs; an
    empty what-if reports no change (its snapshot orders behind the newest tick); a what-if that builds a
    node index leaves the next tick's index decision as it was."""
    t, occ = c3
    reqs = t.place_requests()
    flags = t.flags | R.TICK_PLACE
    rng = np.random.default_rng(11)
    sets = []
    for k in range(10):
        rows = rng.choice(len(t.nodes), size=100, replace=False)
        seg = node_seg(t.nodes, rows, lambda v: v.__setitem__("capacity", rng.integers(0, 16, size=len(v))))
        sets.append([seg])
    doms = rng.choice(t.n_domains, size=10, replace=False)

    def run(with_whatif):
        load(engine, t, reqs)
        arena = Arena(engine)
        out, infos, pending = [], [], 0

        def wait():
            r = engine.resident_tick_wait()
            out.append({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()})

        for k, segs in enumerate(sets):
            if pending == 2:
                wait()
                pending -= 1
            engine.resident_tick_submit(engine.make_tick(arena.put(segs, k & 1), flags))
            pending += 1
            info = (engine.resident_node_info(), engine.resident_tick_info())
            infos.append(info)
            if with_whatif:
                empty = engine.resident_place_whatif()
                assert empty["n_changed"] == 0, k
                cord = node_seg(t.nodes, np.flatnonzero(t.nodes["domain_id"] == doms[k]),
                                lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))
                engine.resident_place_whatif([cord], extra_rows(rng, 16, k % t.n_namespaces, len(t.nodes)))
                assert (engine.resident_node_info(), engine.resident_tick_info()) == info, k
        while pending:
            wait()
            pending -= 1
        return out, infos, engine.resident_place_outputs().copy(), engine.resident_occupancy().copy(), engine.resident_outputs()

    a_out, a_infos, a_rows, a_occ, a_res = run(True)
    b_out, b_infos, b_rows, b_occ, b_res = run(False)
    assert len(a_out) == len(b_out) == len(sets)
    for k, (x, y) in enumerate(zip(a_out, b_out)):
        for key in ("lws_rows", "group_rows", "place_rows"):
            ox, oy = np.argsort(x[key], kind="stable"), np.argsort(y[key], kind="stable")
            assert np.array_equal(x[key][ox], y[key][oy]), (k, key)
            out_key = key.replace("rows", "out")
            assert x[out_key][ox].tobytes() == y[out_key][oy].tobytes(), (k, out_key)
    assert a_infos == b_infos
    assert any(ti["graph"] for _, ti in a_infos)
    assert a_rows.tobytes() == b_rows.tobytes() and np.array_equal(a_occ, b_occ)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a_res, b_res))
    # a what-if that rebuilds the node index, then a tick without patches: no rebuild
    cord = node_seg(t.nodes, np.flatnonzero(t.nodes["domain_id"] == doms[0]),
                    lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))
    engine.resident_place_whatif([cord])
    engine.resident_tick(engine.make_tick((), flags))
    assert not engine.resident_node_info()["index_built"] and not engine.resident_tick_info()["index_built"]
    assert engine.resident_place_outputs().tobytes() == b_rows.tobytes()


def test_general_form(engine, c3):
    """More domain ids than one CTA's shared memory holds: the tick and the what-if run the general form."""
    t, occ = c3
    reqs = t.place_requests()
    load(engine, t, reqs, n_domains=8192)
    assert engine.resident_tick_info()["form"] == "general"
    rng = np.random.default_rng(13)
    d = int(t.nodes["domain_id"][0])
    segs = [node_seg(t.nodes, np.flatnonzero(t.nodes["domain_id"] == d),
                     lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))]
    for s, x in ((segs, None), ([], extra_rows(rng, 16, 0, len(t.nodes))), (segs, extra_rows(rng, 8, 4, len(t.nodes)))):
        got = engine.resident_place_whatif(s, x)
        ref = whatif_ref(t.nodes, occ, 8192, reqs, s, x, n_ns=t.n_namespaces)
        check(got, ref, "general")
        assert got["form"] == "general" and got["namespaces_solved"] == 0


def raw_query(engine, segs=(), n_extra=0, extra=None, capacity=0, rows=None, before=None, after=None, extra_out=None):
    from lws_b200.engine import lib

    tick = engine.make_tick(segs)
    q = R.PlaceWhatIf()
    q.segs = C.cast(tick.segs, C.c_void_p) if len(segs) else None
    q.n_segs = len(segs)
    q.extra, q.n_extra, q.extra_out = R.ptr(extra), n_extra, R.ptr(extra_out)
    q.capacity, q.rows, q.before, q.after = capacity, R.ptr(rows), R.ptr(before), R.ptr(after)
    return lib().lwse_resident_place_whatif(engine._h, C.byref(q)), q


def test_errors(c3):
    from lws_b200.engine import Engine, LwseError

    t, _ = c3
    reqs = t.place_requests()
    e = Engine(0)
    try:
        e.upload_nodes(t.nodes, t.n_domains)
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        assert raw_query(e)[0] == ERR_NOT_READY  # before the place load
        e.resident_place_load(reqs, t.n_namespaces)
        assert raw_query(e)[0] == ERR_NOT_READY  # before the first round
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        assert raw_query(e)[0] == 0
        # a table other than NODES / PLACE_REQS, a row out of range, NULL buffers with a count
        lws_vals = R.aligned_empty(1, R.LWS_REC)
        lws_vals[:] = t.lws[:1]
        assert raw_query(e, [(R.TABLE_LWS, np.zeros(1, np.uint32), lws_vals)])[0] == ERR_INVALID_ARG
        bad = node_seg(t.nodes, [3], lambda v: None)
        bad[1][0] = len(t.nodes) + 5
        assert raw_query(e, [bad])[0] == ERR_INVALID_ARG
        assert raw_query(e, n_extra=3)[0] == ERR_INVALID_ARG
        assert raw_query(e, capacity=4)[0] == ERR_INVALID_ARG
        # row keys are 24-bit
        x = R.aligned_empty(1, R.PLACE_REQ)
        out = R.aligned_empty(1, R.PLACE_OUT)
        assert raw_query(e, n_extra=(1 << 24) - len(reqs), extra=x, extra_out=out)[0] == ERR_UNSUPPORTED
        # request rows patched by a tick without a round: not ready until the next round
        seg = req_seg(reqs, [5], lambda v, rows: v.__setitem__("size", v["size"] + 1))
        e.resident_tick(e.make_tick([seg], R.TICK_NO_SWEEP))
        with pytest.raises(LwseError) as ei:
            e.resident_place_whatif()
        assert ei.value.status == ERR_NOT_READY
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        assert e.resident_place_whatif()["n_changed"] == 0
        # so does lwse_resident_patch of node rows
        e.resident_patch(R.TABLE_NODES, np.array([7], np.uint32), t.nodes[7:8])
        assert raw_query(e)[0] == ERR_NOT_READY
    finally:
        e.close()


def test_capacity_smaller_than_the_change(engine, c3):
    """capacity < n_changed: exactly `capacity` rows are listed, each one a real change, and nothing past the
    end of the buffers is written."""
    t, occ = c3
    reqs = t.place_requests()
    load(engine, t, reqs)
    d = int(t.nodes["domain_id"][5])
    segs = [node_seg(t.nodes, np.flatnonzero(np.isin(t.nodes["domain_id"], [d, (d + 1) % t.n_domains])),
                     lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))]
    ref = whatif_ref(t.nodes, occ, t.n_domains, reqs, segs, None, n_ns=t.n_namespaces)
    assert ref["n_changed"] > 8
    cap, guard = ref["n_changed"] // 2, 64
    rows = np.full(cap + guard, 0xABABABAB, np.uint32)
    before = R.aligned_empty(cap + guard, R.PLACE_OUT)
    after = R.aligned_empty(cap + guard, R.PLACE_OUT)
    before.view(np.uint32)[:] = 0xCDCDCDCD
    after.view(np.uint32)[:] = 0xEFEFEFEF
    rc, q = raw_query(engine, segs, capacity=cap, rows=rows, before=before, after=after)
    assert rc == 0 and q.n_changed == ref["n_changed"]
    assert (rows[cap:] == 0xABABABAB).all()
    assert (before[cap:].view(np.uint32) == 0xCDCDCDCD).all() and (after[cap:].view(np.uint32) == 0xEFEFEFEF).all()
    idx = np.searchsorted(ref["rows"], rows[:cap])
    assert len(set(rows[:cap].tolist())) == cap and np.array_equal(ref["rows"][idx], rows[:cap])
    assert before[:cap].tobytes() == ref["before"][idx].tobytes() and after[:cap].tobytes() == ref["after"][idx].tobytes()


def test_node_index_rebuilds_across_a_domain_growth(engine, c3):
    """A what-if that builds its own node index, then lwse_upload_nodes with a few more domain ids (some nodes
    relabelled into them), a tick, and another index-building what-if: the second build starts from clean
    per-domain counters, and both match the reference."""
    t, occ = c3
    reqs = t.place_requests()
    load(engine, t, reqs)

    def cordon(nodes, d):
        return node_seg(nodes, np.flatnonzero(nodes["domain_id"] == d),
                        lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))

    seg = cordon(t.nodes, 3)
    got = engine.resident_place_whatif([seg])
    check(got, whatif_ref(t.nodes, occ, t.n_domains, reqs, [seg], n_ns=t.n_namespaces), "before the growth")
    grown_dom = t.n_domains + 40
    nodes = t.nodes.copy()
    rng = np.random.default_rng(17)
    moved = rng.choice(np.flatnonzero((nodes["flags"] & R.NODE_HAS_TOPOLOGY) != 0), size=400, replace=False)
    nodes["domain_id"][moved] = rng.integers(t.n_domains, grown_dom, size=len(moved))
    engine.upload_nodes(nodes, grown_dom)
    from lws_b200.engine import LwseError

    with pytest.raises(LwseError):  # the rows of the last round belong to the old node table
        engine.resident_place_whatif()
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))
    assert engine.resident_place_outputs().tobytes() == whatif_ref(nodes, occ, grown_dom, reqs,
                                                                    n_ns=t.n_namespaces)["after_all"].tobytes()
    for d in (5, t.n_domains + 7):
        seg = cordon(nodes, d)
        got = engine.resident_place_whatif([seg])
        check(got, whatif_ref(nodes, occ, grown_dom, reqs, [seg], n_ns=t.n_namespaces), f"after the growth, domain {d}")


def test_empty_request_table_admission(c3):
    """An empty resident request table is ready after a tick with LWSE_TICK_PLACE: extra rows alone are
    solved against the resident nodes and occupancy, also after node patches made by such ticks."""
    import oracle
    from lws_b200.engine import Engine

    t, occ = c3
    e = Engine(0)
    try:
        e.upload_nodes(t.nodes, t.n_domains)
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        e.resident_place_load(R.aligned_empty(0, R.PLACE_REQ), t.n_namespaces)
        e.resident_tick(e.make_tick((), t.flags | R.TICK_PLACE))
        rng = np.random.default_rng(19)
        x = extra_rows(rng, 32, rng.integers(0, 4, size=32), len(t.nodes), pinned=0.2)
        got = e.resident_place_whatif((), x)
        assert got["n_changed"] == 0
        assert got["extra_out"].tobytes() == oracle.place(t.nodes, occ, t.n_domains, t.n_namespaces, x).tobytes()
        # a cordon through a tick (no round runs on an empty table: the resident index is left behind)
        nodes = t.nodes.copy()
        seg = node_seg(nodes, np.flatnonzero(nodes["domain_id"] == 2),
                       lambda v: v.__setitem__("flags", v["flags"] & ~np.uint16(R.NODE_SCHEDULABLE)))
        nodes[seg[1]] = seg[2]
        e.resident_tick(e.make_tick([seg], t.flags | R.TICK_PLACE))
        got = e.resident_place_whatif((), x)
        assert got["extra_out"].tobytes() == oracle.place(nodes, occ, t.n_domains, t.n_namespaces, x).tobytes()
    finally:
        e.close()
