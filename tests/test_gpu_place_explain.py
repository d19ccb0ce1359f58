"""Placement explanation on the device (lwse_resident_place_explain): byte for byte against tests/place_explain_ref.py
on the edge world and fuzz worlds, in the baseline and what-if forms (cordon segments with a node-index rebuild, extra
rows, new namespaces, extra rows on an empty request table, the general form, a list beyond the capacity); at C3 the
certificate on every row of a tick, and the reference on every UNSCHEDULABLE and CONFLICT row of a what-if with every
domain from 24 on cordoned (the C3 tick itself has no such row, so the what-if stands in for it); every stranding
rollout placement entry's E_i; a tick in flight; the refusals."""
import ctypes as C

import numpy as np
import pytest

from lws_b200 import synth
from lws_b200 import records as R
from place_explain_ref import certificate, cordon_seg, edge_world, explain_ref, extra_reqs, fuzz_world, pods_for

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY, ERR_UNSUPPORTED = -1, -6, -7
LWSE_TICK_MAX_SEGS = 8
ALL = R.PLACE_PLACED | R.PLACE_PINNED | R.PLACE_CONFLICT | R.PLACE_UNSCHEDULABLE


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


def load(engine, w, n_domains=None, reqs=None):
    pst, pid = pods_for(w.occ)
    engine.upload_nodes(w.nodes, n_domains or w.n_domains)
    engine.resident_load(R.aligned_empty(0, R.LWS_REC), R.aligned_empty(0, R.GROUP_REC), pst, pid)
    engine.resident_place_load(w.reqs if reqs is None else reqs, w.n_ns)
    engine.resident_tick(engine.make_tick((), R.TICK_PLACE))


def same(got, want, where):
    g, x = got["rows"], want["rows"]
    assert len(g) == len(x), f"{where}: {len(g)} rows, want {len(x)}"
    bad = np.flatnonzero((g.view(np.uint8).reshape(len(g), 64) != x.view(np.uint8).reshape(len(x), 64)).any(axis=1))
    assert len(bad) == 0, f"{where}: rows {bad[:8].tolist()} differ: got {g[bad[:2]]}, want {x[bad[:2]]}"
    for k in ("n_explained", "round_rows", "n_domains", "whatif", "classes", "flags"):
        assert got[k] == want[k], f"{where}: {k} {got[k]} != {want[k]}"


def both(engine, w, where, **kw):
    got = engine.resident_place_explain(**kw)
    want = explain_ref(w, **{("n_ns" if k == "n_namespaces" else k): v for k, v in kw.items()})
    same(got, want, where)
    return got, want


def test_edge_world_equals_the_reference(engine):
    w, rows = edge_world()
    load(engine, w)
    n = len(w.reqs)
    got, _ = both(engine, w, "every row", rows=list(range(n)))
    assert not got["whatif"] and got["form"] is None
    both(engine, w, "by mask")
    both(engine, w, "all by mask", mask=ALL)
    both(engine, w, "listed, repeated", rows=[rows["F5"], rows["B"], rows["F5"], rows["NS"]])
    both(engine, w, "beyond the capacity", mask=ALL, capacity=5)
    both(engine, w, "nothing listed", rows=[])
    got, _ = both(engine, w, "uncordoned", mask=ALL, segs=[cordon_seg(w.nodes, [8, 9], cordon=False)])
    assert got["whatif"] and got["form"] == "namespace"
    both(engine, w, "cordoned", mask=ALL, segs=[cordon_seg(w.nodes, [2, 3, 48, 49], cordon=True)])
    x = extra_reqs([(2, 5, 0), (4, 5, 0), (2, 9, 90), (6, 3, 0)])
    both(engine, w, "extra rows", rows=list(range(n, n + 4)), extra=x, n_namespaces=5)
    both(engine, w, "extra rows, every row", mask=ALL, extra=x)
    both(engine, w, "more namespaces", mask=ALL, n_namespaces=8)


def test_extra_rows_on_an_empty_request_table(engine):
    w, rows = edge_world()
    empty = type(w)(**{**vars(w), "reqs": R.aligned_empty(0, R.PLACE_REQ)})
    load(engine, empty)
    both(engine, empty, "baseline, empty", mask=ALL)
    both(engine, empty, "extra only", mask=ALL, extra=extra_reqs([(0, 5, 0), (0, 5, 1), (3, 20, 0)]))


def test_general_form(engine):
    w, rows = edge_world()
    big = type(w)(**{**vars(w), "n_domains": 5457})
    load(engine, big)
    both(engine, big, "general baseline", mask=ALL)
    got, _ = both(engine, big, "general what-if", mask=ALL, segs=[cordon_seg(w.nodes, [8, 9], cordon=False)],
                  extra=extra_reqs([(2, 5, 0)]))
    assert got["form"] == "general"


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_worlds_equal_the_reference(engine, seed):
    w = fuzz_world(seed)
    load(engine, w)
    got, want = both(engine, w, f"fuzz {seed}", mask=ALL)
    assert certificate({**want, "all_rows": got["rows"]}, w.n_ns, w.n_domains) == []
    seg = cordon_seg(w.nodes, range(0, len(w.nodes), 5), cordon=True)
    both(engine, w, f"fuzz {seed} what-if", mask=ALL, segs=[seg], extra=extra_reqs([(0, 3, 0), (w.n_ns, 2, 0)]),
         n_namespaces=w.n_ns + 1)


@pytest.fixture(scope="module")
def c3():
    from rollout_place_ref import world_of

    t = synth.make("C3", 1.0, seed=synth.SEED)
    return t, world_of(t)


def load_c3(engine, t, w):
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_place_load(w.reqs, w.n_ns)
    engine.resident_tick(engine.make_tick((), t.flags | R.TICK_PLACE))


def test_c3_certificate_on_every_row_and_the_stranded_rows(engine, c3):
    t, w = c3
    load_c3(engine, t, w)
    got = engine.resident_place_explain(mask=ALL)
    assert got["n_explained"] == len(w.reqs)
    assert not (got["rows"]["place_flags"] & (R.PLACE_UNSCHEDULABLE | R.PLACE_CONFLICT)).any()
    want = explain_ref(w, rows=[])  # (the round, without explaining a row on the host)
    assert certificate({**want, "all_rows": got["rows"]}, w.n_ns, w.n_domains) == []
    assert got["round_rows"] == len(w.reqs)
    # every UNSCHEDULABLE and CONFLICT row: the tick has none, so a what-if with most domains cordoned stands in
    seg = cordon_seg(w.nodes, np.flatnonzero(w.nodes["domain_id"] >= 24), cordon=True)
    got, want = both(engine, w, "C3 cordoned", segs=[seg])
    assert got["n_explained"] > 1000


def test_c3_rollout_strands_are_the_unschedulable_extra_rows(engine, c3):
    t, w = c3
    load_c3(engine, t, w)
    rows = np.flatnonzero(t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY).astype(np.uint32)[:40]
    ns = t.ns_of_lws[rows].astype(np.uint32)
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = t.lws[rows.astype(np.int64)]
    recs["replicas"] = recs["replicas"] + np.arange(len(rows)) * 20  # from no surge to more groups than domains
    rp = engine.resident_rollout_place(rows, ns, recs, extra=True)
    n_res, at, checked = len(w.reqs), 0, 0
    for e in rp["rows"]:
        k = int(e["surge"])
        if int(e["flags"]) & R.RPL_STRANDS:
            x = rp["extra"][at: at + k]
            got = engine.resident_place_explain(rows=list(range(n_res, n_res + k)), extra=x)
            assert int(((got["rows"]["place_flags"] & R.PLACE_UNSCHEDULABLE) != 0).sum()) == int(e["stranded"])
            checked += 1
        at += k
    assert checked > 0


def test_tick_in_flight_is_isolated(engine):
    w = fuzz_world(2)
    load(engine, w)
    prow = np.asarray([1, 5, 9], dtype=np.uint32)
    vals = R.aligned_empty(3, R.PLACE_REQ)
    vals[:] = w.reqs[prow]
    vals["leader_node"] = R.NONE
    seg = (R.TABLE_PLACE_REQS, prow, vals)
    t1 = engine.make_tick([seg], R.TICK_PLACE)
    engine.resident_tick_submit(t1)
    ref = engine.resident_tick_wait(t1)
    ref_list = (ref["n_place"], np.sort(ref["place_rows"]).tobytes())
    ref_out = engine.resident_place_outputs().copy()
    after = engine.resident_place_explain(mask=ALL)
    load(engine, w)
    t2 = engine.make_tick([seg], R.TICK_PLACE)
    engine.resident_tick_submit(t2)
    mid = engine.resident_place_explain(mask=ALL)  # behind the submitted tick
    mid_w = engine.resident_place_explain(mask=ALL, segs=[cordon_seg(w.nodes, [0, 1], cordon=True)])
    done = engine.resident_tick_wait(t2)
    assert (done["n_place"], np.sort(done["place_rows"]).tobytes()) == ref_list
    assert engine.resident_place_outputs().tobytes() == ref_out.tobytes()
    assert mid["rows"].tobytes() == after["rows"].tobytes()
    assert mid_w["whatif"]


def _raw(engine, rows=None, n_rows=None, out=None, capacity=4, mask=ALL, n_namespaces=0, segs=None, n_segs=0):
    from lws_b200.engine import lib

    q = R.PlaceExplainQuery()
    q.rows = R.ptr(rows) if rows is not None else None
    q.n_rows = (len(rows) if rows is not None else 0) if n_rows is None else n_rows
    q.mask, q.capacity, q.n_namespaces = mask, capacity, n_namespaces
    q.segs, q.n_segs = segs, n_segs
    o = R.aligned_empty(max(capacity, 1), R.PLACE_EXPLAIN) if out is None else out
    q.out = R.ptr(o) if out is not False else None
    q.n_explained = 0xABCD
    rc = lib().lwse_resident_place_explain(engine._h, C.byref(q))
    return rc, q


def test_refusals():
    from lws_b200.engine import Engine

    w, rows = edge_world()
    e = Engine(0)
    out = R.aligned_empty(4, R.PLACE_EXPLAIN)
    out["flags"] = 0xABCD
    try:
        assert _raw(e, out=out)[0] == ERR_NOT_READY  # nothing loaded
        pst, pid = pods_for(w.occ)
        e.upload_nodes(w.nodes, w.n_domains)
        e.resident_load(R.aligned_empty(0, R.LWS_REC), R.aligned_empty(0, R.GROUP_REC), pst, pid)
        assert _raw(e, out=out)[0] == ERR_NOT_READY  # no request table
        e.resident_place_load(w.reqs, w.n_ns)
        assert _raw(e, out=out)[0] == ERR_NOT_READY  # no round yet
        e.resident_tick(e.make_tick((), R.TICK_PLACE))
        rc, q = _raw(e, np.array([0, 1], np.uint32))
        assert rc == 0 and q.n_explained == 2
        for bad in (dict(rows=np.array([len(w.reqs)], np.uint32)), dict(rows=None, n_rows=3), dict(out=False),
                    dict(segs=None, n_segs=1), dict(n_segs=LWSE_TICK_MAX_SEGS + 1, segs=None)):
            rc, q = _raw(e, **{"out": out, **bad})
            assert rc == ERR_INVALID_ARG and q.n_explained == 0xABCD, bad
        assert (out["flags"] == 0xABCD).all()
        e.resident_patch(R.TABLE_PLACE_REQS, np.array([0], np.uint32), w.reqs[:1].copy())
        assert _raw(e, out=out)[0] == ERR_NOT_READY  # a patch without a round
        assert (out["flags"] == 0xABCD).all()
    finally:
        e.close()
    e = Engine(0)  # an engine with a peer exchange: refused
    try:
        load(e, w)
        assert _raw(e)[0] == 0
        e.exchange_create(len(w.reqs) + 1, 1, 0)
        assert _raw(e, out=out)[0] == ERR_UNSUPPORTED and (out["flags"] == 0xABCD).all()
    finally:
        e.close()

