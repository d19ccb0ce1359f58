"""The DS drain edge worlds (tests/ds_drain_edges_world.py) on the device: both calls byte for byte against the
definitions — ``ds_drain_ref`` (set form, with the after sweep's full role_out / revrole_out on the small worlds)
and ``ds_drain_cost_ref`` or its vectorised restatement (per key, both scopes) — and per-key rows against set-form
calls on sampled keys; change-list capacities around the touched count with a host guard past them; scratch that
shrinks and grows on one engine; and the three refusals' return codes, an untouched ``out`` and a correct answer
from the same engine after each.  ``-k "not entries_2gib"`` deselects the refusal that needs about 1 GiB of index
counting over 3.25 million DS."""
import ctypes as C

import numpy as np
import pytest

import ds_drain_edges_world as X
from ds_drain_ref import (COST_FIELDS, cost_row_of, ds_drain_cost_ref, ds_drain_domains_ref, ds_drain_ref, ds_drain_world,
                          ds_ok)
from lws_b200 import engine as E
from lws_b200 import records as R
from test_gpu_ds_drain import check_set, load

pytestmark = pytest.mark.gpu

ERR_OOM = -4
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def check_cost(engine, w, vec=False):
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_ds_drain_cost(scope)
        want = X.ds_drain_cost_vec(w, by_domain) if vec else ds_drain_cost_ref(w, by_domain)
        assert got.tobytes() == want.tobytes(), scope
        yield scope, got


def check_keys(engine, w, cost, nodes, domains, outputs=False):
    """Set-form calls for ``nodes`` and ``domains`` against the reference and against their per-key rows."""
    for n in nodes:
        got = engine.resident_ds_drain(nodes=[int(n)], outputs=outputs)
        check_set(got, ds_drain_ref(w, [int(n)]), ("node", int(n)), outputs=outputs)
        assert {f: int(cost["nodes"][f][n]) for f in COST_FIELDS} == cost_row_of(got), ("node", int(n))
    for d in domains:
        got = engine.resident_ds_drain(domains=[int(d)], outputs=outputs)
        check_set(got, ds_drain_domains_ref(w, [int(d)]), ("domain", int(d)), outputs=outputs)
        assert {f: int(cost["domains"][f][d]) for f in COST_FIELDS} == cost_row_of(got), ("domain", int(d))


@pytest.mark.parametrize("label", X.SMALL)
def test_small_world(engine, label):
    """Every case node (every node on the child-edge world), both per-key forms against ds_drain_cost_ref, and the
    all-domain drain; the scan worlds run from 2 049 LWS rows down to 1 023 on one engine, so that first[n_lws]
    would be stale from the larger world if the scan did not write it."""
    e = X.world(label)
    w = e.w
    load(engine, w)
    cost = dict(check_cost(engine, w))
    if label == "child_edges":
        nodes, domains = range(len(w.nodes)), range(w.n_domains)
    else:
        nodes = sorted({c.node for c in e.cases})
        domains = sorted({int(w.nodes["domain_id"][n]) for n in nodes})
    check_keys(engine, w, cost, nodes, domains, outputs=True)
    got = engine.resident_ds_drain(domains=list(range(w.n_domains)), outputs=True)
    check_set(got, ds_drain_domains_ref(w, list(range(w.n_domains))), "all", outputs=True)


def raw_rows(engine, nodes, capacity, guard=64):
    """lwse_resident_ds_drain into a host buffer of capacity + guard rows filled with SENTINEL."""
    buf = R.aligned_empty(capacity + guard, R.DS_DRAIN)
    buf.view(np.uint8)[:] = SENTINEL
    ids = np.ascontiguousarray(nodes, np.uint32)
    q = R.DsDrainQuery()
    q.ids, q.n_ids, q.scope, q.capacity, q.rows = R.ptr(ids), len(ids), R.DRAIN_NODES, capacity, R.ptr(buf)
    assert E.lib().lwse_resident_ds_drain(engine._h, C.byref(q)) == 0
    return q, buf


def test_fan_100k_and_capacities(engine):
    """~100 000 rows over 9 968 DS linked to one child: one insert thread walks them all.  Draining its node touches
    every DS; the change list at capacities around that count lists rows equal to the reference's, and no row past
    the listed ones is written."""
    e = X.world("fan_100k")
    w = e.w
    load(engine, w)
    cost = dict(check_cost(engine, w))
    rows, totals, _, _ = ref = ds_drain_ref(w, [0])
    check_set(engine.resident_ds_drain(nodes=[0], outputs=True), ref, "fan", outputs=True)
    assert {f: int(cost["nodes"][f][0]) for f in COST_FIELDS} == cost_row_of(totals)
    n_ds, n_touched = len(w.ds), totals["n_touched"]
    assert n_touched == n_ds
    for cap in sorted({n_touched - 1, n_touched, n_touched + 1, 31, 32, 33, n_ds, n_ds + 1}):
        q, buf = raw_rows(engine, [0], cap)
        listed = min(n_touched, cap)
        assert q.n_touched == n_touched and all(getattr(q, k) == totals[k] for k in R.DS_DRAIN_TOTALS), cap
        got = buf[:listed]
        assert len(np.unique(got["ds"])) == listed, cap
        assert got.tobytes() == rows[np.searchsorted(rows["ds"], got["ds"])].tobytes(), cap
        assert (buf[listed:].view(np.uint8) == SENTINEL).all(), cap


def test_grid_ds(engine, sm_count):
    """16 x 128 x SMs + 37 one-role DS: touched DS in the last stride, on both sides of a warp boundary."""
    e = X.grid_ds_world(sm_count)
    w = e.w
    load(engine, w)
    cost = dict(check_cost(engine, w, vec=True))
    nodes = [c.node for c in e.cases]
    check_keys(engine, w, cost, nodes, sorted({int(w.nodes["domain_id"][n]) for n in nodes}), outputs=True)
    got = engine.resident_ds_drain(nodes=[e.cases[0].node])
    assert sorted(got["rows"]["ds"].tolist()) == [e.notes["G"] + 31, e.notes["G"] + 32]


def test_grid_links(engine, sm_count):
    """One DS per child of grid_world(SMs, "groups"): the lost kernel's last stride, (LWS, key) and (DS, key) tables
    past the pairs, insert and finish grids."""
    e = X.world(f"grid_links_{sm_count}")
    w = e.w
    load(engine, w)
    cost = dict(check_cost(engine, w, vec=True))
    assert 2 * int(cost["nodes"]["ds_touched"].sum()) > X.cost_stride(sm_count)
    # (the set-form reference takes seconds per drain at this size: the case nodes and one domain)
    check_keys(engine, w, cost, [c.node for c in e.cases], [int(w.nodes["domain_id"][e.cases[0].node])], outputs=False)
    got = engine.resident_ds_drain(nodes=[e.cases[0].node])
    assert e.cases[0].ds in got["rows"]["ds"]


def small_check(engine, w):
    """Both calls on a small world, exact, with the full after outputs (rows no DS writes read 0)."""
    load(engine, w)
    for n in range(len(w.nodes)):
        check_set(engine.resident_ds_drain(nodes=[n], outputs=True), ds_drain_ref(w, [n]), ("small", n), outputs=True)
    list(check_cost(engine, w))


def test_scratch_shrinks_and_grows(engine, sm_count):
    small = ds_drain_world(n_ds=40, n_nodes=16, seed=41)
    assert not ds_ok(small.ds, len(small.roles), len(small.revroles)).all()  # (BAD_TABLE rows: outputs left 0)
    for step in range(3):
        if step == 1:
            small_check(engine, small)
            continue
        e = X.grid_ds_world(sm_count)
        load(engine, e.w)
        cost = dict(check_cost(engine, e.w, vec=True))
        check_keys(engine, e.w, cost, [e.cases[0].node], [], outputs=True)


def refused(engine, w, scope):
    """lwse_resident_ds_drain_cost on ``w``: its return code, and whether ``out`` kept its sentinel bytes."""
    load(engine, w)
    n = len(w.nodes) if scope == R.DRAIN_NODES else w.n_domains
    out = R.aligned_empty(n, R.DS_DRAIN_COST)
    out.view(np.uint8)[:] = SENTINEL
    rc = E.lib().lwse_resident_ds_drain_cost(engine._h, scope, R.ptr(out))
    return rc, bool((out.view(np.uint8) == SENTINEL).all())


def test_refuse_ds_pairs(engine):
    """3 178 DS x 330 rows x 1 024 nodes = 1 073 909 760 (DS, key) pairs > 2^30 for the node scope."""
    assert refused(engine, X.refuse_pairs_world().w, R.DRAIN_NODES) == (ERR_OOM, True)
    small_check(engine, ds_drain_world(n_ds=40, n_nodes=16, seed=41))


def test_refuse_entries_2gib(engine):
    """3 253 764 DS x 330 linked rows = 1 073 742 120 reverse-index entries > 2^30, in both scopes."""
    w = X.refuse_entries_world().w
    assert refused(engine, w, R.DRAIN_NODES) == (ERR_OOM, True)
    out = R.aligned_empty(w.n_domains, R.DS_DRAIN_COST)
    out.view(np.uint8)[:] = SENTINEL
    assert E.lib().lwse_resident_ds_drain_cost(engine._h, R.DRAIN_DOMAINS, R.ptr(out)) == ERR_OOM
    assert (out.view(np.uint8) == SENTINEL).all()
    del w
    small_check(engine, ds_drain_world(n_ds=40, n_nodes=16, seed=41))
