"""Placement what-if (lwse_resident_place_whatif) without a GPU: the numpy / oracle reference the GPU tests
compare against, and the informer's what-if builders — exact rows, and no encoder state changes."""
import copy

import numpy as np
import pytest

from lws_b200 import api, encoder, informer
from lws_b200 import records as R


def apply_segments(nodes, reqs, segs):
    """Host copies of the node and request tables with `segs` applied ((table, rows, values), or
    (table, first_row, values, True) for a range): ranges first, then the scattered rows, as a tick."""
    nodes, reqs = nodes.copy(), reqs.copy()
    tables = {R.TABLE_NODES: nodes, R.TABLE_PLACE_REQS: reqs}
    for sg in segs:
        if len(sg) == 4 and sg[3]:
            tables[sg[0]][int(sg[1]): int(sg[1]) + len(sg[2])] = sg[2]
    for sg in segs:
        if not (len(sg) == 4 and sg[3]):
            tables[sg[0]][np.asarray(sg[1], dtype=np.int64)] = sg[2]
    return nodes, reqs


def whatif_ref(nodes, occ, n_domains, reqs, segs=(), extra=None, n_ns=None, base_n_ns=None, threads=16):
    """The what-if by its definition: the spec oracle over the patched tables plus the extra rows, diffed
    against the spec oracle over the tables as they are (``base_n_ns`` namespaces, default ``n_ns``)."""
    import oracle

    base_n_ns = n_ns if base_n_ns is None else base_n_ns
    before = oracle.place(nodes, occ, n_domains, base_n_ns, reqs, threads=threads)
    p_nodes, p_reqs = apply_segments(nodes, reqs, segs)
    extra = R.aligned_empty(0, R.PLACE_REQ) if extra is None else extra
    all_reqs = R.aligned_empty(len(reqs) + len(extra), R.PLACE_REQ)
    all_reqs[: len(reqs)] = p_reqs
    all_reqs[len(reqs):] = extra
    after_all = oracle.place(p_nodes, occ, n_domains, n_ns, all_reqs, threads=threads)
    after = after_all[: len(reqs)]
    a = before.view(np.uint8).reshape(len(reqs), 16)
    b = after.view(np.uint8).reshape(len(reqs), 16)
    rows = np.flatnonzero((a != b).any(axis=1)).astype(np.uint32)
    was = (before["flags"] & R.PLACE_PLACED) != 0
    now = (after["flags"] & R.PLACE_PLACED) != 0
    f = after_all["flags"]
    return {
        "after_all": after_all, "rows": rows, "before": before[rows], "after": after[rows],
        "extra_out": after_all[len(reqs):],
        "n_changed": len(rows), "n_lost": int((was & ~now).sum()),
        "n_moved": int((was & now & (before["domain_id"] != after["domain_id"])).sum()),
        "n_gained": int((~was & now).sum()), "n_placed": int(((f & R.PLACE_PLACED) != 0).sum()),
        "n_unschedulable": int(((f & R.PLACE_UNSCHEDULABLE) != 0).sum()),
        "n_conflict": int(((f & R.PLACE_CONFLICT) != 0).sum()),
    }


def _same(a, b) -> bool:
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, dict):
        return isinstance(b, dict) and list(a) == list(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if hasattr(a, "__dict__") and not isinstance(a, type):
        return type(a) is type(b) and _same(vars(a), vars(b))
    return a == b


@pytest.fixture()
def world():
    from informer_world import make_world

    items, cluster = make_world(7, n_lws=18, n_nodes=40)
    enc = informer.IncrementalEncoder(items, cluster, "zone", spare=1.0, node_spare=8)
    return items, cluster, enc


def _exclusive_key(enc):
    return next(k for k in enc.order if int(enc.lws["flags"][enc.slots[k].lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY)


def test_builders_change_no_encoder_state(world):
    items, _, enc = world
    key = _exclusive_key(enc)
    node_names = list(enc.node_index)[:3]
    fresh = copy.deepcopy(items[0])
    fresh.lws.name, fresh.lws.namespace = "brand-new", "ns-unseen"
    before = copy.deepcopy(vars(enc))
    enc.whatif_cordon(node_names)
    enc.whatif_capacity(node_names[0], 3)
    enc.whatif_new_lws(fresh)
    enc.whatif_scale(key, enc.items[key].lws.replicas + 3)
    after = vars(enc)
    assert list(before) == list(after)
    for k in before:
        assert _same(before[k], after[k]), k


def test_node_builders(world):
    _, _, enc = world
    names = list(enc.node_index)[2:6]
    table, rows, vals = enc.whatif_cordon(names)
    assert table == R.TABLE_NODES and rows.dtype == np.uint32 and vals.dtype == R.NODE_REC
    assert sorted(rows.tolist()) == sorted(enc.node_index[n] for n in names)
    want = enc.node_rec[rows].copy()
    assert not (vals["flags"] & R.NODE_SCHEDULABLE).any()
    for f in ("capacity", "domain_id"):
        assert np.array_equal(vals[f], want[f])
    assert np.array_equal(vals["flags"] | R.NODE_SCHEDULABLE, want["flags"] | R.NODE_SCHEDULABLE)
    table, rows, vals = enc.whatif_capacity(names[0], 5)
    assert rows.tolist() == [enc.node_index[names[0]]] and int(vals["capacity"][0]) == 5
    assert vals["flags"][0] == enc.node_rec[rows[0]]["flags"] and vals["domain_id"][0] == enc.node_rec[rows[0]]["domain_id"]


def test_whatif_scale_matches_the_flushed_rows(world):
    """The rows whatif_scale builds equal, field for field apart from ``group`` (the row id), the request rows
    the informer emits once the scale event and the new groups' leader pods (not yet scheduled) are flushed."""
    _, _, enc = world
    key = _exclusive_key(enc)
    it = copy.deepcopy(enc.items[key])
    old, new = it.lws.replicas, it.lws.replicas + 3
    want = enc.whatif_scale(key, new)
    assert len(want) == new - old
    it.lws.replicas = new
    enc.lws_event("MODIFIED", it)
    for g in range(old, new):
        enc.pod_event("ADDED", api.Pod(name=f"{it.lws.name}-{g}", namespace=it.lws.namespace, phase="Pending",
                                       labels={api.SetNameLabelKey: it.lws.name, api.GroupIndexLabelKey: str(g),
                                               api.WorkerIndexLabelKey: "0", api.RevisionKey: it.revision_key}))
    enc.flush()
    assert not enc.needs_reload
    got = enc.reqs[[enc.group_row(key[0], key[1], g) for g in range(old, new)]]
    for f in R.PLACE_REQ.names:
        if f != "group":
            assert np.array_equal(got[f], want[f]), f


def test_whatif_new_lws_matches_a_created_object(world):
    """A new object in a namespace the encoder has not seen: the provisional namespace id is the one the
    next flush gives it, and the rows equal those the informer emits once its leader pods exist."""
    items, _, enc = world
    src = next(it for it in items if api.ExclusiveKeyAnnotationKey in it.lws.annotations)
    it = copy.deepcopy(src)
    it.lws.name, it.lws.namespace, it.lws.replicas = "whatif-new", "ns-unseen", 4
    it.leader_sts = None
    want, n_ns = enc.whatif_new_lws(it)
    assert len(want) == 4 and n_ns >= int(want["ns"][0]) + 1
    assert int(want["ns"][0]) not in enc.ns_ids.values()
    enc.lws_event("ADDED", it)
    for g in range(4):
        enc.pod_event("ADDED", api.Pod(name=f"{it.lws.name}-{g}", namespace=it.lws.namespace, phase="Pending",
                                       labels={api.SetNameLabelKey: it.lws.name, api.GroupIndexLabelKey: str(g),
                                               api.WorkerIndexLabelKey: "0", api.RevisionKey: it.revision_key}))
    enc.flush()
    assert not enc.needs_reload
    key = (it.lws.namespace, it.lws.name)
    got = enc.reqs[[enc.group_row(key[0], key[1], g) for g in range(4)]]
    for f in R.PLACE_REQ.names:
        if f != "group":
            assert np.array_equal(got[f], want[f]), f


def test_non_exclusive_objects_make_no_rows(world):
    items, _, enc = world
    key = next(k for k in enc.order if not int(enc.lws["flags"][enc.slots[k].lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY)
    assert len(enc.whatif_scale(key, 9)) == 0
    it = copy.deepcopy(enc.items[key])
    it.lws.name = "plain-new"
    rows, _ = enc.whatif_new_lws(it)
    assert len(rows) == 0


def test_reference_on_a_small_table():
    """whatif_ref: no patches and no extra rows change nothing; a cordon of every node unschedules every
    unpinned request; the extra rows alone take part in their own namespace."""
    from informer_world import make_world

    items, cluster = make_world(3, n_lws=12, n_nodes=24)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    reqs = enc.reqs
    occ = R.occupancy_of(enc.pod_ident, len(enc.node_rec))
    ref = whatif_ref(enc.node_rec, occ, enc.n_domains, reqs, n_ns=enc.n_namespaces)
    assert ref["n_changed"] == 0 and len(ref["extra_out"]) == 0
    seg = enc.whatif_cordon(list(enc.node_index))
    ref = whatif_ref(enc.node_rec, occ, enc.n_domains, reqs, [seg], n_ns=enc.n_namespaces)
    live = (reqs["size"] >= 1) & (reqs["leader_node"] == R.NONE)
    assert (ref["after_all"]["flags"][: len(reqs)][live] & R.PLACE_UNSCHEDULABLE).all()
    assert ref["n_gained"] == 0
    it = copy.deepcopy(next(i for i in items if api.ExclusiveKeyAnnotationKey in i.lws.annotations))
    it.lws.name, it.lws.namespace, it.lws.size, it.lws.replicas = "probe", "ns-probe", 1, 2
    extra, n_ns = enc.whatif_new_lws(it)
    ref = whatif_ref(enc.node_rec, occ, enc.n_domains, reqs, (), extra, n_ns=n_ns, base_n_ns=enc.n_namespaces)
    assert ref["n_changed"] == 0 and len(ref["extra_out"]) == 2
    assert (ref["extra_out"]["flags"] & R.PLACE_PLACED).all()
