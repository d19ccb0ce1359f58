"""LeaderWorkerSet ADDED / DELETED through the incremental encoder: new objects take spare rows and
deleted ones give theirs back, by row patches only.  After every flush the patched tables give the
oracle exactly what a fresh encode of the same objects gives, by name, and the row → object maps
agree with the slots; a reload is asked for exactly when a new object does not fit."""
import numpy as np
import pytest

import oracle
from informer_world import make_world, outputs_by_name
from lifecycle_world import LifecycleWorld
from lws_b200 import encoder, informer
from lws_b200 import records as R

BY_TABLE = {R.TABLE_LWS: 0, R.TABLE_GROUPS: 1, R.TABLE_POD_STATE: 2, R.TABLE_POD_IDENT: 3, R.TABLE_PLACE_REQS: 4}


def check_against_fresh(world, enc, mirror, where):
    items = list(world.items.values())
    ft = encoder.encode_lws(items, world.cluster(), "zone")
    w_lo, w_go, _ = oracle.sweep_lws(ft.lws, ft.groups, ft.pod_state, ft.pod_ident, ft.nodes, flags=R.SWEEP_GANG)
    want_l, want_g = outputs_by_name(ft.lws, ft.groups, w_lo, w_go,
                                     {i: (it.lws.namespace, it.lws.name) for i, it in enumerate(items)})
    lws, groups, pst, pid, _ = mirror
    g_lo, g_go, _ = oracle.sweep_lws(lws, groups, pst, pid, enc.node_rec, flags=R.SWEEP_GANG)
    got_l, got_g = outputs_by_name(lws, groups, g_lo, g_go, {sl.lws_row: key for key, sl in enc.slots.items()})
    assert set(enc.slots) == set(world.items), where
    assert got_l == want_l, where
    assert got_g == want_g, where
    assert np.array_equal(R.occupancy_of(pid, len(enc.node_rec)), R.occupancy_of(ft.pod_ident, len(ft.nodes))), where


def check_row_maps(enc, where):
    lws = enc.lws
    owned = set()
    for key, sl in enc.slots.items():
        assert enc.object_of_lws_row(sl.lws_row) == key, where
        owned.add(sl.lws_row)
        n = int(lws["group_count"][sl.lws_row])
        assert int(lws["group_base"][sl.lws_row]) == sl.group_base, where
        for gi in range(sl.group_cap):
            want = (key[0], key[1], gi) if gi < n else None
            assert enc.object_of_group_row(sl.group_base + gi) == want, where
    for row in range(len(lws)):
        if row not in owned:
            assert enc.object_of_lws_row(row) is None, where
            assert lws[row].tobytes() == bytes(R.LWS_REC.itemsize), where  # vacant: all zero
    in_slots = np.zeros(len(enc.groups), bool)
    for sl in enc.slots.values():
        in_slots[sl.group_base: sl.group_base + sl.group_cap] = True
    for row in np.flatnonzero(~in_slots)[:64]:
        assert enc.object_of_group_row(int(row)) is None, where


def apply(mirror, patches):
    for table, rows, vals in patches.segments:
        assert len(np.unique(rows)) == len(rows)
        mirror[BY_TABLE[table]][rows] = vals


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_lifecycle_stream_equals_fresh_encode(seed):
    items, cluster = make_world(seed, n_lws=10)
    world = LifecycleWorld(items, cluster, seed + 20)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=3.0)
    mirror = [a.copy() for a in enc.full_tables()]
    created = deleted = 0
    for tick in range(50):
        n_before = len(world.items)
        for _ in range(int(world.rng.integers(1, 6))):
            world.step(enc)
        if tick % 7 == 3:  # delete and re-create under the same name inside one flush
            key = world.delete(enc)
            if key is not None:
                world.create(enc, ns=key[0], name=key[1])
                created += 1
                deleted += 1
        created += max(0, len(world.items) - n_before)
        deleted += max(0, n_before - len(world.items))
        patches = enc.flush()
        assert not enc.needs_reload, f"tick {tick}"
        apply(mirror, patches)
        for a, b in zip(mirror, enc.full_tables()):
            assert a.tobytes() == b.tobytes(), f"tick {tick}"  # the patches carry every change
        check_against_fresh(world, enc, mirror, f"tick {tick}")
        check_row_maps(enc, f"tick {tick}")
        # every live request row carries its object's namespace id; rows of a namespace need not be adjacent
        reqs = enc.reqs
        for key, sl in enc.slots.items():
            assert (reqs["ns"][sl.req_base: sl.req_base + sl.group_cap] == enc.ns_ids[key[0]]).all()
    assert created > 0 and deleted > 0
    assert any(k[0].startswith("ns-new") for k in enc.slots) or any(k.startswith("ns-new") for k in enc.ns_ids)


def test_pods_before_their_set_are_encoded_with_it():
    items, cluster = make_world(3, n_lws=4)
    world = LifecycleWorld(items, cluster, 5)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone")
    mirror = [a.copy() for a in enc.full_tables()]
    from lifecycle_world import new_object

    item, pods, stss = new_object(world.rng, "early", "ns-1", len(world.nodes), exclusive=True, size=2, replicas=3)
    world._deliver(enc, pods, stss)
    apply(mirror, enc.flush())  # nothing to encode yet: the set is unknown
    assert ("ns-1", "early") not in enc.slots
    world.items[("ns-1", "early")] = item
    enc.lws_event("ADDED", item)
    apply(mirror, enc.flush())
    check_against_fresh(world, enc, mirror, "after ADDED")
    sl = enc.slots[("ns-1", "early")]
    assert int(enc.lws["group_count"][sl.lws_row]) == 3
    assert (enc.reqs["size"][sl.req_base: sl.req_base + 3] == 2).all()


def test_reload_exactly_when_a_create_does_not_fit():
    items, cluster = make_world(11, n_lws=6)
    world = LifecycleWorld(items, cluster, 12)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=0.25)
    caps = None
    for i in range(200):
        fits = caps is None or (enc.n_lws < len(enc.lws) and enc.g_end + caps[0] <= len(enc.groups)
                                and enc.p_end + caps[1] <= len(enc.pod_state))
        key = world.create(enc, ns="ns-0", name=f"extra-{i}", exclusive=True, size=2, replicas=2)
        enc.flush()
        assert enc.needs_reload == (not fits), f"create {i}"
        if enc.needs_reload:
            break
        sl = enc.slots[key]
        caps = (sl.group_cap, sl.pod_cap)
    assert enc.needs_reload
    # a reload lays the objects out in (namespace, name) order: the request table is grouped again
    re = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone")
    ns = re.reqs["ns"].astype(np.int64)
    assert np.all(np.diff(ns) >= 0)


def test_reload_when_namespace_ids_run_out():
    items, cluster = make_world(13, n_lws=4)
    world = LifecycleWorld(items, cluster, 14)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=4.0)
    n_ns = enc.n_namespaces
    for j in range(n_ns + 2):
        fits = len(enc.ns_ids) < n_ns  # the next new namespace takes id len(ns_ids)
        world.create(enc, ns=f"fresh-{j}", name="x", exclusive=False, size=1, replicas=1)
        enc.flush()
        assert enc.needs_reload == (not fits), f"namespace {j}"
        if enc.needs_reload:
            break
    assert enc.needs_reload


def test_churn_of_same_sized_objects_never_reloads():
    items, cluster = make_world(17, n_lws=8)
    world = LifecycleWorld(items, cluster, 18)
    for k in list(world.items):  # same-sized objects throughout
        world.items.pop(k)
    for i in range(8):
        world.create(informer.IncrementalEncoder([], world.cluster(), "zone"), ns=f"ns-{i % 3}", name=f"o{i}",
                     exclusive=i % 2 == 0, size=2, replicas=2)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone")
    mirror = [a.copy() for a in enc.full_tables()]
    for ev in range(1000):  # 1 000 deletions + 1 000 creations
        key = list(world.items)[int(world.rng.integers(0, len(world.items)))]
        world.delete(enc, key)
        world.create(enc, ns=f"ns-{int(world.rng.integers(0, 3))}", name=f"n{ev}", exclusive=bool(ev % 2), size=2, replicas=2)
        if ev % 3 == 2:
            apply(mirror, enc.flush())
            assert not enc.needs_reload, f"event {ev}"
    apply(mirror, enc.flush())
    assert not enc.needs_reload
    check_against_fresh(world, enc, mirror, "end")
    check_row_maps(enc, "end")
