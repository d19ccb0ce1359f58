"""Node ADDED / MODIFIED / DELETED through the incremental encoder: node rows are patched in place, new
nodes take spare rows and new topology values spare domain ids, and the objects with pods bound to an
added or deleted node's name are re-encoded in the same flush.  After every flush the tables equal a
fresh encode of the same cluster by name (node rows translated to node names, domain ids to label values,
because a fresh encode numbers both differently); a reload is asked for exactly when spare node rows or
domain ids run out."""
import numpy as np
import pytest

import oracle
from informer_world import make_world
from node_world import NodeWorld, nodes_by_name, occupancy_by_name
from lws_b200 import encoder, informer
from lws_b200 import records as R

BY_TABLE = {R.TABLE_LWS: 0, R.TABLE_GROUPS: 1, R.TABLE_POD_STATE: 2, R.TABLE_POD_IDENT: 3, R.TABLE_PLACE_REQS: 4,
            R.TABLE_NODES: 5}


def _node_of(row, names_of_row):
    if row == R.NONE or row == R.NODE_NOT_FOUND:
        return int(row)
    return names_of_row.get(int(row), ("vacant", int(row)))


def objects_by_name(lws, groups, pst, pid, reqs, lws_key, names_of_row, domain_values, g_out):
    """{object: (lws row, [(group row, leader node name, domain value, [pods])], {group index: request})} with
    every row number replaced by what it stands for; `g_out`: the oracle's group results of these tables."""
    out = {}
    for row, key in lws_key.items():
        l = lws[row].copy()
        base, count = int(l["group_base"]), int(l["group_count"])
        l["group_base"] = 0
        grp = []
        for gi in range(count):
            g = groups[base + gi].copy()
            leader = _node_of(g["leader_node"], names_of_row)
            pb, pc = int(g["pod_base"]), int(g["pod_count"])
            g["leader_node"] = g["pod_base"] = g["lws_index"] = 0
            pods = []
            for p in range(pb, pb + pc):
                place = int(pid["place"][p])
                node = _node_of(place >> R.PODID_NODE_SHIFT, names_of_row) if place & R.PODID_SCHEDULED else None
                pods.append((int(pst[p]), int(pid["rev_hash"][p]), int(pid["owner_uid_hash"][p]),
                             place & ((1 << R.PODID_NODE_SHIFT) - 1), node))
            o = g_out[base + gi].copy()
            d = int(o["domain_id"])
            o["domain_id"] = 0
            grp.append((g.tobytes(), leader, domain_values[d] if d != R.NONE else None, o.tobytes(), pods))
        rq = {}
        for r in reqs:
            gi = int(r["group"]) - base
            if 0 <= gi < count and (int(r["size"]) or int(r["leader_node"]) != R.NONE or int(r["priority"])):
                rq[gi] = (int(r["priority"]), int(r["group_key"]), int(r["size"]), _node_of(r["leader_node"], names_of_row))
        out[key] = (l.tobytes(), grp, rq)
    return out


def check_against_fresh(world, enc, mirror, where):
    items = list(world.items.values())
    ft = encoder.encode_lws(items, world.cluster(), "zone")
    f_names = {i: n.name for i, n in enumerate(world.nodes)}
    _, f_go, _ = oracle.sweep_lws(ft.lws, ft.groups, ft.pod_state, ft.pod_ident, ft.nodes, flags=R.SWEEP_GANG)
    want = objects_by_name(ft.lws, ft.groups, ft.pod_state, ft.pod_ident, encoder.encode_place_requests(ft.lws, ft.groups),
                           {i: (it.lws.namespace, it.lws.name) for i, it in enumerate(items)}, f_names, ft.domain_values, f_go)
    lws, groups, pst, pid, reqs, nodes = mirror
    e_names = {row: name for name, row in enc.node_index.items()}
    _, e_go, _ = oracle.sweep_lws(lws, groups, pst, pid, nodes, flags=R.SWEEP_GANG)
    got = objects_by_name(lws, groups, pst, pid, reqs, {sl.lws_row: key for key, sl in enc.slots.items()}, e_names,
                          enc.domain_values, e_go)
    assert set(got) == set(want), where
    for key in want:
        assert got[key] == want[key], (where, key)
    # node rows by name; vacant rows are zero (no request can use them)
    assert set(enc.node_index) == {n.name for n in world.nodes}, where
    assert nodes_by_name(nodes, enc.node_index, enc.domain_values) == nodes_by_name(
        ft.nodes, {n: i for i, n in f_names.items()}, ft.domain_values), where
    vacant = np.setdiff1d(np.arange(len(nodes)), list(enc.node_index.values()))
    assert not nodes[vacant].view(np.uint8).any(), where
    # scheduled identity rows per node row = the pods bound to that node's name
    assert occupancy_by_name(pid, len(nodes), enc.node_index) == occupancy_by_name(
        ft.pod_ident, len(ft.nodes), {n: i for i, n in f_names.items()}), where
    assert not R.occupancy_of(pid, len(nodes))[vacant].any(), where
    assert len(enc.domain_values) <= enc.n_domains


def apply(mirror, patches):
    for table, rows, vals in patches.segments:
        assert len(np.unique(rows)) == len(rows)
        mirror[BY_TABLE[table]][rows] = vals


def tables_of(enc):
    return [*enc.full_tables(), enc.node_rec]


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_node_stream_equals_fresh_encode(seed):
    items, cluster = make_world(seed, n_lws=10, n_nodes=24)
    world = NodeWorld(items, cluster, seed + 40)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", spare=3.0, node_spare=64)
    mirror = [a.copy() for a in tables_of(enc)]
    seen = {"ADDED": 0, "MODIFIED": 0, "DELETED": 0}
    for tick in range(60):
        freed = set()
        for _ in range(int(world.rng.integers(1, 8))):
            before = dict(enc.node_index)
            world.step(enc)
            gone = set(before) - set(enc.node_index)
            freed |= {before[n] for n in gone}
            for n in set(enc.node_index) - set(before):  # a row freed in this flush is not taken in it
                assert enc.node_row(n) not in freed, f"tick {tick}"
                seen["ADDED"] += 1
            seen["DELETED"] += len(gone)
        if tick % 5 == 2:  # a node deleted and one added under the same name, with its old pods, in one flush
            node = world.node_event(enc, "DELETED")
            if node is not None:
                row = enc.node_row(node.name)
                assert row is None
                world.node_event(enc, "ADDED", node=node)
                seen["MODIFIED"] += 1
        if tick % 9 == 4:  # pods bound to a node that does not exist yet, then the node
            name = world.future_name()
            world.bind_to_future_node(enc)
            if name not in world.node_names():
                world.node_event(enc, "ADDED", name=name)
        patches = enc.flush()
        assert not enc.needs_reload, f"tick {tick}"
        apply(mirror, patches)
        for a, b in zip(mirror, tables_of(enc)):
            assert a.tobytes() == b.tobytes(), f"tick {tick}"  # the patches carry every change
        check_against_fresh(world, enc, mirror, f"tick {tick}")
    assert seen["ADDED"] > 0 and seen["DELETED"] > 0


def test_no_node_events_keep_the_node_table_and_layout():
    """node_spare=0 (the default) and no node events: the node table is encode_nodes of the cluster, byte
    for byte, the domain capacity is its domain count, and no flush carries a node patch."""
    items, cluster = make_world(7, n_lws=10)
    world = NodeWorld(items, cluster, 8, p_node=0.0)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone")
    rec, values, index = encoder.encode_nodes(cluster.nodes, "zone")
    assert enc.node_rec.tobytes() == rec.tobytes() and enc.domain_values == values and enc.node_index == index
    assert enc.n_domains == len(values)
    for tick in range(20):
        for _ in range(4):
            world.step(enc)
        patches = enc.flush()
        assert all(s[0] != R.TABLE_NODES for s in patches.segments)
        assert enc.node_rec.tobytes() == rec.tobytes()


def test_reload_exactly_when_node_rows_run_out():
    """Two spare rows: two nodes fit; a third added in the flush that deletes another node does not (the
    freed row is free from the next flush on); added after that flush, it takes the freed row."""
    items, cluster = make_world(9, n_lws=4, n_nodes=12)
    for same_flush in (True, False):
        world = NodeWorld(items, cluster, 10, p_node=0.0)
        enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", node_spare=2)
        for j in range(2):
            world.node_event(enc, "ADDED", node=world_node(f"extra-{j}", "z0"))
            enc.flush()
            assert not enc.needs_reload
        victim = world.nodes[3].name
        row = enc.node_row(victim)
        world.node_event(enc, "DELETED", name=victim)
        if not same_flush:
            enc.flush()
            assert not enc.needs_reload
        world.node_event(enc, "ADDED", node=world_node("extra-2", "z1"))
        enc.flush()
        assert enc.needs_reload == same_flush
        if not same_flush:
            assert enc.node_row("extra-2") == row


def world_node(name, zone, capacity=8):
    from lws_b200 import api

    return api.Node(name=name, labels={"zone": zone}, capacity=capacity)


def test_reload_exactly_when_domain_ids_run_out():
    items, cluster = make_world(13, n_lws=4, n_nodes=12)
    world = NodeWorld(items, cluster, 14, p_node=0.0)
    enc = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", node_spare=3)
    for j in range(6):
        fits = len(enc.domain_values) < enc.n_domains
        node = world.nodes[j]
        node.labels = {"zone": f"fresh-{j}"}  # a relabel to a value never seen
        enc.node_event("MODIFIED", node)
        enc.flush()
        assert enc.needs_reload == (not fits), f"value {j}"
        if enc.needs_reload:
            break
    assert enc.needs_reload
    # a relabel back to a known value takes no new id
    enc2 = informer.IncrementalEncoder(list(world.items.values()), world.cluster(), "zone", node_spare=0)
    node = world.nodes[0]
    node.labels = {"zone": enc2.domain_values[0]}
    enc2.node_event("MODIFIED", node)
    enc2.flush()
    assert not enc2.needs_reload
