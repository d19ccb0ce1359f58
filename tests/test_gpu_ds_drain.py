"""DS drain on the device (lwse_resident_ds_drain*): both calls byte for byte against the definition
(tests/ds_drain_ref.py) on the DS drain worlds, with the after sweep's full role_out / revrole_out; per-key rows
against set-form calls; (DS, key) tables at 128 and 129 pairs and with probing that wraps; DS over shared row ranges;
a capacity below the touched count; the error returns; and isolation from LWS ticks in flight and from the next DS
tick, with the resident tables and the link table read back."""
import ctypes as C
import functools

import numpy as np
import pytest

from ds_drain_ref import (COST_FIELDS, TOTALS, cost_row_of, ds_drain_cost_ref, ds_drain_domains_ref, ds_drain_ref,
                          ds_drain_world, index_entries, overlap_worlds, single_row_world, table_slots, wrap_keys)
from lws_b200 import engine as E
from lws_b200 import records as R
from test_gpu_node_events import Arena

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOT_READY = -1, -6
WORLDS = {"w0": dict(n_ds=60, n_nodes=24, seed=3), "w1": dict(n_ds=80, n_nodes=32, seed=11),
          "w2": dict(n_ds=60, n_nodes=24, seed=29, nodes_per_domain=4), "w3": dict(n_ds=40, n_nodes=16, seed=41),
          "big": dict(n_ds=3000, n_nodes=512, seed=7)}


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def world(name):
    return ds_drain_world(**WORLDS[name])


def load(engine, w, link=True):
    engine.upload_nodes(w.nodes, w.n_domains)
    engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    engine.resident_tick(engine.make_tick((), w.flags))
    engine.ds_resident_load(w.ds, w.roles, w.revroles)
    return engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)] if link else [])


def check_set(got, ref, where, outputs=False):
    rows, totals, role_out, revrole_out = ref
    for k in TOTALS:
        assert got[k] == totals[k], (where, k, got[k], totals[k])
    o = np.argsort(got["rows"]["ds"], kind="stable")
    assert got["rows"][o].tobytes() == rows.tobytes(), where
    if outputs:
        assert got["role_out"].tobytes() == role_out.tobytes(), where
        assert got["revrole_out"].tobytes() == revrole_out.tobytes(), where


@pytest.mark.parametrize("name", ["w0", "w1", "w2", "w3"])
def test_small_worlds(engine, name):
    w = world(name)
    load(engine, w)
    res = engine.resident_outputs()
    assert res[0].tobytes() == w.base[0].tobytes() and res[1].tobytes() == w.base[1].tobytes()
    touched = 0
    for n in range(len(w.nodes)):
        got = engine.resident_ds_drain(nodes=[n], outputs=n % 3 == 0)
        check_set(got, ds_drain_ref(w, [n]), (name, n), outputs=n % 3 == 0)
        touched += got["n_touched"]
    assert touched > 0
    for d in range(w.n_domains):
        got = engine.resident_ds_drain(domains=[d], outputs=True)
        check_set(got, ds_drain_domains_ref(w, [d]), (name, "domain", d), outputs=True)
    for ids in ([], list(range(w.n_domains)), [0, 0, 1]):
        got = engine.resident_ds_drain(domains=ids, outputs=True)
        check_set(got, ds_drain_domains_ref(w, ids), (name, ids), outputs=True)
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_ds_drain_cost(scope)
        ref = ds_drain_cost_ref(w, by_domain)
        assert got.tobytes() == ref.tobytes(), (name, scope)


def test_big_world(engine):
    """3 000 DS on 512 nodes: both per-key forms against the restatement, and sampled keys against set-form calls
    (which are themselves checked against the reference)."""
    w = world("big")
    load(engine, w)
    cost = {}
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_ds_drain_cost(scope)
        assert got.tobytes() == ds_drain_cost_ref(w, by_domain).tobytes(), scope
        cost[scope] = got
    assert cost["nodes"]["ds_touched"].sum() > 100 and cost["domains"]["ds_service_lost"].sum() > 0
    rng = np.random.default_rng(4)
    for n in rng.choice(len(w.nodes), size=6, replace=False):
        got = engine.resident_ds_drain(nodes=[int(n)])
        check_set(got, ds_drain_ref(w, [int(n)]), ("big", int(n)))
        assert {f: int(cost["nodes"][f][n]) for f in COST_FIELDS} == cost_row_of(got)
    for d in rng.choice(w.n_domains, size=4, replace=False):
        got = engine.resident_ds_drain(domains=[int(d)], outputs=True)
        check_set(got, ds_drain_domains_ref(w, [int(d)]), ("big", "domain", int(d)), outputs=True)
        assert {f: int(cost["domains"][f][d]) for f in COST_FIELDS} == cost_row_of(got)


@pytest.mark.parametrize("case", ["pairs_128", "pairs_129", "wrap"])
def test_ds_key_table_edges(engine, case):
    """Worlds of single-row DS whose per-key call inserts exactly 128 or 129 (row, node) pairs (a 256- and a 512-slot
    (DS, key) table), or 128 pairs of which 12 home on the table's last slot, so that probing wraps to slot 0."""
    keys = {"pairs_128": {d: d % 63 for d in range(128)}, "pairs_129": {d: d % 63 for d in range(129)},
            "wrap": wrap_keys()}[case]
    w = single_row_world(keys)
    load(engine, w)
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_ds_drain_cost(scope)
        ref = ds_drain_cost_ref(w, by_domain)
        assert got.tobytes() == ref.tobytes(), (case, scope)
    assert int(got["rows_touched"].sum()) == len(keys) and table_slots(len(keys)) == (256 if len(keys) == 128 else 512)
    for n in (0, 1, 62, 63):
        check_set(engine.resident_ds_drain(nodes=[n], outputs=True), ds_drain_ref(w, [n]), (case, n), outputs=True)


def test_overlapping_ranges(engine):
    """200 DS over the revision-role range of one DS: more reverse-index entries than the table has rows.  Both calls
    answer as for a world where each of those DS has a copy of the rows (which the reference checks)."""
    shared, copied = overlap_worlds(world("w0"), 200)
    assert index_entries(shared) > len(shared.revroles)
    got = {}
    for name, w in (("shared", shared), ("copied", copied)):
        load(engine, w)
        got[name] = [engine.resident_ds_drain_cost(scope) for scope in ("nodes", "domains")]
        got[name] += [engine.resident_ds_drain(domains=[d]) for d in range(w.n_domains)]
        got[name] += [engine.resident_ds_drain(nodes=[n]) for n in range(len(w.nodes))]
    for scope, by_domain, x in zip(("nodes", "domains"), (False, True), got["copied"][:2]):
        assert x.tobytes() == ds_drain_cost_ref(copied, by_domain).tobytes(), scope
    for d in range(copied.n_domains):
        check_set(got["copied"][2 + d], ds_drain_domains_ref(copied, [d]), ("copied", d))
    assert got["shared"][0].tobytes() == got["copied"][0].tobytes()
    assert got["shared"][1].tobytes() == got["copied"][1].tobytes()
    assert sum(int(x["ds_touched"].sum()) for x in got["shared"][:2]) > 0
    for k, (x, y) in enumerate(zip(got["shared"][2:], got["copied"][2:])):
        assert all(x[t] == y[t] for t in TOTALS), k
        assert x["rows"][np.argsort(x["rows"]["ds"])].tobytes() == y["rows"][np.argsort(y["rows"]["ds"])].tobytes(), k


def read_back(e, table, n, dtype):
    """A resident input table as the engine holds it (lwse_debug_resident_read, a test aid outside lwse.h)."""
    fn = E.lib().lwse_debug_resident_read
    fn.argtypes, fn.restype = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32], C.c_int
    out = R.aligned_empty(max(n, 1), dtype)
    assert fn(e._h, table, R.ptr(out), n) == 0
    return out[:n]


def resident_tables(e, w):
    return [read_back(e, t, n, dt).tobytes() for t, n, dt in (
        (R.TABLE_LWS, len(w.lws), R.LWS_REC), (R.TABLE_GROUPS, len(w.groups), R.GROUP_REC),
        (R.TABLE_POD_STATE, len(w.pod_state), R.POD_STATE), (R.TABLE_POD_IDENT, len(w.pod_ident), R.POD_IDENT),
        (R.TABLE_DS, len(w.ds), R.DS_REC), (R.TABLE_DS_ROLES, len(w.roles), R.DS_ROLE_REC),
        (R.TABLE_DS_REVROLES, len(w.revroles), R.DS_REVROLE_REC), (R.TABLE_DS_LINKS, len(w.links), R.DS_LINK))]


def raw(e, ids=None, n_ids=0, scope=R.DRAIN_NODES, capacity=0, rows=None):
    q = R.DsDrainQuery()
    q.ids, q.n_ids, q.scope, q.capacity, q.rows = ids, n_ids, scope, capacity, rows
    return E.lib().lwse_resident_ds_drain(e._h, C.byref(q))


def test_errors_no_links_and_capacity():
    w = world("w1")
    e = E.Engine(0)
    try:
        one = np.array([1], np.uint32)
        out = R.aligned_empty(len(w.nodes), R.DS_DRAIN_COST)
        cost = E.lib().lwse_resident_ds_drain_cost
        assert raw(e, R.ptr(one), 1) == ERR_NOT_READY  # nothing loaded
        assert cost(e._h, R.DRAIN_NODES, R.ptr(out)) == ERR_NOT_READY
        e.upload_nodes(w.nodes, w.n_domains)
        e.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        e.resident_tick(e.make_tick((), w.flags))
        assert raw(e, R.ptr(one), 1) == ERR_NOT_READY  # no DS tables
        assert cost(e._h, R.DRAIN_NODES, R.ptr(out)) == ERR_NOT_READY
        e.ds_resident_load(w.ds, w.roles, w.revroles)
        # no link patch since the load: every row falls back
        got = e.resident_ds_drain(domains=list(range(w.n_domains)))
        assert got["n_touched"] == 0 and got["rows_linked"] == 0
        assert not e.resident_ds_drain_cost("domains").view(np.uint8).any()
        assert E.lib().lwse_resident_ds_drain(e._h, None) == ERR_INVALID_ARG
        assert cost(e._h, R.DRAIN_NODES, None) == ERR_INVALID_ARG
        assert cost(e._h, 2, R.ptr(out)) == ERR_INVALID_ARG
        assert raw(e, R.ptr(one), 1, scope=2) == ERR_INVALID_ARG
        assert raw(e, R.ptr(np.array([len(w.nodes)], np.uint32)), 1) == ERR_INVALID_ARG
        assert raw(e, R.ptr(np.array([w.n_domains], np.uint32)), 1, R.DRAIN_DOMAINS) == ERR_INVALID_ARG
        assert raw(e, None, 1) == ERR_INVALID_ARG
        assert raw(e, R.ptr(one), 1, capacity=4) == ERR_INVALID_ARG
        e.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
        # LWS rows patched without a sweep: not ready until the next sweep
        e.resident_patch(R.TABLE_LWS, [0], w.lws[:1])
        assert raw(e, R.ptr(one), 1) == ERR_NOT_READY
        e.resident_tick(e.make_tick((), w.flags))
        ids = list(range(w.n_domains))
        ref_rows, ref, _, _ = ds_drain_domains_ref(w, ids)
        assert ref["n_touched"] > 7
        small = e.resident_ds_drain(domains=ids, capacity=7)
        assert len(small["rows"]) == 7 and all(small[k] == ref[k] for k in TOTALS)
        for r in small["rows"]:
            assert r.tobytes() == ref_rows[np.searchsorted(ref_rows["ds"], r["ds"])].tobytes()
        assert len(e.resident_ds_drain(domains=ids, capacity=0)["rows"]) == 0
    finally:
        e.close()


def test_isolation(engine):
    """DS drain calls between the submit and wait of LWS ticks in flight, and before each DS tick: every LWS tick's
    change lists, the resident LWS rows, every DS tick's changed rows and full outputs, the DS tick info and the DS
    forecast equal a run without them, and every resident table and the link table read back equal too."""
    w = world("big")
    rng = np.random.default_rng(12)
    sets = []
    for _ in range(6):
        rows = np.sort(rng.choice(len(w.groups), size=200, replace=False)).astype(np.uint32)
        v = w.groups[rows].copy()
        v["flags"] ^= np.uint32(R.GRP_POD_READY)
        sets.append([(R.TABLE_GROUPS, rows, v)])

    def snap(r):
        return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()}

    def run(with_drain):
        first = snap(load(engine, w))
        first["info"] = engine.ds_resident_tick_info()
        arena = Arena(engine)
        lws_out, ds_out, answers = [], [first], []
        for k, segs in enumerate(sets):
            engine.resident_tick_submit(engine.make_tick(arena.put(segs, k & 1), w.flags))
            if with_drain:
                answers.append(engine.resident_ds_drain(domains=[k % w.n_domains], outputs=True))
                engine.resident_ds_drain_cost("nodes")
            lws_out.append(snap(engine.resident_tick_wait()))
            if with_drain:
                engine.resident_ds_drain_cost("domains")
            ds_out.append(snap(engine.ds_resident_tick([])))
            ds_out[-1]["info"] = engine.ds_resident_tick_info()
        fc = engine.ds_resident_forecast(steps=False)
        return lws_out, ds_out, [x.copy() for x in engine.resident_outputs()], fc, answers

    a = run(True)
    tables = resident_tables(engine, w)
    b = run(False)
    assert resident_tables(engine, w) == tables  # every resident table and the link table, read back
    # (no DS patch was sent: the DS tables and links are the loaded ones)
    assert tables[4:] == [w.ds.tobytes(), w.roles.tobytes(), w.revroles.tobytes(), w.links.tobytes()]
    before = resident_tables(engine, w)
    engine.resident_ds_drain(nodes=np.arange(len(w.nodes)), outputs=True)
    engine.resident_ds_drain_cost("nodes")
    engine.resident_ds_drain_cost("domains")
    assert resident_tables(engine, w) == before
    for k, (x, y) in enumerate(zip(a[0], b[0])):
        for key in ("lws_rows", "group_rows"):
            ox, oy = np.argsort(x[key], kind="stable"), np.argsort(y[key], kind="stable")
            assert np.array_equal(x[key][ox], y[key][oy]), (k, key)
            assert x[key.replace("rows", "out")][ox].tobytes() == y[key.replace("rows", "out")][oy].tobytes(), (k, key)
    for k, (x, y) in enumerate(zip(a[1], b[1])):
        assert np.array_equal(np.sort(x["rows"]), np.sort(y["rows"])), k
        for key in ("ds_out", "role_out", "revrole_out"):
            assert x[key].tobytes() == y[key].tobytes(), (k, key)
        # (lws_ticks counts the engine's LWS ticks since it was created: compare it from each run's first DS tick)
        ix = dict(x["info"], lws_ticks=x["info"]["lws_ticks"] - a[1][0]["info"]["lws_ticks"])
        iy = dict(y["info"], lws_ticks=y["info"]["lws_ticks"] - b[1][0]["info"]["lws_ticks"])
        assert ix == iy, k
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a[2], b[2]))
    assert a[3]["ds"].tobytes() == b[3]["ds"].tobytes() and a[3]["roles"].tobytes() == b[3]["roles"].tobytes()
    assert any(ans["n_touched"] for ans in a[4])

