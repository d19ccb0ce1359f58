"""The drain kernels at their walk, table and grid edges on the device (tests/drain_edges_world.py): every edge
world through lwse_resident_drain_cost, _drain_budget_cost (both scopes), _drain_whatif and _drain_budget,
byte for byte against the definitions (tests/drain_ref.py, tests/drain_budget_ref.py); change lists at
capacities around their row count; every LWS sweep form under the what-if; and scratch that shrinks and
grows again on one engine."""
import numpy as np
import pytest

import drain_edges_world as W
import lws_forms_world as F
import oracle
from drain_budget_ref import domain_nodes, drain_budget_cost_ref, drain_budget_ref
from drain_ref import COST_OF, TOTALS, drain_cost_ref, drain_whatif_ref
from lws_b200 import engine as E
from lws_b200 import records as R
from test_gpu_drain_budget import check_set
from test_gpu_drain_whatif import check

pytestmark = pytest.mark.gpu

BUDGET_TOTALS = R.DRAIN_BUDGET_TOTALS


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def load(engine, w):
    engine.upload_nodes(w.nodes, w.n_domains)
    engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    engine.resident_tick(engine.make_tick((), w.flags))
    base = oracle.sweep_lws(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.flags)[:2]
    res = engine.resident_outputs()
    assert res[0].tobytes() == base[0].tobytes() and res[1].tobytes() == base[1].tobytes(), w.label
    return base


def check_costs(engine, w, base):
    """drain_cost and both scopes of drain_budget_cost against the references; the NODES head is the cost."""
    cost = engine.resident_drain_cost()
    assert cost.tobytes() == drain_cost_ref(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base[1]).tobytes()
    out = {}
    for scope, by_domain in (("nodes", False), ("domains", True)):
        got = engine.resident_drain_budget_cost(scope)
        ref = drain_budget_cost_ref(w.lws, base[0], w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, base[1],
                                    by_domain)
        if got.tobytes() != ref.tobytes():
            bad = [k for k in range(len(ref)) if got[k].tobytes() != ref[k].tobytes()]
            raise AssertionError(f"{w.label} {scope}: {len(bad)} rows differ; first {bad[0]}: {got[bad[0]]} != {ref[bad[0]]}")
        out[scope] = got
    assert out["nodes"].view(np.uint8).reshape(len(cost), 48)[:, :32].tobytes() == cost.tobytes()
    return cost, out


def node_sets(w, n=24, seed=0):
    """Single nodes (every node of a small table, else the first, the last and a sample), all, none, a
    duplicate set."""
    nn = len(w.nodes)
    rng = np.random.default_rng(seed)
    singles = list(range(nn)) if nn <= 128 else sorted({0, nn - 1, *rng.choice(nn, size=n, replace=False).tolist()})
    return [[s] for s in singles] + [list(range(nn)), [], [singles[0], singles[0], singles[-1]]]


def domain_sets(w, n=16, seed=1):
    nd = w.n_domains
    if nd == 0:
        return [[]]
    rng = np.random.default_rng(seed)
    singles = list(range(nd)) if nd <= 256 else sorted({0, nd - 1, *rng.choice(nd, size=n, replace=False).tolist()})
    return [[s] for s in singles] + [list(range(nd)), [], [singles[0], singles[0], singles[-1]]]


def check_sets(engine, w, base, cost, nodes=None, domains=None):
    for d in nodes if nodes is not None else node_sets(w):
        wf = drain_whatif_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base)
        check(engine.resident_drain_whatif(d), wf, (w.label, "whatif", d[:3]))
        check_set(engine.resident_drain_budget(nodes=d),
                  drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base),
                  (w.label, "budget", d[:3]))
        if len(d) == 1:
            for k in TOTALS:
                assert int(cost[COST_OF[k]][d[0]]) == wf[k], (w.label, d, k)
    for ids in domains if domains is not None else domain_sets(w):
        ref = drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes,
                               domain_nodes(w.nodes, w.n_domains, ids), w.flags, base=base)
        check_set(engine.resident_drain_budget(domains=ids), ref, (w.label, "domains", ids[:3]))


@pytest.mark.parametrize("label", ["walk"] + list(W.SMALL))
def test_edge_world(engine, label):
    w = W.world(label)
    base = load(engine, w)
    cost, _ = check_costs(engine, w, base)
    check_sets(engine, w, base, cost)


def test_int32_floor(engine):
    """replicas 2^30 with maxUnavailable 300 %: mu = 3 221 225 472 is not truncated, the floor is 0 (with mu
    truncated to int32 it was INT32_MAX, and the row ALREADY_BELOW)."""
    w = W.world("budget_edges")
    base = load(engine, w)
    o = w.notes["int32"][W.INT32_FLOORS.index((1 << 30, 300, True))]
    g0 = int(w.lws[o]["group_base"])
    leader = int(w.groups[g0]["leader_node"])
    got = engine.resident_drain_budget(nodes=[leader])
    ref_rows, ref = drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, [leader], w.flags, base=base)
    row = got["rows"][got["rows"]["lws"] == o]
    assert len(row) == 1 and int(row["floor"][0]) == 0 and not (row["flags"][0] & R.DRAINB_ALREADY_BELOW)
    assert got["n_already_below"] == ref["n_already_below"]
    for o, (reps, mu, pct) in zip(w.notes["int32"], W.INT32_FLOORS):
        m = (mu * reps) // 100 if pct else mu
        floor = min(max(0, reps - m), W.I32_MAX)
        g0 = int(w.lws[o]["group_base"])
        r = engine.resident_drain_budget(nodes=[int(w.groups[g0]["leader_node"])])["rows"]
        assert int(r["floor"][r["lws"] == o][0]) == floor, (reps, mu, pct)


@pytest.mark.parametrize("label", ["walk", "budget_edges"])
def test_capacities(engine, label):
    """Change lists of n - 1, n, n + 1 and 1 rows for the what-if and the set-form budget: the listed rows are
    distinct, the reference's, with its before / after rows; the totals are exact."""
    w = W.world(label)
    base = load(engine, w)
    d = list(range(0, len(w.nodes), 3))
    wf = drain_whatif_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base)
    n = wf["n_changed"]
    assert n > 2
    for cap in (n - 1, n, n + 1, 1):
        got = engine.resident_drain_whatif(d, capacity=cap)
        assert len(got["rows"]) == min(cap, n) and len(set(got["rows"].tolist())) == len(got["rows"])
        for k in ("n_changed",) + TOTALS:
            assert got[k] == wf[k], (cap, k)
        i = np.searchsorted(wf["rows"], got["rows"])
        assert np.array_equal(wf["rows"][i], got["rows"]), cap
        assert got["before"].tobytes() == wf["before"][i].tobytes() and got["after"].tobytes() == wf["after"][i].tobytes()
    rows, tot = drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base)
    n = tot["n_touched"]
    assert n > 2
    for cap in (n - 1, n, n + 1, 1):
        got = engine.resident_drain_budget(nodes=d, capacity=cap)
        assert len(got["rows"]) == min(cap, n) and len(set(got["rows"]["lws"].tolist())) == len(got["rows"])
        assert all(got[k] == tot[k] for k in BUDGET_TOTALS), cap
        for r in got["rows"]:
            assert r.tobytes() == rows[np.searchsorted(rows["lws"], r["lws"])].tobytes(), cap


@pytest.mark.parametrize("what", ["nodes", "groups"])
def test_grid_edges(engine, sm_count, what):
    """Tables past the grid caps of this device: the domain mask over more nodes than its grid has threads;
    more groups than the mark kernel's grid has threads (its group loop, the diff's and the budget's
    strides)."""
    w = W.grid_world(sm_count, what)
    base = load(engine, w)
    cost, out = check_costs(engine, w, base)
    rng = np.random.default_rng(6)
    nn, nd = len(w.nodes), w.n_domains
    nodes = [[nn - 1], list(range(0, nn, 97)), rng.choice(nn, size=nn // 50, replace=False).tolist()]
    domains = [[nd - 1], list(range(0, nd, 7))]
    check_sets(engine, w, base, cost, nodes=nodes, domains=domains)
    assert out["domains"]["lws_touched"].sum() > 0


@pytest.mark.parametrize("label", list(F.BUILDERS))
def test_lws_forms_under_the_whatif(engine, label):
    """Every form of the sweep the what-if runs (with the LWS pass skipped) against the spec oracle, and the
    drain cost of the same table."""
    t = F.world(label).tables
    w = W.EdgeWorld(label, t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags)
    base = load(engine, w)
    cost = engine.resident_drain_cost()
    assert cost.tobytes() == drain_cost_ref(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base[1]).tobytes()
    dom = int(w.nodes["domain_id"][3])
    for d in ([3], np.flatnonzero(w.nodes["domain_id"] == dom).tolist(), list(range(len(w.nodes)))):
        check(engine.resident_drain_whatif(d),
              drain_whatif_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base), (label, d[:3]))


def test_scratch_shrinks_and_grows(engine):
    """big → small → big on one engine, every call each time: the scratch only grows, and a smaller table
    after a bigger one reads none of the bigger one's leftovers."""
    for label in ("walk", "wrap", "walk", "pairs_129", "budget_edges"):
        w = W.world(label)
        base = load(engine, w)
        cost, _ = check_costs(engine, w, base)
        nn = len(w.nodes)
        check_sets(engine, w, base, cost, nodes=[[0], [nn - 1], list(range(nn))],
                   domains=[[0], list(range(w.n_domains))] if w.n_domains else [[]])
