"""The kernel launches of one call of each query built from the drain chains' shared host steps: the place what-if,
the per-key forms of the drain budget, the drain placement and the DS drain, and the three waves planners, for both
scopes and, for the planners, with every key and with none.  Counted with ``Engine.launch_count`` on the drain
placement's seeded world and on a seeded DS drain world; a change that drops or adds a launch changes a count."""
import numpy as np
import pytest

from ds_drain_waves_ref import slack_world
from lws_b200 import records as R
from lws_b200.engine import Engine
from test_drain_place_cost import WORLDS

pytestmark = pytest.mark.gpu

# Measured with measure() on an H100 at the commit before these queries' host steps were shared.
EXPECTED = {
    "place_whatif": 6, "place_whatif/cordon": 10, "drain_budget_cost/nodes": 4, "drain_place_cost/nodes": 18,
    "drain_waves/nodes/all": 10, "drain_place_waves/nodes/all": 145, "drain_waves/nodes/none": 10,
    "drain_place_waves/nodes/none": 33, "drain_budget_cost/domains": 4, "drain_place_cost/domains": 18,
    "drain_waves/domains/all": 10, "drain_place_waves/domains/all": 61, "drain_waves/domains/none": 10,
    "drain_place_waves/domains/none": 33, "ds_drain_cost/nodes": 10, "ds_drain_waves/nodes/all": 21,
    "ds_drain_waves/nodes/none": 21, "ds_drain_cost/domains": 10, "ds_drain_waves/domains/all": 21,
    "ds_drain_waves/domains/none": 21,
}


def cordon(nodes, domain):
    rows = np.flatnonzero(nodes["domain_id"] == domain).astype(np.uint32)
    vals = R.aligned_empty(len(rows), R.NODE_REC)
    vals[:] = nodes[rows]
    vals["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
    return (R.TABLE_NODES, rows, vals)


def measure():
    """{call: kernel launches of its second call} (the first sizes the scratch)."""
    engine = Engine(0)
    counts = {}

    def count(name, call):
        call()
        before = engine.launch_count
        call()
        counts[name] = engine.launch_count - before

    try:
        lws, groups, pst, pid, nodes, nd, _, reqs, n_ns = WORLDS["seed3"]()
        engine.upload_nodes(nodes, nd)
        engine.resident_load(lws, groups, pst, pid)
        engine.resident_place_load(reqs, n_ns)
        engine.resident_tick(engine.make_tick((), R.TICK_PLACE))
        count("place_whatif", lambda: engine.resident_place_whatif())
        count("place_whatif/cordon", lambda: engine.resident_place_whatif([cordon(nodes, 0)]))
        for scope, n in (("nodes", len(nodes)), ("domains", nd)):
            count(f"drain_budget_cost/{scope}", lambda: engine.resident_drain_budget_cost(scope))
            count(f"drain_place_cost/{scope}", lambda: engine.resident_drain_place_cost(scope))
            for keys, ids in (("all", np.arange(n)), ("none", np.arange(0))):
                count(f"drain_waves/{scope}/{keys}", lambda: engine.resident_drain_waves(**{scope: ids}))
                count(f"drain_place_waves/{scope}/{keys}", lambda: engine.resident_drain_place_waves(**{scope: ids}))
        w = slack_world(n_ds=30, n_nodes=96, seed=3)
        engine.upload_nodes(w.nodes, w.n_domains)
        engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        engine.resident_tick(engine.make_tick((), w.flags))
        engine.ds_resident_load(w.ds, w.roles, w.revroles)
        engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
        for scope, n in (("nodes", len(w.nodes)), ("domains", w.n_domains)):
            count(f"ds_drain_cost/{scope}", lambda: engine.resident_ds_drain_cost(scope))
            for keys, ids in (("all", np.arange(n)), ("none", np.arange(0))):
                count(f"ds_drain_waves/{scope}/{keys}", lambda: engine.resident_ds_drain_waves(**{scope: ids}))
    finally:
        engine.close()
    return counts


def test_launches_per_call():
    assert measure() == EXPECTED
