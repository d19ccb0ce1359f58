"""The kernel launches of one call of each entry point test_gpu_drain_launches.py does not count: the resident tick
(sweep only, placement only, both, and two in flight), the resident and host sweeps, the host placement and
reconcile, the set-form drain queries, the DS tick, forecasts and what-if, the LWS forecasts and what-if, the rollout
placement and its waves, and the SHA-1 keys.  Counted with ``Engine.launch_count`` on the rollout placement's fuzz
world and on a seeded DS drain world; a change that drops or adds a launch, or counts a launcher's result wrongly,
changes a count."""
import numpy as np
import pytest

from ds_drain_waves_ref import slack_world
from lws_b200 import records as R
from lws_b200.engine import Engine
from rollout_place_ref import fuzz_world, proposals
from test_gpu_ds_rollout_whatif import random_proposals
from test_rollout_place_waves import fuzz_query

pytestmark = pytest.mark.gpu

# Measured with measure() on an H100 at the commit before launchers returned their CUDA error negated.
EXPECTED = {
    "tick/sweep": 3, "tick/place": 3, "tick/both": 5, "tick/pipelined": 10, "resident_sweep": 3, "drain_whatif": 3,
    "drain_cost": 1, "drain_budget/nodes": 4, "drain_budget/domains": 5, "resident_forecast": 17, "rollout_whatif": 33,
    "rollout_place": 18, "rollout_place/recs": 26, "rollout_place_waves": 48, "rollout_place_waves/recs": 46,
    "sweep_lws_host": 3, "reconcile_host": 4, "place_host": 2, "lws_forecast": 17, "group_keys_host": 1,
    "subgroup_keys_host": 1, "ds_resident_tick": 1, "ds_drain/nodes": 8, "ds_drain/domains": 9, "ds_forecast_host": 9,
    "ds_resident_forecast": 9, "ds_rollout_whatif": 21,
}


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
        w = fuzz_world(1)
        engine.upload_nodes(w.nodes, w.n_domains)
        engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
        engine.resident_place_load(w.reqs, w.n_ns)
        sweep = engine.make_tick((), w.flags)
        place = engine.make_tick((), w.flags | R.TICK_PLACE | R.TICK_NO_SWEEP)
        both = engine.make_tick((), w.flags | R.TICK_PLACE)
        count("tick/sweep", lambda: engine.resident_tick(sweep))
        count("tick/place", lambda: engine.resident_tick(place))
        count("tick/both", lambda: engine.resident_tick(both))

        def pipelined():
            engine.resident_tick_submit(both)
            engine.resident_tick_submit(both)
            engine.resident_tick_wait()
            engine.resident_tick_wait()

        count("tick/pipelined", pipelined)
        count("resident_sweep", lambda: engine.resident_sweep(w.flags))
        engine.resident_tick(both)
        drained = np.arange(4)
        count("drain_whatif", lambda: engine.resident_drain_whatif(drained))
        count("drain_cost", lambda: engine.resident_drain_cost())
        count("drain_budget/nodes", lambda: engine.resident_drain_budget(nodes=drained))
        count("drain_budget/domains", lambda: engine.resident_drain_budget(domains=np.arange(2)))
        rows, ns = fuzz_query(w, 1)
        recs = proposals(w.lws, rows, 1)[1]
        count("resident_forecast", lambda: engine.resident_forecast())
        count("rollout_whatif", lambda: engine.resident_rollout_whatif(rows, recs))
        count("rollout_place", lambda: engine.resident_rollout_place(rows, ns))
        count("rollout_place/recs", lambda: engine.resident_rollout_place(rows, ns, recs))
        count("rollout_place_waves", lambda: engine.resident_rollout_place_waves(rows, ns))
        count("rollout_place_waves/recs", lambda: engine.resident_rollout_place_waves(rows, ns, recs))
        tables = (w.lws, w.groups, w.pod_state, w.pod_ident)
        count("sweep_lws_host", lambda: engine.sweep_lws_host(*tables, flags=w.flags, want_occupancy=True))
        _, group_out, occ = engine.sweep_lws_host(*tables, flags=w.flags, want_occupancy=True)
        count("reconcile_host", lambda: engine.reconcile_host(*tables, w.reqs, occ, w.n_ns, flags=w.flags))
        count("place_host", lambda: engine.place_host(w.reqs, occ, w.n_ns))
        count("lws_forecast", lambda: engine.lws_forecast(w.lws, group_out))
        names = [f"leader-{i}" for i in range(40)]
        count("group_keys_host", lambda: engine.group_keys_host(names))
        ones = np.ones(len(names), np.int32)
        count("subgroup_keys_host", lambda: engine.subgroup_keys_host(names, 4 * ones, 2 * ones, ones))

        d = slack_world(n_ds=30, n_nodes=96, seed=3)
        engine.upload_nodes(d.nodes, d.n_domains)
        engine.resident_load(d.lws, d.groups, d.pod_state, d.pod_ident)
        engine.resident_tick(engine.make_tick((), d.flags))
        engine.ds_resident_load(d.ds, d.roles, d.revroles)
        engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, d.links, True)])
        count("ds_resident_tick", lambda: engine.ds_resident_tick())
        count("ds_drain/nodes", lambda: engine.resident_ds_drain(nodes=np.arange(8)))
        count("ds_drain/domains", lambda: engine.resident_ds_drain(domains=np.arange(2)))
        count("ds_forecast_host", lambda: engine.ds_forecast_host(d.ds, d.roles, d.revroles))
        count("ds_resident_forecast", lambda: engine.ds_resident_forecast())
        props, qroles = random_proposals(d.ds, d.roles, 64, 5)
        count("ds_rollout_whatif", lambda: engine.resident_ds_rollout_whatif(props, qroles))
    finally:
        engine.close()
    return counts


def test_launches_per_call():
    assert measure() == EXPECTED

