"""An engine gives back every CUDA object it holds when it is closed: device and pinned allocations, streams,
events, graph executables and peer mappings, counted process-wide by lwse_debug_cuda_objects (a test aid outside
lwse.h).  One engine answers every drain query (test_gpu_drain_launches.measure), a second every other entry point
that reserves scratch or creates a handle lazily; after both are closed the count is back where it started."""
import ctypes as C
import gc

import numpy as np
import pytest

from ds_drain_ref import ds_drain_world
from lws_b200 import engine as E
from lws_b200 import records as R
from rollout_place_ref import fuzz_world, proposals
from test_gpu_drain_launches import measure
from test_gpu_ds_drain import load as ds_load
from test_gpu_ds_rollout_whatif import random_proposals

pytestmark = pytest.mark.gpu


def live_objects() -> int:
    fn = E.lib().lwse_debug_cuda_objects
    fn.argtypes, fn.restype = [], C.c_int64
    return fn()


def other_entry_points(engine):
    """The host sweep and placement, the forecasts, the rollout what-ifs and placement, the drain what-if, budget
    and DS drain, the group keys and a world-1 exchange."""
    w = fuzz_world(1)
    engine.upload_nodes(w.nodes, w.n_domains)
    _, go, _ = engine.sweep_lws_host(w.lws, w.groups, w.pod_state, w.pod_ident, flags=w.flags, want_occupancy=True)
    engine.place_host(w.reqs, w.occ, w.n_ns)
    engine.lws_forecast(w.lws, go)
    engine.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    engine.resident_place_load(w.reqs, w.n_ns)
    engine.resident_tick(engine.make_tick((), w.flags | R.TICK_PLACE))
    engine.resident_forecast()
    rows = np.arange(min(len(w.lws), 64), dtype=np.uint32)
    ns = (rows.astype(np.int64) % w.n_ns).astype(np.uint32)
    engine.resident_rollout_whatif(*proposals(w.lws, rows, 1))
    engine.resident_rollout_place(rows, ns, extra=True)
    engine.resident_rollout_place(rows, ns, proposals(w.lws, rows, 2)[1], extra=True)
    engine.resident_drain_whatif([0, 1])
    engine.resident_drain_budget(nodes=[0, 1])
    engine.resident_drain_budget(domains=[0])
    engine.group_keys_host(["a", "bc", "lws-0"])

    d = ds_drain_world(n_ds=300, n_nodes=48, seed=31)
    ds_load(engine, d)
    engine.ds_forecast_host(d.ds, d.roles, d.revroles)
    engine.ds_resident_forecast()
    engine.resident_ds_rollout_whatif(*random_proposals(d.ds, d.roles, 40, 5))
    engine.resident_ds_drain(nodes=[0], outputs=True)
    engine.resident_ds_drain(domains=[0])
    engine.exchange_connect(engine.exchange_create(16, 1, 0))


def test_closed_engines_hold_nothing():
    gc.collect()
    base = live_objects()
    measure()
    engine = E.Engine(0)
    try:
        assert live_objects() > base  # the engine's streams, events and pinned words
        other_entry_points(engine)
        assert live_objects() > base
    finally:
        engine.close()
    gc.collect()
    assert live_objects() == base
