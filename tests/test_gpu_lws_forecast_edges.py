"""The LWS rolling-update forecast at its slot, cycle, tile and grid edges on the device
(tests/lws_forecast_edges_world.py): every world through lwse_lws_forecast_host with steps, without, and
at the capacities around its row count, byte for byte against tests/lws_forecast_ref.py; the tile and
grid worlds also through lwse_resident_forecast after a sweep of their group rows; the cycle-cap rollout
against its closed form; and the slot sum at 2^31 - 8 (runs) and 2^31 (refused, writes nothing, the engine
right on the next call).  The slot-sum test needs about 2 GiB of device scratch: deselect it with
``-k "not slot_sum"``."""
import ctypes as C

import numpy as np
import pytest

import lws_forecast_edges_world as W
import oracle
from lws_b200 import engine as E
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast
from test_gpu_lws_forecast import _same

pytestmark = pytest.mark.gpu

ERR_UNSUPPORTED = -7  # lwse_status


@pytest.fixture(scope="module")
def engine():
    e = E.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def check_three_ways(engine, lws, go, want, where):
    """With steps, without, and at capacities one below and at the rows needed."""
    _same(engine.lws_forecast(lws, go), want, where)
    summ = engine.lws_forecast(lws, go, steps=False)
    assert summ["steps"] is None and summ["lws"].tobytes() == want["lws"].tobytes(), where
    assert summ["n_steps_needed"] == want["n_steps_needed"] and summ["n_steps_written"] == 0
    need = want["n_steps_needed"]
    for cap in sorted({max(need - 1, 0), need}):
        _same(engine.lws_forecast(lws, go, step_capacity=cap), lws_forecast(lws, go, step_capacity=cap),
              f"{where} capacity {cap}")


@pytest.mark.parametrize("label", W.SMALL + ("w1_sts", "slot_cap"))
def test_world(engine, label):
    w = W.world(label)
    want = lws_forecast(w.lws, w.group_out)
    check_three_ways(engine, w.lws, w.group_out, want, label)


def resident(engine, w):
    """Load the group rows the reference builds, run one sweep, forecast the resident tables."""
    groups = w.groups()
    pst, pid = np.zeros(1, R.POD_STATE), np.zeros(1, R.POD_IDENT)
    engine.resident_load(w.lws, groups, pst, pid)
    engine.resident_tick(engine.make_tick((), 0))
    go = engine.resident_outputs()[1]
    want_go = oracle.sweep_lws(w.lws, groups, pst, pid, threads=8)[1]
    assert go.tobytes() == want_go.tobytes(), w.label
    assert np.array_equal(go["flags"] & W.FLAG_MASK, w.group_out["flags"] & W.FLAG_MASK), w.label
    want = lws_forecast(w.lws, go)
    _same(engine.resident_forecast(), want, f"{w.label} resident")
    summ = engine.resident_forecast(steps=False)
    assert summ["lws"].tobytes() == want["lws"].tobytes()
    return want


@pytest.mark.parametrize("avg", W.TILE_AVGS)
def test_tile_threshold_resident(engine, avg):
    resident(engine, W.world(f"tile_{avg}"))


@pytest.mark.parametrize("width", W.WIDTHS)
def test_grid_stride(engine, sm_count, width):
    w = W.grid(sm_count, width)
    assert W.pick_tile(len(w.group_out), len(w.lws)) == width
    assert len(w.lws) > sm_count * W.GRID_CTAS_PER_SM * (W.BLOCK // width)
    want = lws_forecast(w.lws, w.group_out)
    check_three_ways(engine, w.lws, w.group_out, want, w.label)
    got = resident(engine, w)
    assert (got["lws"]["n_steps"][-4:] > 0).all()  # the last objects, past the grid's first stride, roll


def test_capacity_edges(engine):
    """step_capacity at exactly an object's step_base + n_steps and one below, objects of no rows
    between: TRUNCATED falls only on objects with rows."""
    w = W.world("capacity")
    full = lws_forecast(w.lws, w.group_out)
    n = full["lws"]["n_steps"].astype(np.int64)
    base = full["lws"]["step_base"].astype(np.int64)
    for i in np.flatnonzero(n > 0):
        for cap in (base[i] + n[i], base[i] + n[i] - 1):
            want = lws_forecast(w.lws, w.group_out, step_capacity=cap)
            got = engine.lws_forecast(w.lws, w.group_out, step_capacity=cap)
            _same(got, want, f"object {i} capacity {cap}")
            trunc = (got["lws"]["flags"] & R.LWSF_TRUNCATED) != 0
            assert not trunc[n == 0].any() and trunc[i] == (cap < base[i] + n[i])


def test_cycle_cap(engine):
    """A rollout still changing after MAX_CYCLES cycles: exactly the first MAX_CYCLES rows of its closed
    form, n_steps = MAX_CYCLES, UNFINISHED and not DONE; beside it the same rollout one cycle short of
    the cap ends DONE with its whole closed form."""
    w = W.world("cycle_cap")
    cap, below = w.of("cap")[0].row, w.of("below_cap")[0].row
    for steps in (True, False):
        got = engine.lws_forecast(w.lws, w.group_out, steps=steps)
        fc = got["lws"]
        assert fc[cap]["n_steps"] == fc[cap]["cycles"] == W.MAX_CYCLES
        assert fc[cap]["flags"] == R.LWSF_ROLLING | R.LWSF_UNFINISHED
        want = W.cap_rows(W.CAP_REPLICAS, 1, W.MAX_CYCLES)
        assert (fc[cap]["peak_sts_replicas"], fc[cap]["floor_ready"]) == (W.CAP_REPLICAS, W.CAP_REPLICAS - 1)
        assert (fc[cap]["final_partition"], fc[cap]["final_replicas"]) == (int(want["partition"][-1]), W.CAP_REPLICAS)
        full = W.cap_rows(W.MAX_CYCLES - 2, 1)
        assert fc[below]["n_steps"] == len(full) == W.MAX_CYCLES - 1
        assert fc[below]["flags"] == R.LWSF_ROLLING | R.LWSF_DONE
        assert got["n_steps_needed"] == W.MAX_CYCLES + len(full)
        if steps:
            st = got["steps"]
            assert st[fc[cap]["step_base"]: fc[cap]["step_base"] + W.MAX_CYCLES].tobytes() == want.tobytes()
            assert st[fc[below]["step_base"]: fc[below]["step_base"] + len(full)].tobytes() == full.tobytes()


def _tiled(one, kinds):
    """The reference's result for a table of objects of the kinds ``kinds`` (indices into ``one``), each
    object's rows after the previous one's."""
    fc = one["lws"][kinds].copy()
    n = fc["n_steps"].astype(np.int64)
    fc["step_base"] = np.cumsum(n) - n
    rows = np.concatenate([one["steps"][one["lws"][k]["step_base"]: one["lws"][k]["step_base"] + one["lws"][k]["n_steps"]]
                           for k in (0, 1)])
    per = {0: rows[: one["lws"][0]["n_steps"]], 1: rows[one["lws"][0]["n_steps"]:]}
    steps = np.concatenate([per[k] for k in kinds])
    return {"lws": fc, "steps": steps, "n_steps_written": int(n.sum()), "n_steps_needed": int(n.sum())}


def test_slot_sum_2gib(engine):
    one = lws_forecast(W.world("slot_sum_objects").lws, W.world("slot_sum_objects").group_out)
    runs = W.slot_sum(False)
    kinds = np.zeros(W.SUM_OBJECTS, np.int64)
    kinds[-1] = 1
    _same(engine.lws_forecast(runs.lws, runs.group_out), _tiled(one, kinds), "2^31 - 8 slots")
    # 2^31 slots: refused, nothing written
    ref = W.slot_sum(True)
    fc = R.aligned_empty(len(ref.lws), R.LWS_FORECAST)
    fc.view(np.uint8)[:] = 0xA5
    traj = R.aligned_empty(16, R.LWS_FORECAST_STEP)
    traj.view(np.uint8)[:] = 0x5A
    out = R.LwsForecastOut(R.ptr(fc), R.ptr(traj), 16, 0xDEAD, 0xBEEF)
    lws, go = ref.lws, ref.group_out
    rc = E.lib().lwse_lws_forecast_host(engine._h, R.ptr(lws), len(lws), R.ptr(go), len(go), C.byref(out))
    assert rc == ERR_UNSUPPORTED
    assert (fc.view(np.uint8) == 0xA5).all() and (traj.view(np.uint8) == 0x5A).all()
    assert (out.n_steps_written, out.n_steps_needed) == (0xDEAD, 0xBEEF)
    # the same engine, right away: a small world and the 2^31 - 8 table again
    w = W.world("words_8")
    _same(engine.lws_forecast(w.lws, w.group_out), lws_forecast(w.lws, w.group_out), "after the refusal")
    _same(engine.lws_forecast(runs.lws, runs.group_out), _tiled(one, kinds), "2^31 - 8 slots again")
