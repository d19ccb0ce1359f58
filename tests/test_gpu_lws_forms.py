"""Every form of the LWS sweep (tests/lws_forms_world.py) through every entry point on the GPU: the
stateless host and device entries, the resident patch + sweep, the eager tick, pipelined ticks and
graph-replayed ticks.  Every output byte and every change list against ``oracle.sweep_lws`` — the
per-object restatement, not the kernels' SWAR form."""
import os

import numpy as np
import pytest

import lws_forms_world as W
from lws_b200 import records as R

pytestmark = pytest.mark.gpu

LABELS = list(W.BUILDERS)


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def graph_engine():
    """An engine that replays every eligible tick as a CUDA graph (LWSE_TICK_GRAPH=2, read at creation)."""
    from lws_b200.engine import Engine

    old = os.environ.get("LWSE_TICK_GRAPH")
    os.environ["LWSE_TICK_GRAPH"] = "2"
    try:
        e = Engine(0)
    finally:
        if old is None:
            del os.environ["LWSE_TICK_GRAPH"]
        else:
            os.environ["LWSE_TICK_GRAPH"] = old
    yield e
    e.close()


def _oracle(t, m=None, occupancy=False):
    import oracle

    lws, groups, pst, pid = m if m is not None else (t.lws, t.groups, t.pod_state, t.pod_ident)
    return oracle.sweep_lws(lws, groups, pst, pid, t.nodes, flags=t.flags, want_occupancy=occupancy)


def _same(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    if got.tobytes() != want.tobytes():
        bad = [i for i in range(len(got)) if got[i].tobytes() != want[i].tobytes()]
        raise AssertionError(f"{what}: {len(bad)} rows differ; first {bad[0]}: got {got[bad[0]]!r} want {want[bad[0]]!r}")


def _diff_rows(a, b):
    n = a.dtype.itemsize
    return np.flatnonzero(np.any(a.view(np.uint8).reshape(len(a), n) != b.view(np.uint8).reshape(len(b), n), axis=1))


def _check_lists(what, rows, outs, count, before, after):
    want = _diff_rows(before, after)
    assert count == len(want), what
    o = np.argsort(rows)
    assert np.array_equal(rows[o], want), what
    assert outs[o].tobytes() == after[want].tobytes(), what


def _mirrors(t):
    return (t.lws.copy(), t.groups.copy(), t.pod_state.copy(), t.pod_ident.copy())


# --------------------------------------------------------------------------- #
# 1. lwse_sweep_lws_host: pageable (launch counts name the form), with occupancy, pinned
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("label", LABELS)
def test_host_entry(engine, label):
    import torch

    w = W.world(label)
    t = w.tables
    form = W.form_of(t)
    engine.upload_nodes(t.nodes, t.n_domains)
    want = _oracle(t, occupancy=True)
    for occupancy in (False, True):
        before = engine.launch_count
        got = engine.sweep_lws_host(t.lws, t.groups, t.pod_state, t.pod_ident, flags=t.flags, want_occupancy=occupancy)
        # fused = 2, three-kernel = 3, no pods = 2, no groups = 1; the occupancy count when there are pods
        assert engine.launch_count - before == form.kernels + int(occupancy and len(t.pod_state) > 0), (label, form)
        _same(got[0], want[0], f"{label} lws_out")
        _same(got[1], want[1], f"{label} group_out")
        if occupancy:
            assert np.array_equal(got[2], want[2]), f"{label} occupancy"
    keep = []

    def pinned(a):
        ten = torch.empty(max(a.nbytes, 16), dtype=torch.uint8).pin_memory()
        v = ten.numpy()[: a.nbytes].view(a.dtype)
        v[...] = a
        keep.append(ten)
        return v

    lws, grp, pst, pid = pinned(t.lws), pinned(t.groups), pinned(t.pod_state), pinned(t.pod_ident)
    for _ in range(2):  # the first call reads event pods' identity rows in place; the second as the first measured
        before = engine.launch_count
        got = engine.sweep_lws_host(lws, grp, pst, pid, flags=t.flags)
        assert engine.launch_count - before in (form.kernels, form.kernels + 1), label  # (+ the identity prefetch)
        _same(got[0], want[0], f"{label} pinned lws_out")
        _same(got[1], want[1], f"{label} pinned group_out")


# --------------------------------------------------------------------------- #
# 2. lwse_sweep_lws_device on a non-default torch stream
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("label", ["fused_hi", "three_w8_2049", "lws_w32_1025"])
def test_device_entry_on_a_torch_stream(engine, label):
    import torch

    w = W.world(label)
    t = w.tables
    engine.upload_nodes(t.nodes, t.n_domains)
    dev = torch.device("cuda:0")

    def up(a):
        return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(dev)

    d_lws, d_grp, d_pst, d_pid = up(t.lws), up(t.groups), up(t.pod_state), up(t.pod_ident)
    d_lo = torch.full((len(t.lws) * R.LWS_OUT.itemsize,), 0xAB, dtype=torch.uint8, device=dev)
    d_go = torch.full((len(t.groups) * R.GROUP_OUT.itemsize,), 0xAB, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    before = engine.launch_count
    engine.sweep_lws_device(d_lws, len(t.lws), d_grp, len(t.groups), d_pst, d_pid, len(t.pod_state), d_lo, d_go,
                            flags=t.flags, stream=side.cuda_stream)
    torch.cuda.synchronize()
    assert engine.launch_count - before == W.form_of(t).kernels
    want = _oracle(t)
    _same(d_lo.cpu().numpy().view(R.LWS_OUT), want[0], f"{label} lws_out")
    _same(d_go.cpu().numpy().view(R.GROUP_OUT), want[1], f"{label} group_out")


# --------------------------------------------------------------------------- #
# 3. lwse_resident_load -> lwse_resident_patch -> lwse_resident_sweep
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("label", LABELS)
def test_resident_patch_and_sweep(engine, label):
    w = W.world(label)
    t = w.tables
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    m = _mirrors(t)
    prev = _oracle(t, m)
    lr, lo, gr, go, nl, ng = engine.resident_sweep(t.flags)
    assert (nl, ng) == (len(t.lws), len(t.groups))
    full = engine.resident_outputs()
    _same(full[0], prev[0], f"{label} lws_out")
    _same(full[1], prev[1], f"{label} group_out")
    for k, tick in enumerate(w.plan):
        for tb, (rows, vals) in tick.items():
            engine.resident_patch(tb, rows, vals)
        W.apply_tick(tick, *m)
        now = _oracle(t, m)
        lr, lo, gr, go, nl, ng = engine.resident_sweep(t.flags)
        _check_lists(f"{label} tick {k} lws", lr, lo, nl, prev[0], now[0])
        _check_lists(f"{label} tick {k} groups", gr, go, ng, prev[1], now[1])
        full = engine.resident_outputs()
        _same(full[0], now[0], f"{label} tick {k} lws_out")
        _same(full[1], now[1], f"{label} tick {k} group_out")
        prev = now


# --------------------------------------------------------------------------- #
# 4-6. lwse_resident_tick: eager (segments in the arena and staged), two in flight, graph replay
# --------------------------------------------------------------------------- #
def _arena_ticks(engine, plan, flags):
    """Every tick's rows and values in its own region of the engine's patch arena."""
    need = 4096 + sum(((a.nbytes + 255) // 256 + 1) * 256 for tick in plan for rv in tick.values() for a in rv)
    arena = engine.resident_arena(need)
    cursor, ticks = 0, []
    for tick in plan:
        segs = []
        for tb, (rows, vals) in tick.items():
            views = []
            for a in (rows, vals):
                cursor = (cursor + 255) // 256 * 256
                v = arena[cursor: cursor + a.nbytes].view(a.dtype)
                v[...] = a
                cursor += a.nbytes
                views.append(v)
            segs.append((tb, views[0], views[1]))
        ticks.append(engine.make_tick(segs, flags))
    return ticks


def _load(engine, t):
    engine.upload_nodes(t.nodes, t.n_domains)
    engine.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    engine.resident_tick(engine.make_tick((), t.flags))  # every row once; the ticks below list changes


def _check_tick(label, k, res, before, after):
    res = {key: (v.copy() if isinstance(v, np.ndarray) else v) for key, v in res.items()}
    _check_lists(f"{label} tick {k} lws", res["lws_rows"], res["lws_out"], res["n_lws"], before[0], after[0])
    _check_lists(f"{label} tick {k} groups", res["group_rows"], res["group_out"], res["n_groups"], before[1], after[1])


@pytest.mark.parametrize("in_arena", [True, False])
@pytest.mark.parametrize("label", LABELS)
def test_eager_ticks(engine, label, in_arena):
    w = W.world(label)
    t = w.tables
    _load(engine, t)
    m = _mirrors(t)
    prev = _oracle(t, m)
    if in_arena:
        ticks = _arena_ticks(engine, w.plan, t.flags)
    else:  # caller-owned pageable buffers: the call stages them
        ticks = [engine.make_tick([(tb, rows, vals) for tb, (rows, vals) in tick.items()], t.flags) for tick in w.plan]
    for k, tick in enumerate(w.plan):
        W.apply_tick(tick, *m)
        now = _oracle(t, m)
        res = engine.resident_tick(ticks[k])
        _check_tick(label, k, res, prev, now)
        full = engine.resident_outputs()
        _same(full[0], now[0], f"{label} tick {k} lws_out")
        _same(full[1], now[1], f"{label} tick {k} group_out")
        assert np.array_equal(engine.resident_occupancy(), R.occupancy_of(m[3], len(t.nodes))), f"{label} tick {k}"
        prev = now


@pytest.mark.parametrize("label", LABELS)
def test_pipelined_ticks(engine, label):
    """Two ticks in flight (resident_tick_submit / _wait): each tick's lists are the oracle's diff."""
    w = W.world(label)
    t = w.tables
    _load(engine, t)
    m = _mirrors(t)
    states = [_oracle(t, m)]
    for tick in w.plan:
        W.apply_tick(tick, *m)
        states.append(_oracle(t, m))
    ticks = _arena_ticks(engine, w.plan, t.flags)
    engine.resident_tick_submit(ticks[0])
    for k in range(1, len(ticks)):
        engine.resident_tick_submit(ticks[k])
        _check_tick(label, k - 1, engine.resident_tick_wait(), states[k - 1], states[k])
    _check_tick(label, len(ticks) - 1, engine.resident_tick_wait(), states[-2], states[-1])
    full = engine.resident_outputs()
    _same(full[0], states[-1][0], f"{label} lws_out")
    _same(full[1], states[-1][1], f"{label} group_out")


@pytest.mark.parametrize("label", LABELS)
def test_graph_replayed_ticks(graph_engine, label):
    """LWSE_TICK_GRAPH=2: the plan twice over (each of the two tick slots runs eagerly once, is captured,
    then replayed) — full outputs and change lists after every tick."""
    engine = graph_engine
    w = W.world(label)
    t = w.tables
    _load(engine, t)
    m = _mirrors(t)
    prev = _oracle(t, m)
    ticks = _arena_ticks(engine, w.plan, t.flags)
    replayed = 0
    for k in range(2 * len(ticks)):
        tick = w.plan[k % len(ticks)]
        W.apply_tick(tick, *m)
        now = _oracle(t, m)
        res = engine.resident_tick(ticks[k % len(ticks)])
        replayed += engine.resident_tick_info()["graph"]
        _check_tick(label, k, res, prev, now)
        full = engine.resident_outputs()
        _same(full[0], now[0], f"{label} tick {k} lws_out")
        _same(full[1], now[1], f"{label} tick {k} group_out")
        prev = now
    assert replayed >= 2 * len(ticks) - 2, label
