"""The placement round on every launch path at that path's thresholds (tests/place_edges_world.py), bit for
bit against the spec oracle on the same node table, occupancy, domain count and namespace count:
general form through ``place_host`` and ``place_device``, namespace forms through
``place_grouped_device``, and the resident tick."""
import numpy as np
import pytest

import place_edges_world as W
from lws_b200 import records as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from lws_b200.engine import Engine

    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def same(got, want, what):
    for name in want.dtype.names:
        a, b = got[name], want[name]
        if not np.array_equal(a, b):
            i = int(np.flatnonzero(a != b)[0])
            raise AssertionError(f"{what}.{name}: {int((a != b).sum())} rows differ; row {i}: got {a[i]} want {b[i]}")


def _up(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to("cuda:0")


def _want(c, reqs):
    import oracle

    return oracle.place(c.nodes, c.occ, c.n_domains, c.n_namespaces, reqs, threads=16)


@pytest.mark.parametrize("name", W.GENERAL)
def test_general_form_paths(engine, sm_count, name):
    """G1-G4 — the cluster at 1 024 requests (8 per warp, half of them in their result rows) and the grid at
    1 025; a quiet call, a burst that the quiet history sends to the cluster (128 per warp) and the same
    burst on the grid; the grid with more than 4 x GW unpinned requests; the cluster's node (65 536 /
    65 537) and holder-table (65 536 / 65 552 keys, odd domain count) bounds and the 16-CTA grid floor.
    Each call in order through ``place_host``, then again through ``place_device`` after a fresh upload."""
    import torch

    c = W.BUILDERS[name](sm_count)
    assert [x["path"] for x in W.general_calls(c, sm_count)] == c.paths
    wants = [_want(c, reqs) for reqs in c.calls]
    engine.upload_nodes(c.nodes, c.n_domains)  # (a fresh geometry: no history)
    for k, (reqs, want) in enumerate(zip(c.calls, wants)):
        got, rounds = engine.place_host(reqs, c.occ, c.n_namespaces)
        torch.cuda.synchronize()  # (the unpinned count the next call's path depends on has landed)
        same(got, want, f"{name} host call {k} ({c.paths[k]})")
        assert rounds >= 1
    engine.upload_nodes(c.nodes, c.n_domains)
    d_occ = _up(c.occ)
    for k, (reqs, want) in enumerate(zip(c.calls, wants)):
        d_reqs = _up(reqs)
        d_out = torch.zeros(len(reqs) * R.PLACE_OUT.itemsize, dtype=torch.uint8, device="cuda:0")
        engine.place_device(d_reqs, len(reqs), d_occ, c.n_namespaces, d_out)
        torch.cuda.synchronize()  # (the unpinned count the next call's path depends on has landed)
        same(d_out.cpu().numpy().view(R.PLACE_OUT), want, f"{name} device call {k} ({c.paths[k]})")


@pytest.mark.parametrize("name", W.NAMESPACE)
def test_namespace_form_paths(engine, sm_count, name):
    """N1, N2, N4, N5 — namespaces of 256 / 257 / 640 live unpinned requests (state past 256 in the result
    rows), of 512 / 513 and 1 024 / 1 025 rows with pinned claims decided past the kept positions, the scan
    form's word table staged and not (11 520 / 11 521 nodes, 9 728 / 9 729 at 1 000 domains), and
    2 x sm_count + 5 namespaces whose CTAs find their work late or never — two-level and scan, each twice
    in a row (the scratch counters alternate between calls)."""
    import torch

    c = W.BUILDERS[name](sm_count)
    reqs = c.calls[0]
    assert W.ns_view(c, sm_count)["supported"]
    want = _want(c, reqs)
    engine.upload_nodes(c.nodes, c.n_domains)
    d_reqs, d_occ = _up(reqs), _up(c.occ)
    d_out = torch.zeros(len(reqs) * R.PLACE_OUT.itemsize, dtype=torch.uint8, device="cuda:0")
    live = int(W.live_unpinned(reqs, c.n_namespaces).sum())
    for flags, form in ((0, "two-level"), (R.SWEEP_PLACE_SCAN, "scan")):
        for k in range(2):
            d_out.fill_(0xA5)
            rounds, scans = engine.place_grouped_device(d_reqs, len(reqs), d_occ, c.n_namespaces, d_out, flags=flags,
                                                        want_rounds=True)
            same(d_out.cpu().numpy().view(R.PLACE_OUT), want, f"{name} {form} call {k}")
            assert rounds >= 1 and scans >= live


def _pods(occ):
    """Identity rows whose scheduled pods give ``occ`` per node (the resident tables count it themselves)."""
    node = np.repeat(np.arange(len(occ), dtype=np.uint64), occ.astype(np.int64))
    pid = R.pod_ident_table(np.arange(len(node), dtype=np.uint64), np.zeros(len(node), np.uint32),
                            (R.PODID_SCHEDULED | (node << np.uint64(R.PODID_NODE_SHIFT))).astype(np.uint32))
    pst = R.aligned_empty(len(node), R.POD_STATE)
    pst[:] = 0
    return pst, pid


def _resident(engine, c, reqs, flags):
    pst, pid = _pods(c.occ)
    engine.upload_nodes(c.nodes, c.n_domains)
    engine.resident_load(R.aligned_empty(0, R.LWS_REC), R.aligned_empty(0, R.GROUP_REC), pst, pid)
    assert np.array_equal(engine.resident_occupancy(), c.occ)
    engine.resident_place_load(reqs, c.n_namespaces)
    return engine.resident_tick(engine.make_tick((), flags))


def _patch_tick(engine, c, reqs, prev, flags, seed):
    """One tick of request-row patches (pins, unpins, new sizes): its change list against the oracle."""
    rng = np.random.default_rng(seed)
    rows = np.sort(rng.choice(len(reqs), size=max(8, len(reqs) // 50), replace=False)).astype(np.uint32)
    vals = R.aligned_empty(len(rows), R.PLACE_REQ)
    vals[:] = reqs[rows]
    pin = rng.random(len(rows)) < 0.3
    vals["leader_node"] = np.where(pin, rng.integers(0, len(c.nodes), size=len(rows)), R.NONE).astype(np.uint32)
    vals["size"] = rng.integers(-1, 4, size=len(rows))
    mirror = reqs.copy()
    mirror[rows] = vals
    res = engine.resident_tick(engine.make_tick([(R.TABLE_PLACE_REQS, rows, vals)], flags))
    want = _want(c, mirror)
    assert engine.resident_place_outputs().tobytes() == want.tobytes()
    changed = np.flatnonzero((want.view(np.uint8).reshape(len(want), -1) != prev.view(np.uint8).reshape(len(prev), -1)).any(axis=1))
    assert len(changed) > 0 and res["n_place"] == len(changed)
    order = np.argsort(res["place_rows"])
    assert np.array_equal(res["place_rows"][order], changed)
    assert res["place_out"][order].tobytes() == want[changed].tobytes()


@pytest.mark.parametrize("name", W.TICK)
def test_tick_form_at_the_domain_limit(engine, sm_count, name):
    """N3 — the resident tick runs the namespace form at 5 456 domains (its shared memory just fits) and the
    general form at 5 457, as the mirror says; the rows, and a tick of request patches, equal the oracle's."""
    c = W.BUILDERS[name](sm_count)
    reqs = c.calls[0]
    flags = R.TICK_PLACE | R.TICK_NO_SWEEP
    res = _resident(engine, c, reqs, flags)
    info = engine.resident_tick_info()
    assert info["form"] == ("namespace" if W.place_ns_supported(len(c.nodes), c.n_domains) else "general")
    assert info["form"] == ("namespace" if c.n_domains == W.NS_DOMAIN_LIMIT else "general")
    want = _want(c, reqs)
    assert engine.resident_place_outputs().tobytes() == want.tobytes()
    assert res["n_place"] == len(reqs)
    _patch_tick(engine, c, reqs, want, flags, seed=5)


@pytest.mark.parametrize("scan", [False, True], ids=["two_level", "scan"])
def test_tick_indexed_cache_overflow(engine, sm_count, scan):
    """N1 through the resident tick with the request table ungrouped (the indexed form): namespaces of
    256 / 257 / 640 live unpinned requests reached through the namespace index; then a tick of patches."""
    from test_gpu_lifecycle import ungroup

    c = W.BUILDERS["n1_cache"](sm_count)
    reqs = ungroup(c.calls[0])
    assert list(np.bincount(reqs["ns"][W.live_unpinned(reqs, c.n_namespaces)], minlength=4)) == [256, 257, 640, 0]
    flags = R.TICK_PLACE | R.TICK_NO_SWEEP | (R.SWEEP_PLACE_SCAN if scan else 0)
    _resident(engine, c, reqs, flags)
    info = engine.resident_tick_info()
    assert info["form"] == ("scan" if scan else "namespace") and info["indexed"]
    want = _want(c, reqs)
    assert engine.resident_place_outputs().tobytes() == want.tobytes()
    _patch_tick(engine, c, reqs, want, flags, seed=6)
