"""The DS drain edge worlds (tests/ds_drain_edges_world.py) without a GPU: the launch constants and refusal limits
they restate against the kernel and engine sources, every case on its declared side of its edge for a few SM
counts, each world holding what its labels say, and the vectorised per-key restatement against
``ds_drain_cost_ref`` and against set-form answers."""
import os
import re

import numpy as np
import pytest

import ds_drain_edges_world as X
from ds_drain_ref import (COST_FIELDS, cost_row_of, ds_drain_cost_ref, ds_drain_domains_ref, ds_drain_ref, link_targets,
                          lost_ref)
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lws_b200", "csrc")
SMS = (1, 16, 78, 114, X.H100_SMS)


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def _body(src, signature):
    """The text of the function that starts at ``signature``, up to its closing brace at column 0."""
    i = src.index(signature)
    return src[i: src.index("\n}\n", i)]


# --------------------------------------------------------------------------- #
# constants
# --------------------------------------------------------------------------- #
def test_constants_match_the_sources():
    ds = _src("lwse_ds_kernels.cu")
    grid = _body(ds, "static unsigned ds_grid(")
    m = re.search(r"want = \(n_ds \+ (\d+)u\) / (\d+)u, cap = \(uint32_t\)sm_count \* (\d+)u;", grid)
    assert int(m.group(1)) + 1 == int(m.group(2)) == X.DS_THREADS and int(m.group(3)) == X.DS_CAP
    # the drain sweep, the diff and both links passes: ds_grid CTAs of DS_THREADS
    for k in ("ds_sweep_kernel<false, true>", "ds_drain_diff_kernel", "ds_drain_links_kernel<true>",
              "ds_drain_links_kernel<false>"):
        assert re.search(re.escape(k) + rf"<<<ds_grid\(t->n_ds, sm_count\), {X.DS_THREADS}, 0, s>>>", ds), k
    dr = _src("lwse_drain_kernels.cu")
    assert f"__launch_bounds__({X.LOST_THREADS}) ds_drain_lost_kernel" in dr
    assert (f"ds_drain_lost_kernel<<<grid_for(n_lws, {X.LOST_THREADS} / 32, (uint32_t)sm_count * {X.LOST_CAP}u), "
            f"{X.LOST_THREADS}, 0, s>>>") in dr
    assert (f"lws_grid = grid_for((uint64_t)p->lws_mask + 1, {X.COST_THREADS}, (uint32_t)sm_count * {X.COST_CAP}u);"
            in dr)
    for k in ("ds_drain_pairs_kernel", "ds_drain_insert_kernel"):
        assert f"{k}<<<lws_grid, {X.COST_THREADS}, 0, s>>>" in dr, k
    assert (f"ds_drain_finish_kernel<<<grid_for((uint64_t)p->table_mask + 1, {X.COST_THREADS}, (uint32_t)sm_count * "
            f"{X.COST_CAP}u), {X.COST_THREADS}, 0, s>>>") in dr
    for k in ("ds_drain_pairs_kernel", "ds_drain_insert_kernel", "ds_drain_finish_kernel"):
        assert f"__launch_bounds__({X.COST_THREADS}) {k}" in dr, k
    # every grid-stride loop of the five kernels strides by the whole grid
    for k, step in (("ds_drain_lost_kernel", "L += n_warps"), ("ds_drain_pairs_kernel", "h += gridDim.x * blockDim.x"),
                    ("ds_drain_insert_kernel", "h += gridDim.x * blockDim.x"),
                    ("ds_drain_finish_kernel", "h += gridDim.x * blockDim.x")):
        assert step in _body(dr, f") {k}("), k
    for k in ("ds_drain_diff_kernel", "ds_drain_links_kernel"):
        assert "d += gridDim.x * blockDim.x" in _body(ds, f") {k}("), k
    ns = _src("lwse_place_ns_kernels.cu")
    assert int(re.search(r"constexpr uint32_t kIndexScanThreads = (\d+);", ns).group(1)) == X.INDEX_SCAN_THREADS
    scan = _body(ns, "__global__ void __launch_bounds__(kIndexScanThreads) place_index_scan_kernel")
    assert "a.first[a.n] = s_carry;" in scan
    lc = _src("lwse_launch.cuh")
    assert int(re.search(r"kDsDrainNewSlot = 0x([0-9A-F]+)u;", lc).group(1), 16) == X.NEW_SLOT
    assert int(re.search(r"kDsDrainSpec = 0x([0-9A-F]+)u;", lc).group(1), 16) == X.SPEC
    cost = _body(_src("lwse_engine.cu"), "LWSE_API int lwse_resident_ds_drain_cost(")
    limit = int(np.log2(X.REFUSE_ABOVE))
    for what in ("n_entries", "pairs", "ds_pairs"):
        assert len(re.findall(rf"\bif \({what} > \(1ull << {limit}\)\) return LWSE_ERR_OOM;", cost)) == 1, what
        assert len(re.findall(rf"\b{what} > ", cost)) == 1, what
    # both refusals read at the first synchronisation come before the next launch
    sync1 = cost.index("cudaStreamSynchronize(s)")
    fill = cost.index("launch_ds_drain_links(&t, &lk, d_count, d_cursor, (uint4*)")
    assert sync1 < cost.index("n_entries > ") < fill and sync1 < cost.index("pairs > (1ull") < fill
    assert "uint64_t ds_slots = 256;" in cost and "while (ds_slots < 2 * ds_pairs) ds_slots <<= 1;" in cost


def test_grid_arithmetic():
    assert X.ds_grid(1, 132) == 1 and X.ds_grid(16 * 128 * 132, 132) == 16 * 132
    assert X.ds_stride(132) == 270_336 and X.lost_stride(132) == 8448 and X.cost_stride(132) == 270_336
    assert X.grid_for(0, 256, 8) == 1


# --------------------------------------------------------------------------- #
# 1. limit DS
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def limit():
    e = X.world("limit")
    return e, {c.label: (c, ds_drain_ref(e.w, [c.node])) for c in e.cases}


def test_limit_shapes(limit):
    e, _ = limit
    ds = e.w.ds
    for V in X.LIMIT_V:
        for S, Xr in X.LIMIT_ROLES:
            d = e.notes[f"V{V}_S{S}_X{Xr}"]
            assert (int(ds["n_old_revs"][d]), int(ds["n_spec_roles"][d]), int(ds["n_roles"][d])) == (V, S, S + Xr)
    # every existing row links to a child of its own, accepted by the link rule
    L = link_targets(e.w.revroles, e.w.links, e.w.lws, e.w.base[0])
    ex = (e.w.revroles["flags"] & R.RR_EXISTS) != 0
    assert (L[ex] >= 0).all() and (L[~ex] < 0).all() and len(np.unique(L[ex])) == int(ex.sum())


def test_limit_cases(limit):
    """Each case's drain touches its DS alone, zeroes its row alone (or none), and gives its expected masks and
    verdicts; the label's facts about the DS hold before and after."""
    e, got = limit
    w = e.w
    for label, (c, (rows, tot, _, _)) in got.items():
        x = c.expect
        if x["rows_touched"] == 0:
            assert tot["n_touched"] == 0 and tot["rows_touched"] == 0, label
            continue
        assert tot["n_touched"] == 1 and tot["rows_touched"] == 1 and tot["rows_zeroed"] == x["rows_zeroed"], label
        r = rows[0]
        assert int(r["ds"]) == c.ds, label
        for f in ("rows_touched", "rows_zeroed", "new_zeroed_roles", "old_zeroed_roles"):
            assert int(r[f]) == x[f], (label, f)
        fl = int(r["flags"])
        assert fl & x["set"] == x["set"] and not fl & x["clear"], (label, fl)
        b, a = int(r["before"]["ready_revs"]), int(r["after"]["ready_revs"])
        assert b & ~a == x["fell"], label
        if "stable_before" in x:
            assert bool(r["before"]["flags"] & R.DOUT_STABLE) == x["stable_before"], label
        if "ready_bit_clear_before" in x:
            assert not (b >> x["ready_bit_clear_before"]) & 1, label
        if "drained_bit" in x:
            assert (int(r["before"]["drained_revs"]) >> x["drained_bit"]) & 1, label
        if x.get("init"):
            assert r["before"]["flags"] & R.DOUT_INIT and r["before"]["flags"] & R.DOUT_ROLLING, label
        # the zeroed row is the case's row
        lost = lost_ref(w, [c.node])
        L = link_targets(w.revroles, w.links, w.lws, w.base[0])
        hit = np.flatnonzero((L >= 0) & (lost[np.maximum(L, 0)] > 0))
        assert list(hit) == [c.row], label
    labels = set(got)
    # bit 31 of ready_revs falls; role 9 of the new revision; removed roles of a stable DS do not stall
    assert "old31_spec_role9_V32_S10_X0" in labels and "new_spec_role9_V32_S10_X0" in labels
    r = got["old31_spec_role9_V32_S10_X0"][1][0][0]
    assert r["before"]["ready_revs"] == 0xFFFFFFFF and r["after"]["ready_revs"] == 0x7FFFFFFF
    r = got["new_removed_role9_V32_S9_X1"][1][0][0]
    assert r["before"]["flags"] & R.DOUT_STABLE and r["after"]["flags"] & R.DOUT_STABLE
    assert not r["flags"] & R.DSD_STALLS
    # every shape has a case on its new revision's last role and, with V > 0, on its last old revision's
    for V in X.LIMIT_V:
        for S, Xr in X.LIMIT_ROLES:
            i, tag = S + Xr - 1, "spec" if Xr == 0 else "removed"
            assert f"new_{tag}_role{i}_V{V}_S{S}_X{Xr}" in labels
            assert (f"old{V - 1}_{tag}_role{i}_V{V}_S{S}_X{Xr}" in labels) == (V > 0)
    for ready, lost in X.MATRIX:
        assert f"ready{ready}_lost{lost}" in labels


def test_lost_never_exceeds_ready_before():
    """ready_after < 0 needs lost(L, key) > ready_before(L).  The LWS sweep counts every COND_READY group in an
    object's range as ready, and lost counts only COND_READY groups of the range that name the object, so no child
    of the limit or child-edge worlds — replicas 0 and -4, surge groups, foreign and overlapping groups included —
    gives one: the clamp of ready_after is never below 0 in them."""
    for label in ("limit", "child_edges"):
        w = X.world(label).w
        ready = w.base[0]["ready_replicas"].astype(np.int64)
        for by_domain in (False, True):
            L, _, lost = X.lost_pair_arrays(w, by_domain)
            assert len(L) and (lost <= ready[L]).all(), label
    # the surge child: more COND_READY groups than replicas, all counted ready
    e = X.world("child_edges")
    s = e.notes["named"]["surge"]
    assert int(e.w.base[0]["ready_replicas"][s]) > int(e.w.lws["replicas"][s])


# --------------------------------------------------------------------------- #
# 2. child LWS edges
# --------------------------------------------------------------------------- #
def test_child_edges_world():
    e = X.world("child_edges")
    w, named = e.w, e.notes["named"]
    for g in (31, 32, 33, 64, 65, 1000):
        assert int(w.lws["group_count"][named[f"rows_{g}"]]) == g
    assert int(w.lws["replicas"][named["replicas_0"]]) == 0 and int(w.lws["replicas"][named["replicas_m4"]]) == -4
    hg = e.notes["host_group"]
    h = named["host"]
    assert int(w.lws["group_base"][h]) <= hg < int(w.lws["group_base"][h] + w.lws["group_count"][h])
    assert int(w.groups["lws_index"][hg]) == named["other"]
    a, b = named["overlap_a"], named["overlap_b"]
    assert int(w.lws["group_base"][b]) < int(w.lws["group_base"][a] + w.lws["group_count"][a])
    p = named["past"]
    assert int(w.lws["group_base"][p] + w.lws["group_count"][p]) > len(w.groups)
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    for name, row in named.items():
        vb = int(w.ds["rev_base"][e.notes["ds_of"][row]])
        assert (w.links["lws_row"][vb: vb + 4] == row).all(), name  # four rows of one DS, one child
    lost_any = np.zeros(len(w.lws), bool)
    for by_domain in (False, True):
        lost_any[X.lost_pair_arrays(w, by_domain)[0]] = True
    # the children the walk reaches lose groups through linked rows; the range past the table loses none
    for name in ("rows_31", "rows_32", "rows_33", "rows_64", "rows_65", "rows_1000", "surge", "host", "overlap_a"):
        assert lost_any[named[name]] and (L == named[name]).any(), name
    assert not lost_any[p]


# --------------------------------------------------------------------------- #
# 3. fan-out and the scan
# --------------------------------------------------------------------------- #
def test_fan_worlds():
    for label, rows in (("fan_330", 330), ("fan_100k", X.FAN_ROWS)):
        e = X.world(label)
        w = e.w
        L = link_targets(w.revroles, w.links, w.lws, w.base[0])
        assert (L == e.notes["child"]).all() and len(L) == e.notes["rows"] >= rows
        assert int(w.ds["n_old_revs"][0]) == 32 and int(w.ds["n_roles"][0]) == 10
        pl, pk, lost = X.lost_pair_arrays(w, False)
        c = e.notes["child"]
        assert [(int(a), int(b)) for a, b, x in zip(pl, pk, lost) if a == c] == [(c, 0)] and lost[pl == c] == 1
    _, tot, _, _ = ds_drain_ref(X.world("fan_330").w, [0])
    assert tot["rows_zeroed"] == 330 and tot["n_service_lost"] == tot["n_old_service_lost"] == tot["n_stalled"] == 1


def test_scan_worlds_on_chunk_edges():
    C = X.INDEX_SCAN_THREADS
    sides = {}
    for n in X.SCAN_N_LWS:
        e = X.world(f"scan_{n}")
        w = e.w
        assert len(w.lws) == n and e.notes["last"] == n - 1
        L = link_targets(w.revroles, w.links, w.lws, w.base[0])
        assert set(L.tolist()) == {n - 1}
        pl, pk, _ = X.lost_pair_arrays(w, False)
        assert (n - 1, 0) in set(zip(pl.tolist(), pk.tolist())) and all(l_ != n - 1 for l_, k in zip(pl, pk) if k)
        sides[n] = (n - 1) // C, n % C  # the chunk holding the last row's count, and first[n]'s offset in its chunk
    assert sides == {1023: (0, 1023), 1024: (0, 0), 1025: (1, 1), 2049: (2, 1)}


# --------------------------------------------------------------------------- #
# 4. grids
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("sms", SMS)
def test_grid_ds_cases_on_their_side(sms):
    G = X.ds_stride(sms)
    n_ds = G + 37
    assert X.ds_grid(n_ds, sms) == X.DS_CAP * sms and n_ds > G  # every ds_grid kernel runs a second pass
    e = X.grid_ds_world(sms) if sms <= 16 else None
    last = [G + 30, G + 31, G + 32, G + 33, G + 36, G]
    assert all(d >= G for d in last) and (G + 32) % 32 == 0  # G + 31 | G + 32: both sides of a warp boundary
    if e is not None:
        w = e.w
        L = link_targets(w.revroles, w.links, w.lws, w.base[0])
        assert (L[last] >= 0).all() and L[G - 1] >= 0 and (L[G + 1: G + 30] < 0).all()
        for c in e.cases:
            rows, tot, _, _ = ds_drain_ref(w, [c.node])
            assert c.ds in rows["ds"], c.label
        rows = ds_drain_ref(w, [e.cases[0].node])[0]
        assert list(rows["ds"]) == [G + 31, G + 32]


@pytest.mark.parametrize("sms", (1, 16, X.H100_SMS))
def test_grid_links_cases_on_their_side(sms):
    e = X.world(f"grid_links_{sms}")
    w = e.w
    n = len(w.lws)
    assert n > X.lost_stride(sms) and n > X.ds_stride(sms)
    pl, pk, lost = X.lost_pair_arrays(w, False)
    c = e.cases[0]
    # lost groups in the lost kernel's last stride, reached by the drained node
    assert c.ds // X.lost_stride(sms) == (n - 1) // X.lost_stride(sms) >= 1 and ((pl == c.ds) & (pk == c.node)).any()
    # the (LWS, key) table (at least 2 x its entries) is past the pairs / insert grid, and the (DS, key) table past
    # the finish grid
    v = X.ds_drain_cost_vec(w, False)
    assert 2 * len(pl) > X.cost_stride(sms)
    assert 2 * int(v["ds_touched"].sum()) > X.cost_stride(sms)
    assert int(v["ds_touched"].sum()) > X.COST_CAP * sms * 128


# --------------------------------------------------------------------------- #
# 5. refusals
# --------------------------------------------------------------------------- #
def test_refusal_counts():
    """Both sides of the (DS, key) pairs and index entries limits; the accepted sides would allocate 32 GiB and
    16 GiB, so they are checked here only."""
    for n_ds, refused in ((X.PAIRS_REFUSED, True), (X.PAIRS_ACCEPTED, False)):
        w = X.refuse_pairs_world(n_ds).w
        pairs = X.ds_pairs_of(w, False)
        assert pairs == n_ds * 330 * 1024 and (pairs > X.REFUSE_ABOVE) == refused
        assert X.ds_pairs_of(w, True) <= X.REFUSE_ABOVE  # (the domain scope is accepted and large: never called)
        assert n_ds * 330 <= X.REFUSE_ABOVE
    assert X.PAIRS_REFUSED * 330 * 1024 == 1_073_909_760 and X.PAIRS_ACCEPTED * 330 * 1024 == 1_073_571_840
    for n_ds, refused in ((X.ENTRIES_REFUSED, True), (X.ENTRIES_ACCEPTED, False)):
        assert (n_ds * X.SHARED_ROWS > X.REFUSE_ABOVE) == refused
    w = X.refuse_entries_world().w
    assert len(w.ds) == X.ENTRIES_REFUSED
    assert (w.ds["rev_base"] == 0).all() and (w.ds["n_old_revs"] == 32).all() and (w.ds["n_roles"] == 10).all()
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    assert sorted(L.tolist()) == list(range(330))  # 330 children, one counter each
    assert X.ENTRIES_REFUSED * 330 == 1_073_742_120 and X.ENTRIES_ACCEPTED * 330 == 1_073_741_790


# --------------------------------------------------------------------------- #
# the vectorised per-key form
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("label", X.SMALL + ("fan_100k", "grid_ds_1"))
def test_vec_equals_cost_ref(label):
    w = X.world(label).w
    for by_domain in (False, True):
        assert X.ds_drain_cost_vec(w, by_domain).tobytes() == ds_drain_cost_ref(w, by_domain).tobytes(), by_domain


@pytest.mark.parametrize("label", ("limit", "child_edges"))
def test_vec_equals_set_form(label):
    e = X.world(label)
    w = e.w
    nodes = sorted({c.node for c in e.cases} | set(range(0, len(w.nodes), 7))) if label == "limit" else range(len(w.nodes))
    for by_domain, keys in ((False, nodes), (True, range(w.n_domains))):
        v = X.ds_drain_cost_vec(w, by_domain)
        for k in keys:
            tot = (ds_drain_domains_ref(w, [k]) if by_domain else ds_drain_ref(w, [k]))[1]
            assert cost_row_of(tot) == {f: int(v[f][k]) for f in COST_FIELDS}, (by_domain, k)
