"""The drain edge worlds (tests/drain_edges_world.py) without a GPU: the constants they restate against the
kernel and engine sources, every case on its declared side of its edge (the restated warp walk's list
overflow, the (LWS, key) table's size and probe wrap, group counts per LWS row, the grid caps, the int32
floor), and the drain references against each other on the new worlds."""
import os
import re

import numpy as np
import pytest

import drain_edges_world as W
import oracle
from drain_budget_ref import budgets, domain_nodes, drain_budget_cost_ref, drain_budget_ref, key_of, owners
from drain_ref import COST_OF, TOTALS, drain_cost_ref, drain_whatif_ref, restart_pairs
from lws_b200 import records as R
from test_drain_budget import check_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lws_b200", "csrc")


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def _base(w):
    return oracle.sweep_lws(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, w.flags)[:2]


_BASES = {}


def base_of(label):
    if label not in _BASES:
        _BASES[label] = _base(W.world(label))
    return _BASES[label]


# --------------------------------------------------------------------------- #
# the restated constants
# --------------------------------------------------------------------------- #
def test_constants_match_the_sources():
    src = _src("lwse_drain_kernels.cu")
    assert int(re.search(r"constexpr uint32_t kCostList = (\d+);", src).group(1)) == W.K_COST_LIST
    assert int(re.search(r"constexpr uint32_t kCostThreads = (\d+);", src).group(1)) == W.K_COST_THREADS
    caps = {m.group(1): int(m.group(3)) for m in re.finditer(
        r"(\w+_kernel)(<\w+>)?<<<grid_for\([^;]*?sm_count \* (\d+)u\)", src)}
    caps["drain_budget_walk_kernel"] = int(re.search(r"walk_grid = grid_for\([^;]*?sm_count \* (\d+)u\)", src).group(1))
    for k, v in W.GRID_CAP.items():
        assert caps[k] == v, k
    for k in ("drain_mark_kernel", "drain_diff_kernel", "drain_domain_mask_kernel", "drain_budget_kernel"):
        assert re.search(k + r"<<<[^;]*, 256, 0, s>>>", src), k
    mix = re.search(r"table_slot\(unsigned long long k, uint32_t mask\) \{(.*?)\n\}", src, re.S).group(1)
    assert f"0x{W.MIXER:X}ull" in mix and mix.count(">> 33") == 2
    eng = _src("lwse_engine.cu")
    assert f"uint64_t slots = {W.TABLE_MIN_SLOTS};" in eng
    assert f"while (slots < {W.TABLE_PAIRS_FACTOR} * pairs) slots <<= 1;" in eng


def test_table_slot_restatement():
    """The mixer restated: a few values worked by hand with 64-bit wraparound."""
    for k in (0, 1, 5 << 32 | 17, (1 << 64) - 2):
        x = k ^ (k >> 33)
        x = (x * W.MIXER) % (1 << 64)
        x ^= x >> 33
        assert W.table_slot(k, 0xFFFF) == x & 0xFFFF
    assert [W.table_slots(p) for p in (1, 127, 128, 129, 256, 257)] == [256, 256, 256, 512, 512, 1024]


# --------------------------------------------------------------------------- #
# the walk: every group on its side of the list's edge
# --------------------------------------------------------------------------- #
def group_keys(w, by_domain, base_out):
    """{group row: per-pod keys (NONE for a pod that restarts nothing)} for every group with a restart pair.
    The restarting pods come from ``restart_pairs`` over a copy of the identity rows in which every pod bound
    to a node of the table stands on a node row of its own (its pod row), so that each pair names the pod."""
    n_nodes, P = len(w.nodes), len(w.pod_ident)
    assert P <= R.POD_NODE_MAX
    place = w.pod_ident["place"].astype(np.int64)
    node = place >> R.PODID_NODE_SHIFT
    bound = ((place & R.PODID_SCHEDULED) != 0) & (node < n_nodes)
    low = place & ((1 << R.PODID_NODE_SHIFT) - 1)
    pid = w.pod_ident.copy()
    pid["place"] = np.where(bound, low | (np.arange(P) << R.PODID_NODE_SHIFT), low & ~R.PODID_SCHEDULED)
    g, p = restart_pairs(w.lws, w.groups, w.pod_state, pid, P, base_out)
    key = key_of(w.nodes, w.n_domains, by_domain)
    out = {}
    for gg in np.unique(g).tolist():
        base, cnt = int(w.groups[gg]["pod_base"]), int(w.groups[gg]["pod_count"])
        keys = [W.NONE] * cnt
        for q in p[g == gg].tolist():
            keys[q - base] = int(key[node[q]])
        out[gg] = keys
    return out


@pytest.fixture(scope="module")
def walks():
    w = W.world("walk")
    base = base_of("walk")
    out = {}
    for scope, by_domain in (("nodes", False), ("domains", True)):
        keys = group_keys(w, by_domain, base[1])
        g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base[1])
        kk = key_of(w.nodes, w.n_domains, by_domain)[n]
        want = {}
        for gg, k in zip(g.tolist(), kk.tolist()):
            if k >= 0:
                want.setdefault(gg, set()).add(k)
        out[scope] = {gg: (keys[gg], W.warp_walk(keys[gg]), want.get(gg, set())) for gg in keys}
    return w, out


def test_walk_fresh_pairs_equal_restart_pairs(walks):
    """Every group, both scopes: the restated walk's fresh keys are restart_pairs' keys, each once."""
    _, out = walks
    for scope, per in out.items():
        for g, (_, walk, want) in per.items():
            assert sorted(walk.fresh) == sorted(want), (scope, g)
            assert len(set(walk.fresh)) == len(walk.fresh), (scope, g)


def test_walk_list_edges(walks):
    w, out = walks
    n = w.notes
    nodes, doms = out["nodes"], out["domains"]
    # 63 and 64 distinct nodes stay in the list; the 65th overflows it in the third batch (the earliest)
    for name, k in (("distinct_63", 63), ("distinct_64", 64)):
        _, walk, want = nodes[n[name]]
        assert len(want) == k and walk.overflow is None and walk.listed == k, name
    keys, walk, want = nodes[n["distinct_65_early"]]
    assert len(want) == 65 and walk.overflow == 2 and walk.listed == 64
    b2 = keys[64:96]
    assert any(k in keys[:64] for k in b2) and any(k not in keys[:64] and k >= 0 for k in b2)
    assert any(k in b2 and k not in keys[:64] for k in keys[96:])  # the overflowing batch's key repeats later
    # a late overflow: batch 6; keys of the list, of batch 6 and of batch 7 repeat in batches 7-9
    keys, walk, want = nodes[n["distinct_late"]]
    assert walk.overflow == 6 and walk.listed == 60 and len(want) > 65
    lst, b6, b7 = set(keys[:192]), set(keys[192:224]) - set(keys[:192]), set(keys[224:256]) - set(keys[:224])
    later = keys[224:]
    assert lst & set(later) and b6 & set(later) and b7 and b7 & set(keys[256:])
    # a duplicate key in one batch, its lanes split by every failing kind of pod
    keys, walk, want = nodes[n["dup_in_batch"]]
    assert len(want) == 2 and keys.count(W.NONE) == 15 and walk.overflow is None
    # DOMAINS: 64 and 65 distinct domains through more nodes; both overflow the node list
    for name, k, over in (("domains_64", 64, None), ("domains_65", 65, 8)):  # (4 pods per domain: batch 8)
        keys, walk, want = doms[n[name]]
        assert len(want) == k and walk.overflow == over, name
        assert nodes[n[name]][1].overflow is not None and len(nodes[n[name]][2]) > 2 * k, name
        assert W.NONE in keys[1:5], name  # nodes of no domain and beyond the last between them
    # every pod count, the 5 003-pod group overflowing in both scopes
    counts = [int(w.groups[g]["pod_count"]) for g in n["counts"]]
    assert counts == list(W.WALK_POD_COUNTS)
    big = n["counts"][-1]
    assert nodes[big][1].overflow is not None and doms[big][1].overflow is not None
    assert len(nodes[big][2]) > 1000


def test_walk_pending_gate(walks):
    """The only pending pod at positions 0, 31, 32, 33 and pod_count - 1 closes the gate of AfterStart and of
    the annotation when size == pod_count; size != pod_count closes it with no pending pod at all."""
    w, out = walks
    open_groups = set(out["nodes"])  # (every leader here is bound to a node: a group has pairs iff its gate is open)
    for (policy, annot, size, at), g in w.notes["pending"].items():
        assert int(w.groups[g]["pod_count"]) == 65
        if at is not None:
            st = w.pod_state[int(w.groups[g]["pod_base"]): int(w.groups[g]["pod_base"]) + 65] & R.POD_PHASE_MASK
            assert np.flatnonzero(st == R.POD_PHASE_PENDING).tolist() == [at]
        assert (g in open_groups) == (size == 65 and at is None), (policy, annot, size, at)


def test_walk_overlapping_ranges():
    w = W.world("walk")
    g = w.groups
    for a, b in (w.notes["overlap_same"], w.notes["overlap_other"]):
        a0, a1 = int(g[a]["pod_base"]), int(g[a]["pod_base"] + g[a]["pod_count"])
        b0 = int(g[b]["pod_base"])
        assert a0 < b0 < a1
    _, base = base_of("walk")
    g_, n_ = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base)
    a, b = w.notes["overlap_same"]
    shared = set(n_[g_ == a].tolist()) & set(n_[g_ == b].tolist())
    assert len(shared) > 5  # the shared pods restart both groups


# --------------------------------------------------------------------------- #
# the budget edges
# --------------------------------------------------------------------------- #
def _floor_def(reps, mu, pct):
    m = (mu * reps) // 100 if pct else mu  # Python ints: never truncated
    return min(max(0, reps - m), W.I32_MAX)


def _floor_i32_mu(reps, mu, pct):
    """The floor with mu truncated to int32, as the unfixed kernel computed it."""
    m = (mu * reps) // 100 if pct else mu
    m = (m + (1 << 31)) % (1 << 32) - (1 << 31)
    return min(max(0, reps - m), W.I32_MAX)


def test_budget_edges():
    w = W.world("budget_edges")
    lo, go = base_of("budget_edges")
    own = owners(w.lws, w.groups)
    n = w.notes
    for k, o in n["rows"].items():
        if isinstance(k, int):
            assert int((own == o).sum()) == k, k
    assert {int((own == o).sum()) for o in n["rows"].values() if True} >= {31, 32, 33, 64, 65, 1000}
    floor, ready, evaluated, available, gb, gc = budgets(w.lws, lo, len(w.groups))
    # surge: index replicas - 1 and replicas, each alone on its node, the object Available
    o, g_in, g_surge = n["surge"]
    assert available[o] and evaluated[o]
    assert (g_in - gb[o], g_surge - gb[o]) == (w.lws[o]["replicas"] - 1, w.lws[o]["replicas"])
    # a row of another LWS inside a range, overlapping ranges, a range past the table
    host, row, other = n["host"]
    assert w.groups[row]["lws_index"] == other and gb[host] <= row < gb[host] + gc[host] and own[row] == -1
    a, b = n["overlap"]
    assert gb[b] < gb[a] + gc[a] and gc[b] > 0
    assert gc[n["past"]] == 0 and int(w.lws[n["past"]]["group_base"] + w.lws[n["past"]]["group_count"]) > len(w.groups)
    assert int(w.lws[n["rows"]["replicas_0"]]["replicas"]) == 0 and int(w.lws[n["rows"]["replicas_-4"]]["replicas"]) < 0


def test_int32_floors():
    """The floor of every int32-edge row against the definition in Python integers; three of them (a percentage
    above 100 whose mu passes 2^31) differ from the floor with mu truncated to int32."""
    w = W.world("budget_edges")
    lo, _ = base_of("budget_edges")
    floor, ready, evaluated, *_ = budgets(w.lws, lo, len(w.groups))
    wrapped = 0
    for o, (reps, mu, pct) in zip(w.notes["int32"], W.INT32_FLOORS):
        assert evaluated[o], o
        assert int(floor[o]) == _floor_def(reps, mu, pct), (reps, mu, pct)
        wrapped += _floor_i32_mu(reps, mu, pct) != _floor_def(reps, mu, pct)
    assert wrapped == 3
    o = w.notes["int32"][W.INT32_FLOORS.index((1 << 30, 300, True))]
    assert int(floor[o]) == 0 and _floor_i32_mu(1 << 30, 300, True) == W.I32_MAX


# --------------------------------------------------------------------------- #
# the table edges
# --------------------------------------------------------------------------- #
def member_pairs(w, base_out):
    g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base_out)
    return int((owners(w.lws, w.groups)[g] >= 0).sum())


@pytest.mark.parametrize("pairs,slots", [(128, 256), (129, 512)])
def test_table_size_edge(pairs, slots):
    label = f"pairs_{pairs}"
    assert member_pairs(W.world(label), base_of(label)[1]) == pairs
    assert W.table_slots(pairs) == slots


def test_probe_wraps():
    """Whatever order the entries go in, the chain homed at the last slot runs past it to slot 0 and on."""
    w = W.world("wrap")
    mask = w.notes["mask"]
    assert member_pairs(w, base_of("wrap")[1]) == 64 and W.table_slots(64) == mask + 1
    g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base_of("wrap")[1])
    entries = [int(w.groups[a]["lws_index"]) << 32 | int(b) for a, b in zip(g, n)]
    assert set(w.notes["entries"]) <= set(entries)
    homes = [W.table_slot(e, mask) for e in entries]
    assert homes.count(mask) >= 12 and homes.count(0) >= 4
    rng = np.random.default_rng(1)
    for _ in range(20):
        lay = W.probe_layout([entries[i] for i in rng.permutation(len(entries))], mask)
        wrapped = [e for e, (h, s) in lay.items() if s < h]
        assert len(wrapped) >= 11
        assert max((s - h) & mask for h, s in lay.values()) >= 15


# --------------------------------------------------------------------------- #
# the grid edges and the degenerate node tables
# --------------------------------------------------------------------------- #
def test_grid_edges():
    sms = W.H100_SMS
    t = W.grid_world(sms, "nodes")
    assert len(t.nodes) > W.GRID_CAP["drain_domain_mask_kernel"] * W.GRID_THREADS * sms
    t = W.grid_world(sms, "groups")
    G = len(t.groups)
    assert G > W.GRID_CAP["drain_mark_kernel"] * W.GRID_THREADS * sms          # the mark kernel's group loop
    assert G > 2 * W.GRID_CAP["drain_diff_kernel"] * W.GRID_THREADS * sms      # the diff's second stride
    assert len(t.lws) > W.GRID_CAP["drain_budget_kernel"] * (W.GRID_THREADS // 32) * sms  # the budget's L loop
    assert set(np.unique(t.groups["pod_count"]).tolist()) == {1, 2}
    assert np.array_equal(owners(t.lws, t.groups), t.groups["lws_index"].astype(np.int64))


def test_degenerate_node_tables():
    w = W.world("no_domains")
    assert w.n_domains == 0 and (key_of(w.nodes, 0, True) == -1).all()
    w = W.world("sparse_domains")
    assert w.n_domains > len(w.nodes) and (w.nodes["domain_id"] < w.n_domains).all()


# --------------------------------------------------------------------------- #
# the references against each other on the new worlds
# --------------------------------------------------------------------------- #
def _sample_nodes(label):
    w = W.world(label)
    if len(w.nodes) <= 128:
        return list(range(len(w.nodes)))
    g, n = restart_pairs(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base_of(label)[1])
    rng = np.random.default_rng(4)
    picks = set(rng.choice(np.unique(n), size=min(40, len(np.unique(n))), replace=False).tolist())
    if label == "walk":
        picks |= set(W.WALK_NO_DOMAIN[:2] + W.WALK_BEYOND[:2])
        for name in ("distinct_65_early", "domains_65"):
            picks |= set(n[g == w.notes[name]][:4].tolist())
    picks |= {0, len(w.nodes) - 1}
    return sorted(picks)


@pytest.mark.parametrize("label", ["walk"] + list(W.SMALL))
def test_cost_equals_the_whatif_of_each_node(label):
    w = W.world(label)
    base = base_of(label)
    cost = drain_cost_ref(w.lws, w.groups, w.pod_state, w.pod_ident, len(w.nodes), base[1])
    for n in _sample_nodes(label):
        got = drain_whatif_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, [n], w.flags, base=base)
        for k in TOTALS:
            assert int(cost[COST_OF[k]][n]) == got[k], (label, n, k)


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("label", ["budget_edges", "no_domains", "sparse_domains", "wrap"])
def test_per_key_equals_the_set_form(label, by_domain):
    w = W.world(label)
    base = base_of(label)
    cost = drain_budget_cost_ref(w.lws, base[0], w.groups, w.pod_state, w.pod_ident, w.nodes, w.n_domains, base[1],
                                 by_domain)
    keys = range(len(cost)) if len(cost) <= 256 else _sample_nodes(label)
    for k in keys:
        d = domain_nodes(w.nodes, w.n_domains, [k]) if by_domain else [k]
        rows, totals = drain_budget_ref(w.lws, w.groups, w.pod_state, w.pod_ident, w.nodes, d, w.flags, base=base)
        check_key(cost[k], rows, totals, (label, k))
