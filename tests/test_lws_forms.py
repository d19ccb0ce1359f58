"""The LWS-sweep form worlds (tests/lws_forms_world.py) without a GPU: the launcher's constants are
the ones the builders assume, every world lands on the form its label names, and the oracle's sweep
of every world reaches the cases the GPU tests are meant to cover."""
import os
import re

import numpy as np
import pytest

import lws_forms_world as W
from lws_b200 import records as R

KERNELS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lws_b200", "csrc",
                       "lwse_lws_kernels.cu")
LABELS = list(W.BUILDERS)


def _src() -> str:
    with open(KERNELS) as f:
        return f.read()


def _avg_pods(t) -> int:
    return -(-len(t.pod_state) // len(t.groups))


def _label_number(label: str) -> int:
    return int(label.rsplit("_", 1)[1])


def test_the_builders_use_the_launchers_constants():
    src = _src()

    def const(name):
        m = re.search(rf"constexpr uint32_t {name} = (\d+);", src)
        assert m, name
        return int(m.group(1))

    assert const("kFusedThreads") == W.K_FUSED_THREADS
    assert const("kWinWords") == W.K_WIN_WORDS
    assert const("kPairCap") == W.K_PAIR_CAP
    m = re.search(r"avg_pods <= (\d+) && avg_pods >= (\d+)", src)
    assert m and (int(m.group(2)), int(m.group(1))) == (W.FUSED_MIN_AVG, W.FUSED_MAX_AVG)
    m = re.search(r"avg_pods > (\d+) \? 8 : avg_pods > (\d+) \? 4 : avg_pods > (\d+) \? 2 : 1", src)
    assert m and (int(m.group(3)), int(m.group(2)), int(m.group(1))) == W.GROUP_W_ABOVE
    body = src[src.index("int pick_tile("):]
    body = body[: body.index("\n}\n")]
    m = re.search(r"constexpr uint64_t div = (\d+);", body)
    assert m and int(m.group(1)) == W.LWS_TILE_DIV
    m = re.search(r"while \(w < (\d+) &&", body)
    assert m and int(m.group(1)) == W.LWS_TILE_CAP


def test_the_restated_selection_rule_at_its_thresholds():
    f = W.sweep_form
    assert f(10, 100, 1500) == W.Form(False, True, 1, 1)     # avg 15
    assert f(10, 100, 1600) == W.Form(True, False, None, 1)  # avg 16
    assert f(1, 100, 25600).fused and not f(1, 100, 25601).fused
    assert [f(1, 10, 10 * a).group_w for a in (512, 513, 1024, 1025, 2048, 2049)] == [1, 2, 2, 4, 4, 8]
    assert f(1, 5, 0) == W.Form(False, False, 1, 1)
    assert f(3, 0, 0) == W.Form(False, False, None, 1)
    assert [W.pick_tile(a, 1) for a in (64, 65, 128, 129, 256, 257, 512, 513, 1024, 1025, 5000)] == \
        [1, 2, 2, 4, 4, 8, 8, 16, 16, 32, 32]


def _boundary_groups(t) -> dict:
    base = t.groups["pod_base"].astype(np.int64)
    cnt = t.groups["pod_count"].astype(np.int64)
    full_word = (cnt > 0) & (base % 32 == 0) & ((base + cnt - 1) % 32 == 31)
    mid_single = (cnt == 1) & (base % 32 > 0) & (base % 32 < 31)
    empty_between = np.zeros(len(cnt), bool)
    empty_between[1:-1] = (cnt[1:-1] == 0) & (cnt[:-2] > 0) & (cnt[2:] > 0)
    return {"full_word": int(full_word.sum()), "mid_single": int(mid_single.sum()),
            "empty_between": int(empty_between.sum())}


@pytest.mark.parametrize("label", LABELS)
def test_every_world_lands_on_its_form(label):
    w = W.world(label)
    t = w.tables
    form = W.form_of(t)
    for key, want in W.expected_form(label).items():
        assert getattr(form, key) == want, (label, form)
    if len(t.pod_state):
        assert all(v > 0 for v in _boundary_groups(t).values()), _boundary_groups(t)
    ctas = W.fused_ctas(t.lws, t.groups, t.pod_state) if form.fused else []
    if label in ("fused_lo", "three_w1_below", "three_w1_above") or label.startswith("three_w") and label[-1].isdigit():
        want = {"fused_lo": 16, "three_w1_below": 15, "three_w1_above": 257}.get(label) or _label_number(label)
        assert _avg_pods(t) == want
    if label == "fused_hi":
        assert _avg_pods(t) == 256
        assert all(c.words == W.K_WIN_WORDS and c.windowed for c in ctas)
        assert max(c.max_rel for c in ctas) == 65535 and all(c.pairs <= W.K_PAIR_CAP for c in ctas)
    if label == "fused_direct":
        assert _avg_pods(t) == 256 and ctas[0].windowed
        assert len(ctas) > 1 and all(c.words == W.K_WIN_WORDS + 1 and not c.windowed for c in ctas[1:])
        assert sum(c.pairs for c in ctas[1:]) > 0
    if label == "fused_one_giant":
        assert _avg_pods(t) <= 256 and [c.windowed for c in ctas].count(False) == 1
        assert next(c for c in ctas if not c.windowed).pairs > 0
    if label.startswith("fused_pairs_"):
        assert ctas[0].windowed and ctas[0].pairs == _label_number(label)
    if label == "three_w1_skew":
        assert _avg_pods(t) < 16 and int(t.groups["pod_count"].max()) == 60_000
    if label.startswith("lws_w"):
        assert -(-len(t.groups) // len(t.lws)) == _label_number(label)
    if label == "lws_skew":
        assert form.lws_w == 1 and int(t.lws["group_count"].max()) == 20_000
    if label.startswith("lws_align"):
        assert form.lws_w == (8 if label.endswith("w8") else 1)
    if label == "no_pods":
        assert len(t.pod_state) == 0 and len(t.groups) > 0 and form.kernels == 2
    if label == "no_groups":
        assert len(t.groups) == 0 and len(t.lws) > 0 and form.kernels == 1
    if label == "no_lws":
        assert len(t.lws) == 0 and len(t.groups) > 0 and form.lws_w is None


@pytest.mark.parametrize("label", LABELS)
def test_every_plan_patches_the_same_tables_every_tick(label):
    w = W.world(label)
    t = w.tables
    sizes = {R.TABLE_LWS: len(t.lws), R.TABLE_GROUPS: len(t.groups), R.TABLE_POD_STATE: len(t.pod_state),
             R.TABLE_POD_IDENT: len(t.pod_ident)}
    assert len(w.plan) >= 3
    tables = set(w.plan[0])
    assert tables == {tb for tb, n in sizes.items() if n} or label in ("no_pods", "no_groups")
    for tick in w.plan:
        assert set(tick) == tables
        for tb, (rows, vals) in tick.items():
            assert rows.dtype == np.uint32 and len(rows) == len(vals) > 0
            assert np.all(np.diff(rows.astype(np.int64)) > 0) and int(rows[-1]) < sizes[tb]
        if label == "no_pods":
            assert len(tick[R.TABLE_GROUPS][0]) == len(t.groups)
        if label == "no_groups":
            assert set(tick) == {R.TABLE_LWS} and len(tick[R.TABLE_LWS][0]) == len(t.lws)
    # patches keep the layout: the form of the table is the same after every tick
    m = (t.lws.copy(), t.groups.copy(), t.pod_state.copy(), t.pod_ident.copy())
    for tick in w.plan:
        W.apply_tick(tick, *m)
        for f in ("group_base", "group_count"):
            assert np.array_equal(m[0][f], t.lws[f])
        for f in ("pod_base", "pod_count", "lws_index"):
            assert np.array_equal(m[1][f], t.groups[f])


def _sweep(t, lws=None, groups=None, pst=None, pid=None):
    import oracle

    return oracle.sweep_lws(t.lws if lws is None else lws, t.groups if groups is None else groups,
                            t.pod_state if pst is None else pst, t.pod_ident if pid is None else pid, t.nodes, flags=t.flags)


def test_the_oracle_sweeps_every_world_and_reaches_every_case():
    seen = {"restart_verdict": 0, "update_done": 0, "case": set(), "walk_stops": 0}
    for label in LABELS:
        w = W.world(label)
        t = w.tables
        states = [_sweep(t)]
        m = (t.lws.copy(), t.groups.copy(), t.pod_state.copy(), t.pod_ident.copy())
        for tick in w.plan:
            W.apply_tick(tick, *m)
            states.append(_sweep(t, *m))
        for k, (lo, go, _) in enumerate(states):
            bad_g = (go["flags"] & R.GOUT_BAD_TABLE) != 0
            assert bad_g.all() if w.bad_groups else not bad_g.any(), (label, k)
            assert not ((lo["flags"] & R.LOUT_BAD_TABLE) != 0).any(), (label, k)
            seen["restart_verdict"] += int(((go["flags"] & (R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING)) != 0).sum())
            seen["update_done"] += int(((lo["flags"] & R.LOUT_UPDATE_DONE) != 0).sum())
        lo, go, _ = states[0]
        for i, l in enumerate(t.lws):
            c = W.lws_case(l)
            seen["case"].add(c)
            if c == 5:
                wk = W.case5_walk(l, go)
                seen["walk_stops"] += int(wk["walk"] and 0 <= wk["blocker"] < wk["hi"])
        # the changes of every tick are visible in the results (the GPU tests compare change lists);
        # a table whose every group is BAD_TABLE keeps its results
        assert w.bad_groups or any(a[0].tobytes() != b[0].tobytes() or a[1].tobytes() != b[1].tobytes()
                   for a, b in zip(states, states[1:])), label
    assert seen["restart_verdict"] > 0 and seen["update_done"] > 0 and seen["walk_stops"] > 0
    assert {1, 2, 3, 4, 5} <= seen["case"]


@pytest.mark.parametrize("label", ["lws_align", "lws_align_w8"])
def test_case5_walk_bounds_fall_on_word_edges(label):
    """Every group_base % 8 x group_count % 8 among the Case-5 objects, the walk's bounds and the
    highest bad slot each on flag bytes 8k-1, 8k and 8k+1, and the restated walk giving the oracle's
    partition for every object."""
    w = W.world(label)
    t = w.tables
    lo, go, _ = _sweep(t)
    combos, at = set(), {"rsp": set(), "hi": set(), "max_bad": set()}
    outcomes, more_n, more_rows = set(), 0, 0
    for i, l in enumerate(t.lws):
        if W.lws_case(l) != 5:
            continue
        gb, gc, n = int(l["group_base"]), int(l["group_count"]), int(l["sts_replicas"])
        combos.add((gb % 8, gc % 8))
        wk = W.case5_walk(l, go)
        for k in at:
            at[k].add((gb + wk[k]) % 8)
        outcomes.add("none" if wk["blocker"] < 0 else "at_hi" if wk["blocker"] == wk["hi"] else "below_hi")
        more_n += n > gc
        more_rows += gc > n
        want = max(min(wk["part"], int(l["sts_partition"])), int(l["partition"]))
        assert int(lo["sts_partition"][i]) == want, (i, wk)
    assert combos == {(b, c) for b in range(8) for c in range(8)}
    for k, v in at.items():
        assert {7, 0, 1} <= v, (k, v)
    assert outcomes == {"none", "at_hi", "below_hi"}
    assert more_n > 0 and more_rows > 0
