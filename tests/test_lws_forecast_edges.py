"""The LWS forecast edge worlds (tests/lws_forecast_edges_world.py) without a GPU: the constants they restate
against the kernel and engine sources, every case on its declared side of its edge (C against the slot
cap, word counts against the tile width, the tile width against the table's average, n' against C, group
ranges, the slot sum, the grid caps), the reference on every world small enough for the CPU with the
property each case exists for, and the closed form of the cycle-cap rollout."""
import os
import re

import numpy as np
import pytest

import lws_forecast_edges_world as W
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lws_b200", "csrc")


def _src(name):
    return open(os.path.join(CSRC, name)).read()


_REFS = {}


def ref_of(label):
    if label not in _REFS:
        w = W.world(label)
        _REFS[label] = lws_forecast(w.lws, w.group_out)
    return _REFS[label]


def side(a, b):
    return "below" if a < b else ("at" if a == b else "above")


# --------------------------------------------------------------------------- #
# the restated constants
# --------------------------------------------------------------------------- #
def test_constants_match_the_sources():
    fk = _src("lwse_lws_forecast_kernels.cu")
    m = re.search(r"constexpr uint32_t kForecastFlagMask = ([^;]*);", fk, re.S).group(1)
    bits = {"LWSE_GOUT_STATE_READY": R.GOUT_STATE_READY, "LWSE_GOUT_STATE_UPDATED": R.GOUT_STATE_UPDATED,
            "LWSE_GOUT_COUNTED": R.GOUT_COUNTED, "LWSE_GOUT_COND_READY": R.GOUT_COND_READY,
            "LWSE_GOUT_COND_UPDATED": R.GOUT_COND_UPDATED}
    names = re.findall(r"LWSE_GOUT_\w+", m)
    assert sorted(names) == sorted(bits) and sum(bits[k] for k in names) == W.FLAG_MASK
    # the slot rounding, in the slot pass and the replay's word count
    assert "(unsigned long long)((C + 7) & ~7ll)" in fk and "(uint32_t)((C + 7) >> 3)" in fk
    assert W.SLOT_ROUND == 8
    # the slot cap, both checks
    assert fk.count("C > (long long)LWSE_LWS_FORECAST_MAX_SLOTS") == 2
    # the cycle cap and the n' > C stop
    cap = re.search(r"const uint32_t cap = \(uint32_t\)min\((\d+) \* C \+ (\d+), \(long long\)LWSE_LWS_FORECAST_MAX_CYCLES\);",
                    fk)
    assert (int(cap.group(1)), int(cap.group(2))) == (W.CAP_MUL, W.CAP_ADD)
    assert "if ((long long)n2 > C) break;" in fk
    # the private-slot copy: group bytes below group_count, zeros past it
    assert "if (idx < gc) w |= " in fk
    # the grids: sm_count * 8 CTAs of 256 threads, slot pass and replay
    assert fk.count(f"cap = (uint32_t)sm_count * {W.GRID_CTAS_PER_SM}u;") == 2
    assert f"lws_forecast_slots_kernel<<<want < cap ? want : cap, {W.BLOCK}, 0, s>>>" in fk
    assert f"lws_forecast_kernel<W, kWrite><<<want < cap ? want : cap, {W.BLOCK}, 0, s>>>" in fk
    assert f"constexpr uint32_t kTilesPerBlock = {W.BLOCK} / W;" in fk
    assert fk.count("__launch_bounds__(256)") == 2
    # the replay's width is the sweep's pick_tile over the group table and the objects
    assert "switch (pick_tile(a.n_groups, a.n_lws))" in fk
    assert [int(x) for x in re.findall(r"case (\d+): launch_tiles<", fk)] == [32, 16, 8, 4, 2]
    lk = _src("lwse_lws_kernels.cu")
    body = re.search(r"int pick_tile\(uint64_t items, uint64_t owners\) \{(.*?)\n\}", lk, re.S).group(1)
    assert int(re.search(r"constexpr uint64_t div = (\d+);", body).group(1)) == W.TILE_DIV
    assert f"while (w < {W.TILE_MAX} && (uint64_t)w < avg) w <<= 1;" in body and "int w = 1;" in body
    assert "if (owners == 0) return 1;" in body
    # the engine's slot-sum check
    eng = _src("lwse_engine.cu")
    assert re.search(r"if \(n_slots >= 0x([0-9a-f]+)ull\) return LWSE_ERR_UNSUPPORTED;", eng).group(1) == \
        f"{W.SLOT_SUM_LIMIT:x}"
    h = open(os.path.join(ROOT, "include", "lwse.h")).read()
    assert f"#define LWSE_LWS_FORECAST_MAX_CYCLES {W.MAX_CYCLES}u" in h
    assert "#define LWSE_LWS_FORECAST_MAX_SLOTS (1u << 20)" in h and W.MAX_SLOTS == 1 << 20


def test_pick_tile_restatement():
    """Worked by hand: one lane up to 64 groups per object on average, then the next power of two of
    avg / 64, at most 32; the average rounds up."""
    for (g, n), w in {(0, 0): 1, (5, 0): 1, (64, 1): 1, (65, 1): 2, (128, 1): 2, (129, 1): 4, (1024, 1): 16,
                      (1025, 1): 32, (2048, 1): 32, (10**9, 1): 32, (128, 2): 1, (129, 2): 2}.items():
        assert W.pick_tile(g, n) == w, (g, n)


# --------------------------------------------------------------------------- #
# every case on its declared side
# --------------------------------------------------------------------------- #
def test_slot_cap_sides():
    w = W.world("slot_cap")
    C = W.slots_of(w.lws, len(w.group_out))
    terms = {}
    for c in w.cases:
        assert C[c.row] == c.value, c.name
        edge = W.MAX_SLOTS
        assert side(C[c.row], edge) == c.side, c.name
        terms.setdefault(c.name.rsplit("_", 1)[0], set()).add(c.side)
        r = w.lws[c.row]
        reps, gc, sts = int(r["replicas"]), int(r["group_count"]), int(r["sts_replicas"])
        s = W.scaled_surge(int(r["max_surge"]), bool(r["flags"] & R.LWS_SURGE_IS_PERCENT), reps)
        term = c.name.rsplit("_", 1)[0]
        # the term the case is for carries C alone
        carried = {"groups": gc, "sts": sts}.get(term, reps + min(s, reps))
        assert carried == C[c.row] and sorted([gc, sts, reps + min(s, reps)])[1] < C[c.row], c.name
        if term == "percent":  # the round-up is what crosses
            assert reps + (int(r["max_surge"]) * reps) // 100 == C[c.row] - 1
        if term == "clamp":
            assert s > reps
    assert all(v == {"below", "at", "above"} for v in terms.values()) and len(terms) == 5


@pytest.mark.parametrize("w", W.WIDTHS)
def test_words_sides(w):
    wd = W.world(f"words_{w}")
    assert W.pick_tile(len(wd.group_out), len(wd.lws)) == w
    C = W.slots_of(wd.lws, len(wd.group_out))
    seen = set()
    for c in wd.cases:
        nw = -(-int(C[c.row]) // 8)
        assert C[c.row] == c.value and side(nw, w) == c.side, c.name
        seen.add((nw - w, int(C[c.row]) % 8))
    assert seen == {(d, m) for d in (-1, 0, 1) for m in range(8) if w + d >= 1}
    surge = [c.row for c in wd.cases if C[c.row] > wd.lws[c.row]["group_count"]]
    assert len(surge) >= 8  # slots past group_count


@pytest.mark.parametrize("avg", W.TILE_AVGS)
def test_tile_sides(avg):
    wd = W.world(f"tile_{avg}")
    G, n = len(wd.group_out), len(wd.lws)
    assert -(-G // n) == avg
    k = -(-avg // 64)
    assert W.pick_tile(G, n) == min(32, 1 << (k - 1).bit_length())
    if avg % 64 == 0 and avg <= 1024:
        assert W.pick_tile(G, n) == avg // 64 and W.pick_tile(G + n, n) == 2 * (avg // 64)
    if avg % 64 == 1:
        assert W.pick_tile(G - n, n) == (avg - 1) // 64  # one group fewer per object: the width below


def test_mixed_tables():
    w1 = W.world("w1_sts")
    assert W.pick_tile(len(w1.group_out), len(w1.lws)) == 1
    C = W.slots_of(w1.lws, len(w1.group_out))
    big = [c for c in w1.cases]
    assert max(C[c.row] for c in big) == W.MAX_SLOTS and -(-W.MAX_SLOTS // 8) == 1 << 17
    assert all(C[c.row] >= 100 * w1.lws[c.row]["group_count"] for c in big)
    w32 = W.world("w32_small")
    assert W.pick_tile(len(w32.group_out), len(w32.lws)) == 32
    C = W.slots_of(w32.lws, len(w32.group_out))
    assert all(0 < C[c.row] <= 8 for c in w32.cases) and len(w32.cases) == len(w32.lws)


def test_ranges_sides():
    w = W.world("ranges")
    G = len(w.group_out)
    for c in w.cases:
        end = int(w.lws[c.row]["group_base"]) + int(w.lws[c.row]["group_count"])
        assert end == c.value and side(end, G) == c.side, c.name
    wrap = w.of("u32_wrap")[0].row
    assert (int(w.lws[wrap]["group_base"]) + int(w.lws[wrap]["group_count"])) % (1 << 32) == 0


def test_slot_sum_sides():
    for refused in (False, True):
        w = W.slot_sum(refused)
        total = int(W.round8(W.slots_of(w.lws, len(w.group_out))).sum())
        c = w.cases[0]
        assert total == c.value and side(total, W.SLOT_SUM_LIMIT) == c.side and len(w.lws) == W.SUM_OBJECTS
        assert W.pick_tile(len(w.group_out), len(w.lws)) == 32
    assert total == 1 << 31


@pytest.mark.parametrize("width", W.WIDTHS)
def test_grid_sides(width):
    w = W.grid(W.H100_SMS, width)
    tiles = W.H100_SMS * W.GRID_CTAS_PER_SM * (W.BLOCK // width)
    assert tiles < len(w.lws) <= tiles + 3
    assert W.pick_tile(len(w.group_out), len(w.lws)) == width
    if width > 1:  # the least average that picks this width
        assert W.pick_tile(len(w.group_out) - len(w.lws), len(w.lws)) == width // 2
    else:  # the slot pass's grid has fewer threads than objects too
        assert len(w.lws) > W.H100_SMS * W.GRID_CTAS_PER_SM * W.BLOCK


# --------------------------------------------------------------------------- #
# the reference on the worlds: the property each case exists for
# --------------------------------------------------------------------------- #
def _flags(res, i):
    return int(res["lws"][i]["flags"])


@pytest.mark.parametrize("label", W.SMALL + ("w1_sts",))
def test_reference_never_reaches_the_cycle_cap(label):
    """The replay stops by itself well before min(2C + 8, MAX_CYCLES) (DESIGN.md: after the first apply
    p' and n' only fall); the only stops without DONE / a quiet apply are n' > C."""
    w = W.world(label)
    res = ref_of(label)
    C = W.slots_of(w.lws, len(w.group_out))
    run = (res["lws"]["flags"] & (R.LWSF_NOT_FORECAST | R.LWSF_BAD_TABLE)) == 0
    st = res["lws"]["n_steps"].astype(np.int64)
    assert (st[run] <= C[run] + 2).all() and (st[run] < W.cycle_cap(C[run])).all()


def test_slot_cap_reference():
    w = W.world("slot_cap")
    res = ref_of("slot_cap")
    for c in w.cases:
        f = _flags(res, c.row)
        if c.side == "above":
            assert f == R.LWSF_NOT_FORECAST and res["lws"][c.row]["n_steps"] == 0, c.name
        else:
            assert not f & (R.LWSF_NOT_FORECAST | R.LWSF_UNFINISHED) and f & R.LWSF_DONE, c.name
            assert res["lws"][c.row]["peak_sts_replicas"] >= min(c.value, int(w.lws[c.row]["sts_replicas"])), c.name


@pytest.mark.parametrize("label", [f"words_{w}" for w in W.WIDTHS] + ["w32_small"])
def test_words_reference(label):
    """n' and p' land on every byte lane of a word (its first slot, its last, and the lanes between), n'
    at C on every surge object, and every rollout ends DONE."""
    w = W.world(label)
    res = ref_of(label)
    st = res["steps"]
    assert set((st["sts_replicas"] % 8).tolist()) == set(range(8))
    assert set((st["partition"] % 8).tolist()) == set(range(8))
    C = W.slots_of(w.lws, len(w.group_out))
    past = 0
    for c in w.cases:
        f = _flags(res, c.row)
        assert f & R.LWSF_DONE and not f & R.LWSF_UNFINISHED, c.name
        rows = st[res["lws"][c.row]["step_base"]: res["lws"][c.row]["step_base"] + res["lws"][c.row]["n_steps"]]
        r = w.lws[c.row]
        if r["max_surge"] < r["replicas"] - r["max_unavailable"]:  # the surge is up while any group is unready
            assert rows["sts_replicas"].max() == C[c.row], c.name
        past += int(rows["sts_replicas"].max() > r["group_count"])
    assert past >= 4  # n' past the object's groups: its surge slots are applied


def test_n_over_c_reference():
    w = W.world("n_over_c")
    res = ref_of("n_over_c")
    C = W.slots_of(w.lws, len(w.group_out))
    for c in w.cases:
        fc = res["lws"][c.row]
        if c.side == "at":
            assert C[c.row] == c.value and fc["n_steps"] > 0 and fc["peak_sts_replicas"] == c.value, c.name
            assert not fc["flags"] & R.LWSF_UNFINISHED
        else:
            assert C[c.row] == c.value - 1
            assert fc["flags"] & R.LWSF_UNFINISHED and fc["n_steps"] == 0 and fc["cycles"] == 0, c.name
            assert fc["peak_sts_replicas"] == C[c.row] < c.value, c.name  # n' = C + 1 is not a peak


def test_ranges_and_degenerate_reference():
    w = W.world("ranges")
    res = ref_of("ranges")
    for c in w.cases:
        bad = _flags(res, c.row) == R.LWSF_BAD_TABLE
        assert bad == (c.side == "above"), c.name
    assert res["lws"][w.of("end_at")[0].row]["n_steps"] > 0
    w = W.world("degenerate")
    res = ref_of("degenerate")
    C = W.slots_of(w.lws, len(w.group_out))
    for c in w.cases:
        assert C[c.row] == c.value, c.name
        assert not _flags(res, c.row) & (R.LWSF_NOT_FORECAST | R.LWSF_BAD_TABLE | R.LWSF_UNFINISHED), c.name
    assert res["lws"][w.of("c0")[0].row]["peak_sts_replicas"] == 0


def test_capacity_reference():
    """At a capacity of exactly an object's step_base + n_steps the object fits and the next object with
    rows does not; one row less truncates it, and no object without rows is ever TRUNCATED."""
    w = W.world("capacity")
    full = ref_of("capacity")
    n = full["lws"]["n_steps"].astype(np.int64)
    base = full["lws"]["step_base"].astype(np.int64)
    with_rows = np.flatnonzero(n > 0)
    assert (np.diff(with_rows) > 1).sum() >= 6  # objects without rows between them
    for i in with_rows[:-1]:
        nxt = with_rows[with_rows > i][0]
        for cap in (base[i] + n[i], base[i] + n[i] - 1):
            res = lws_forecast(w.lws, w.group_out, step_capacity=cap)
            trunc = (res["lws"]["flags"] & R.LWSF_TRUNCATED) != 0
            assert not trunc[n == 0].any()
            assert trunc[i] == (cap < base[i] + n[i]) and trunc[nxt]
            assert res["n_steps_written"] == (cap if cap == base[i] + n[i] else base[i])


# --------------------------------------------------------------------------- #
# the closed form of the cycle-cap rollout
# --------------------------------------------------------------------------- #
CLOSED = [(r, u) for r in (1, 2, 7, 8, 9, 10, 63, 64, 65, 500, 2000) for u in (1, 2, 3, 4)]


def test_closed_form_trajectory():
    b = W.Builder("closed", noise=False)
    for reps, u in CLOSED:
        b.add(reps, reps, reps, mu=u)
    w = b.world()
    res = lws_forecast(w.lws, w.group_out)
    for i, (reps, u) in enumerate(CLOSED):
        fc = res["lws"][i]
        want = W.cap_rows(reps, u)
        assert fc["n_steps"] == len(want) == -(-reps // u) + 1, (reps, u)
        got = res["steps"][fc["step_base"]: fc["step_base"] + fc["n_steps"]]
        assert got.tobytes() == want.tobytes(), (reps, u)
        assert fc["flags"] == R.LWSF_ROLLING | R.LWSF_DONE, (reps, u)
        assert (fc["peak_sts_replicas"], fc["final_partition"], fc["final_replicas"]) == (reps, 0, reps)
        assert fc["floor_ready"] == max(reps - u, 0), (reps, u)


def test_cycle_cap_world_sides():
    w = W.world("cycle_cap")
    cap, below = w.of("cap")[0], w.of("below_cap")[0]
    C = W.slots_of(w.lws, len(w.group_out))
    # the rollout needs R + 1 cycles (closed form); the cap is MAX_CYCLES, not 2C + 8
    assert W.cycle_cap(C[cap.row]) == W.MAX_CYCLES < cap.value == len(W.cap_rows(W.CAP_REPLICAS, 1))
    assert W.cycle_cap(C[below.row]) == W.MAX_CYCLES > below.value == len(W.cap_rows(W.MAX_CYCLES - 2, 1))
