"""The DS planner arithmetic at the limit tables of ``ds_limits_world``, restated on Python ints and
``fractions.Fraction`` (the real-number value of the reference's float64 expressions, planner.go:68-149,
252-352, and intstr.GetScaledValueFromIntOrPercent), against the oracle's float64 form; the generator's
invariants; and what the DS encoders emit at 32 / 33 old revisions and at 10 spec roles + 1 removed."""
import math
from fractions import Fraction

import numpy as np
import pytest

import ds_limits_world as W
import oracle
from lws_b200 import api, ds_informer, encoder
from lws_b200 import records as R

LIMIT_53 = 1 << 53


# --------------------------------------------------------------------------------------------------
# exact restatement; every division a·b / c is recorded as (kind, a·b, c)
# --------------------------------------------------------------------------------------------------
def f_scaled(val, is_percent, total, round_up):
    if not is_percent:
        return val
    q = Fraction(val * total, 100)
    return math.ceil(q) if round_up else math.floor(q)


def f_total_steps(initial, target, ms, mu):
    total = 0
    for i in range(len(initial)):
        b = ms[i] if ms[i] > 0 else max(1, mu[i])
        total = max(total, (max(initial[i], target[i], 0) + b - 1) // b)
    return total


def f_next_new(target, cur_new, T, points=None):
    if T == 0:
        return list(target)
    idx = []
    for t, c in zip(target, cur_new):
        if t == 0:
            idx.append(T)
        else:
            idx.append(int(Fraction(c * T, t)))  # int(): truncation
            points is not None and points.append(("new_idx", c * T, t))
    nxt = min([T] + idx) + 1
    out = []
    for t, c in zip(target, cur_new):
        points is not None and points.append(("new_progress", nxt * t, T))
        out.append(max(min(math.ceil(Fraction(nxt * t, T)), t), c))
    return out


def f_next_old(initial, cur_old, T, points=None):
    if T == 0:
        return [0] * len(initial)
    mx = 0
    for s, c in zip(initial, cur_old):
        if s:
            mx = max(mx, int(Fraction((s - c) * T, s)))
            points is not None and points.append(("old_idx", (s - c) * T, s))
    nxt = mx + 1
    out = []
    for s, c in zip(initial, cur_old):
        points is not None and points.append(("old_progress", nxt * s, T))
        out.append(min(max(0, s - math.floor(Fraction(nxt * s, T))), c))
    return out


def _orphans(nxt, cur_new, initial, target, mu):
    vals = [nxt[i] for i in range(len(nxt)) if initial[i]]
    if not any(v == 0 for v in vals) or all(v == 0 for v in vals):
        return nxt
    if all(not (initial[i] >= target[i]) or cur_new[i] >= target[i] - mu[i] for i in range(len(nxt))):
        return [0] * len(nxt)
    return [1 if nxt[i] == 0 and initial[i] > 0 else nxt[i] for i in range(len(nxt))]


def f_next_step(initial, cur_old, cur_new, target, ms, mu, points=None):
    """planner.go:320-352 ComputeNextStep → (past, new) or None."""
    n = len(initial)
    if all(cur_old[i] == 0 and cur_new[i] >= target[i] for i in range(n)):
        return None
    T = f_total_steps(initial, target, ms, mu)
    if T == 0:
        return None
    exp = [min(initial[i], cur_old[i]) for i in range(n)]
    if any(cur_old[i] > exp[i] for i in range(n)):
        return exp, list(cur_new)
    if all(cur_new[i] >= target[i] for i in range(n)):
        return [0] * n, list(cur_new)
    nn = f_next_new(target, cur_new, T, points)
    min_old = [max(0, target[i] - mu[i] - cur_new[i]) if initial[i] >= target[i] else 0 for i in range(n)]
    if any(nn[i] > cur_new[i] for i in range(n)) and all(
            target[i] == 0 or cur_old[i] + nn[i] <= target[i] + ms[i] for i in range(n)):
        return list(cur_old), nn
    no = [max(v, m) for v, m in zip(f_next_old(initial, cur_old, T, points), min_old)]
    no = _orphans(no, cur_new, initial, target, mu)
    if any(no[i] < cur_old[i] for i in range(n)):
        return no, list(cur_new)
    dr = []
    for i in range(n):
        v = max(0, min(cur_old[i], target[i] + ms[i] - nn[i]))
        if initial[i] >= target[i]:
            v = max(v, max(0, target[i] - mu[i] - nn[i]))
        dr.append(v)
    if any(dr[i] < cur_old[i] for i in range(n)):
        return _orphans(dr, nn, initial, target, mu), nn
    return None


def planner_state(ds, roles, rr, d):
    """buildPlannerState (executor.go:199-260) of DS d, restated over its rows, and whether the sweep
    calls ComputeNextStep for it (rolling, a new revision, stable)."""
    h = ds[d]
    n, S, V = int(h["n_roles"]), int(h["n_spec_roles"]), int(h["n_old_revs"])
    ro = roles[int(h["role_base"]): int(h["role_base"]) + n]
    x = rr[int(h["rev_base"]): int(h["rev_base"]) + (V + 1) * n]
    ex = (x["flags"] & R.RR_EXISTS) != 0
    ini, cold, cnew, tgt, ms, mu = [0] * n, [0] * n, [0] * n, [0] * n, [1] * n, [0] * n
    for i in range(n):
        for r in range(V):
            k = r * n + i
            if ex[k]:
                cold[i] += int(x["replicas"][k])
                ini[i] += int(x["initial_replicas"][k]) if x["initial_replicas"][k] >= 0 else int(x["replicas"][k])
        f = int(ro["flags"][i])
        if f & R.ROLE_IN_SPEC:
            if ex[V * n + i]:
                cnew[i] = int(x["replicas"][V * n + i])
            tgt[i] = int(ro["target_replicas"][i])
            if f & R.ROLE_HAS_ROLLING_CONFIG:
                s = 0 if f & R.ROLE_SURGE_INVALID else f_scaled(int(ro["max_surge"][i]), f & R.ROLE_SURGE_IS_PERCENT, tgt[i], True)
                u = 0 if f & R.ROLE_UNAVAIL_INVALID else f_scaled(int(ro["max_unavailable"][i]), f & R.ROLE_UNAVAIL_IS_PERCENT, tgt[i], False)
                if u > 0:
                    ms[i], mu[i] = s, u
                elif s > 0:
                    ms[i] = s
    total_old = sum(int(x["replicas"][r * n + i]) for r in range(V) for i in range(S) if ex[r * n + i])
    stable = all(ex[V * n + i] and x["replicas"][V * n + i] == x["ready_replicas"][V * n + i] for i in range(S))
    reaches = V > 0 and total_old > 0 and bool(h["flags"] & R.DS_HAS_NEW_REVISION) and stable
    return (ini, cold, cnew, tgt, ms, mu), reaches


def _one(ds, roles, rr, d):
    """DS d alone in a table of its own (bases rebased)."""
    h = ds[d: d + 1].copy()
    n, V = int(h["n_roles"][0]), int(h["n_old_revs"][0])
    rb, vb = int(h["role_base"][0]), int(h["rev_base"][0])
    h["role_base"], h["rev_base"] = 0, 0
    return h, roles[rb: rb + n].copy(), rr[vb: vb + (V + 1) * n].copy()


def _boundary(points):
    """Kinds with an exact quotient (a·b ≡ 0 mod c, a·b > 0) and kinds one away (a·b ≡ ±1 mod c, c > 2)."""
    exact = {k for k, ab, c in points if ab > 0 and ab % c == 0 and c > 1}
    near = {k for k, ab, c in points if c > 2 and ab % c in (1, c - 1)}
    return exact, near


# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", sorted(W.FAMILIES))
def test_float64_planner_equals_exact_restatement(family):
    """Every DS that reaches ComputeNextStep: the Fraction restatement, the oracle's float64 planner and
    helpers, and the oracle's sweep of the DS alone give the same step; every product stays < 2^53."""
    ds, roles, rr = W.FAMILIES[family]()
    reached = 0
    all_points = []
    for d in range(len(ds)):
        st, reaches = planner_state(ds, roles, rr, d)
        if not reaches:
            continue
        reached += 1
        ini, cold, cnew, tgt, ms, mu = st
        points = []
        want = f_next_step(ini, cold, cnew, tgt, ms, mu, points)
        all_points += points
        assert all(ab < LIMIT_53 for _, ab, _ in points), (family, d)
        got = oracle.ds_compute_next_step(ini, cold, cnew, tgt, ms, mu)
        assert got == (None if want is None else (list(want[0]), list(want[1]))), (family, d)
        T = f_total_steps(ini, tgt, ms, mu)
        assert oracle.ds_total_steps(ini, tgt, ms, mu) == T
        assert oracle.ds_next_new(tgt, cnew, T) == f_next_new(tgt, cnew, T), (family, d)
        assert oracle.ds_next_old(ini, cold, T) == f_next_old(ini, cold, T), (family, d)
        o = oracle.sweep_ds(*_one(ds, roles, rr, d))
        if want is None:
            assert o[0]["flags"][0] & R.DOUT_COMPLETE
        else:
            assert o[0]["flags"][0] & R.DOUT_STEP
            assert o[1]["next_old"].tolist() == list(want[0]) and o[1]["next_new"].tolist() == list(want[1])
    assert reached >= 10
    if family == "rounding":  # the divisions the generator aims at land on and next to integers
        exact, near = _boundary(all_points)
        for kind in ("new_idx", "new_progress", "old_progress"):
            assert kind in exact and kind in near, (kind, exact, near)


def test_percent_scaling_equals_exact():
    ds, roles, rr = W.rounding()
    lib = oracle.lib()
    n = 0
    for t, s, u in zip(roles["target_replicas"], roles["max_surge"], roles["max_unavailable"]):
        t, s, u = int(t), int(s), int(u)
        assert s * t < LIMIT_53 and u * t < LIMIT_53
        assert lib.lwso_scaled_value(s, 1, t, 1) == f_scaled(s, True, t, True)
        assert lib.lwso_scaled_value(u, 1, t, 0) == f_scaled(u, True, t, False)
        assert W.planner_config(t, s, u)[0] in (f_scaled(s, True, t, True), 1)
        n += (s * t) % 100 in (1, 99)
    assert n > 0  # some surge lands one away from a whole replica
    assert set(roles["max_surge"]) == set(W.PERCENTS) and set(roles["max_unavailable"]) == set(W.PERCENTS)
    assert roles["target_replicas"].max() >= 99_999


def newest_first(ds, rr, d):
    """Old revisions of DS d newest-first by the max creation stamp over their existing rows; equal
    stamps keep row order (sortByNewestTimestamp, executor.go:283-302)."""
    h = ds[d]
    n, V, vb = int(h["n_roles"]), int(h["n_old_revs"]), int(h["rev_base"])
    f = rr["flags"][vb: vb + V * n].reshape(V, n)
    ts = np.where(f & R.RR_EXISTS, f >> R.RR_TS_SHIFT, 0).max(axis=1) if V else np.zeros(0)
    return sorted(range(V), key=lambda r: -int(ts[r]))


def zeroed_revisions(ds, rr, rro, d):
    """Old revisions of DS d that held replicas and that the sweep set to 0 on every existing row."""
    h = ds[d]
    n, V, vb = int(h["n_roles"]), int(h["n_old_revs"]), int(h["rev_base"])
    x = rr[vb: vb + V * n].reshape(V, n)
    o = rro[vb: vb + V * n].reshape(V, n)
    ex = (x["flags"] & R.RR_EXISTS) != 0
    return [r for r in range(V) if ex[r].any() and (x["replicas"][r][ex[r]] > 0).any() and (o[r][ex[r]] == 0).all()]


def test_drain_follows_the_newest_stamp_not_row_order():
    ds, roles, rr = W.stamp_orders()
    out = oracle.sweep_ds(ds, roles, rr)
    drains = not_last = 0
    for d in range(len(ds)):
        if not out[0]["flags"][d] & R.DOUT_STEP or roles["target_replicas"][int(ds["role_base"][d])] != ds["n_old_revs"][d]:
            continue
        order = newest_first(ds, rr, d)
        z = zeroed_revisions(ds, rr, out[2], d)
        assert order[0] in z, d
        drains += 1
        not_last += order[0] != int(ds["n_old_revs"][d]) - 1
    assert drains >= 40 and not_last >= 20


def test_generator_invariants():
    fam = {k: f() for k, f in W.FAMILIES.items()}
    ds, roles, rr = fam["v_sweep"]
    combos = {(int(v), int(n)) for v, n in zip(ds["n_old_revs"], ds["n_roles"])}
    assert {(V, n) for V in (0, 1, 2, 31, 32) for n in (2, 3, 10)} <= combos
    assert ((ds["n_roles"] == 10) & (ds["n_spec_roles"] == 9)).any()
    assert ((ds["n_roles"] == 3) & (ds["n_spec_roles"] == 2)).any()
    for name, (ds, roles, rr) in fam.items():  # contiguous ranges, every DS inside the format
        n = ds["n_roles"].astype(np.int64)
        assert np.array_equal(ds["role_base"], np.concatenate([[0], np.cumsum(n)[:-1]]))
        nrr = (ds["n_old_revs"].astype(np.int64) + 1) * n
        assert np.array_equal(ds["rev_base"], np.concatenate([[0], np.cumsum(nrr)[:-1]]))
        assert len(rr) == nrr.sum() and len(roles) == n.sum()
        assert (n <= R.DS_MAX_ROLES).all() and (ds["n_old_revs"] <= R.DS_MAX_OLD_REVS).all()
        assert (ds["n_spec_roles"] <= n).all()
        out = oracle.sweep_ds(ds, roles, rr)[0]
        assert not (out["flags"] & R.DOUT_BAD_TABLE).any(), name
    out = oracle.sweep_ds(*fam["bit31"])[0]
    assert ((out["drained_revs"] >> 31) & 1).sum() >= 6 and ((out["ready_revs"] >> 31) & 1).sum() >= 6
    assert (((out["drained_revs"] >> 31) & (out["ready_revs"] >> 31)) & 1).any()
    # stamp orders: the extremes of the 30-bit field, ties at the newest, rows that do not exist
    ds, roles, rr = fam["stamps"]
    ts = rr["flags"] >> R.RR_TS_SHIFT
    ex = (rr["flags"] & R.RR_EXISTS) != 0
    assert (ts[ex] == 0).any() and (ts[ex] == W.TS_MAX).any() and (ts[~ex] == W.TS_MAX).any()
    orders = [newest_first(ds, rr, d) for d in range(len(ds))]
    assert sum(o != list(range(len(o)))[::-1] for o in orders) > len(ds) // 2
    assert sum(o == list(range(len(o))) and len(o) > 1 for o in orders) > 0  # reversed / equal stamps
    # the mixed table: narrow and limit DS alternate
    ds, roles, rr = W.mixed()
    big = ds["n_old_revs"] > 3
    assert big[1::2].any() and not big[0::2].any()


def _child(role, rev, ts, replicas=2):
    return api.ChildLWS(role, rev, replicas, replicas, float(ts))


def _ds_item(name, n_spec, n_old, extra_role=None, t0=0.0):
    roles = [api.DisaggregatedRoleSpec(f"r{i}", 2) for i in range(n_spec)]
    kids = []
    for v in range(n_old):
        for i in range(n_spec):
            kids.append(_child(f"r{i}", f"old{v}", t0 + v))
        if extra_role and v == 0:
            kids.append(_child(extra_role, f"old{v}", t0 + v))
    kids += [_child(f"r{i}", "new", t0 + n_old) for i in range(n_spec)]
    return encoder.DsItem(api.DisaggregatedSet(name, roles=roles), "new", kids)


def test_encoder_at_and_past_the_limits():
    """encode_ds emits 32 old revisions as a valid DS, and 33 old revisions or 10 spec roles + 1 removed
    role as rows the sweep reports BAD_TABLE; the neighbours' rows and results do not change."""
    a, c = _ds_item("a", 2, 2), _ds_item("c", 3, 1)
    base = encoder.encode_ds([a, c])
    ob = oracle.sweep_ds(base.ds, base.roles, base.revroles)

    def check(mid, V, n, S):
        t = encoder.encode_ds([a, mid, c])
        assert (int(t.ds["n_old_revs"][1]), int(t.ds["n_roles"][1]), int(t.ds["n_spec_roles"][1])) == (V, n, S)
        assert len(t.old_revisions[1]) == V and t.role_names[1][:S] == [f"r{i}" for i in range(S)]
        assert int(t.ds["rev_base"][2]) - int(t.ds["rev_base"][1]) == (V + 1) * n
        # the neighbours' rows: the same, with c's ranges moved behind the middle DS
        for d_new, d_old in ((0, 0), (2, 1)):
            h0, h1 = t.ds[d_new].copy(), base.ds[d_old].copy()
            m, rb0, rb1 = int(h0["n_roles"]), int(h0["role_base"]), int(h1["role_base"])
            assert t.roles[rb0: rb0 + m].tobytes() == base.roles[rb1: rb1 + m].tobytes()
            vb0, vb1 = int(h0["rev_base"]), int(h1["rev_base"])
            k = (int(h0["n_old_revs"]) + 1) * int(h0["n_roles"])
            assert t.revroles[vb0: vb0 + k].tobytes() == base.revroles[vb1: vb1 + k].tobytes()
            h0["role_base"] = h1["role_base"] = h0["rev_base"] = h1["rev_base"] = 0
            assert h0.tobytes() == h1.tobytes()
        o = oracle.sweep_ds(t.ds, t.roles, t.revroles)
        for d_new, d_old in ((0, 0), (2, 1)):
            assert o[0][d_new].tobytes() == ob[0][d_old].tobytes()
        return t, o

    t, o = check(_ds_item("b", 2, 32, t0=1000.0), 32, 2, 2)
    assert not o[0]["flags"][1] & R.DOUT_BAD_TABLE and o[0]["flags"][1] & R.DOUT_ROLLING
    t, o = check(_ds_item("b", 2, 33, t0=1000.0), 33, 2, 2)
    assert o[0]["flags"][1] == R.DOUT_BAD_TABLE
    t, o = check(_ds_item("b", 10, 1, extra_role="gone", t0=1000.0), 1, 11, 10)
    assert t.role_names[1][-1] == "gone" and o[0]["flags"][1] == R.DOUT_BAD_TABLE
    t, o = check(_ds_item("b", 9, 1, extra_role="gone", t0=1000.0), 1, 10, 9)
    assert not o[0]["flags"][1] & R.DOUT_BAD_TABLE


def test_incremental_encoder_grows_a_ds_past_the_limits():
    """DsIncrementalEncoder: a DS that goes from 32 to 33 old revisions, and one that gains an 11th role
    (10 spec + 1 removed), patch only their own rows; the sweep reports them BAD_TABLE and every
    neighbour keeps its rows and results."""
    items = [_ds_item("a", 2, 2), _ds_item("b", 2, 32, t0=1000.0), _ds_item("c", 10, 1, t0=2000.0), _ds_item("e", 3, 1)]
    enc = ds_informer.DsIncrementalEncoder(items, spare=1.0)
    before = [x.copy() for x in enc.tables()]
    ob = oracle.sweep_ds(*before)
    rows = {k: enc.ds_row("default", k) for k in "abce"}
    assert ob[0]["flags"][rows["b"]] & R.DOUT_ROLLING and not ob[0]["flags"][rows["b"]] & R.DOUT_BAD_TABLE
    enc.child_event("ADDED", "default", "b", _child("r0", "old32", 1032.0))
    enc.child_event("ADDED", "default", "c", _child("gone", "old0", 1999.0))
    p = enc.flush()
    assert not enc.needs_reload
    assert int(enc.ds["n_old_revs"][rows["b"]]) == 33 and len(enc.old_revisions(rows["b"])) == 33
    assert (int(enc.ds["n_roles"][rows["c"]]), int(enc.ds["n_spec_roles"][rows["c"]])) == (11, 10)
    assert enc.role_names(rows["c"])[-1] == "gone"
    after = enc.tables()
    o = oracle.sweep_ds(*after)
    assert o[0]["flags"][rows["b"]] == R.DOUT_BAD_TABLE and o[0]["flags"][rows["c"]] == R.DOUT_BAD_TABLE
    own = {R.TABLE_DS: set(), R.TABLE_DS_ROLES: set(), R.TABLE_DS_REVROLES: set()}
    for k in "ae":
        d = rows[k]
        h = after[0][d]
        assert h.tobytes() == before[0][d].tobytes()
        rb, n, vb = int(h["role_base"]), int(h["n_roles"]), int(h["rev_base"])
        k2 = (int(h["n_old_revs"]) + 1) * n
        assert after[1][rb: rb + n].tobytes() == before[1][rb: rb + n].tobytes()
        assert after[2][vb: vb + k2].tobytes() == before[2][vb: vb + k2].tobytes()
        assert o[0][d].tobytes() == ob[0][d].tobytes()
        assert o[1][rb: rb + n].tobytes() == ob[1][rb: rb + n].tobytes()
        assert o[2][vb: vb + k2].tobytes() == ob[2][vb: vb + k2].tobytes()
        own[R.TABLE_DS].add(d)
        own[R.TABLE_DS_ROLES].update(range(rb, rb + n))
        own[R.TABLE_DS_REVROLES].update(range(vb, vb + k2))
    for seg in p.segments:  # no patch touches a neighbour's rows
        table, rws = seg[0], seg[1]
        rws = range(rws, rws + len(seg[2])) if len(seg) == 4 else [int(r) for r in rws]
        assert not own.get(table, set()) & set(rws), table
