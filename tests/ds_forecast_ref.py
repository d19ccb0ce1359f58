"""CPU reference of the rollout forecast (include/lwse.h, "rollout forecast").

The same cycle rules as the engine, applied to every DS of a table at once with numpy, and
``oracle.sweep_ds`` (the C restatement of the reference's planner and executor) as the sweep of each
cycle.  DS that stop early keep their state while the others go on.  Output layout and values are
those of ``Engine.ds_forecast_host``; the trajectory holds the written rows only.
"""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import records as R

_I32 = np.iinfo(np.int32)


def _clamp(v):
    return np.clip(v, _I32.min, _I32.max).astype(np.int32)


def _counts(rr, row, row_j, row_new, n_j):
    ex = (rr["flags"][row] & R.RR_EXISTS) != 0
    rep = rr["replicas"][row].astype(np.int64)
    old = np.bincount(row_j, weights=np.where(ex & ~row_new, rep, 0), minlength=n_j)
    new = np.bincount(row_j, weights=np.where(ex & row_new, rep, 0), minlength=n_j)
    return np.rint(old).astype(np.int64), np.rint(new).astype(np.int64)


def ds_forecast(ds, roles, revroles, steps=True, step_capacity=None):
    """→ dict as ``Engine.ds_forecast_host``: ds, roles, steps (or None), n_steps_written, n_steps_needed,
    plus ``cycles_run`` (the replay's global cycle count)."""
    n_ds = len(ds)
    fc = np.zeros(n_ds, R.DS_FORECAST)
    fr = np.zeros(len(roles), R.DS_FORECAST_ROLE)
    n = ds["n_roles"].astype(np.int64)
    S = ds["n_spec_roles"].astype(np.int64)
    V = ds["n_old_revs"].astype(np.int64)
    ok = ((n <= R.DS_MAX_ROLES) & (S <= n) & (V <= R.DS_MAX_OLD_REVS)
          & (ds["role_base"].astype(np.int64) + n <= len(roles))
          & (ds["rev_base"].astype(np.int64) + (V + 1) * n <= len(revroles)))
    fc["flags"][~ok] = R.DSF_BAD_TABLE
    # role rows (compact index j) and revision-role rows of the valid DS
    rcnt = np.where(ok, n, 0)
    role_off = np.cumsum(rcnt) - rcnt
    role_d = np.repeat(np.arange(n_ds), rcnt)
    role_i = np.arange(len(role_d)) - role_off[role_d]
    role_idx = ds["role_base"].astype(np.int64)[role_d] + role_i
    n_j = len(role_d)
    cnt = np.where(ok, (V + 1) * n, 0)
    row_d = np.repeat(np.arange(n_ds), cnt)
    k = np.arange(len(row_d)) - (np.cumsum(cnt) - cnt)[row_d]
    row = ds["rev_base"].astype(np.int64)[row_d] + k
    row_i = k % np.maximum(n[row_d], 1)
    row_r = k // np.maximum(n[row_d], 1)
    row_new = row_r == V[row_d]
    row_j = role_off[row_d] + row_i

    rr = revroles.copy()
    dsc = ds.copy()
    target = roles["target_replicas"][role_idx].astype(np.int64)
    # the cycle cap: M = max(any role's target, any role's sum of max(replicas, initial) over existing rows)
    ex0 = (rr["flags"][row] & R.RR_EXISTS) != 0
    mx = np.rint(np.bincount(row_j, weights=np.where(ex0, np.maximum(rr["replicas"][row], rr["initial_replicas"][row])
                                                       .astype(np.int64), 0), minlength=n_j)).astype(np.int64)
    M = np.zeros(n_ds, np.int64)
    np.maximum.at(M, role_d, np.maximum(mx, target))
    cap = np.minimum(2 * M + 12, R.DS_FORECAST_MAX_CYCLES)
    rank = np.zeros(n_ds, np.uint32)
    np.maximum.at(rank, row_d[ex0], rr["flags"][row[ex0]] >> np.uint32(R.RR_TS_SHIFT))

    old, new = _counts(rr, row, row_j, row_new, n_j)
    peak, floor = old + new, old + new
    now = oracle.sweep_ds(dsc, roles, rr)[0]["flags"]
    rolling = ok & ((now & R.DOUT_ROLLING) != 0)
    waiting = rolling & ((now & (R.DOUT_INIT | R.DOUT_STABLE)) == 0)
    active = rolling.copy()
    stopped = np.zeros(n_ds, bool)
    cycles = np.zeros(n_ds, np.int64)
    n_steps = np.zeros(n_ds, np.int64)
    records = []  # per cycle: (role j, step index, old, new) of the DS that made a step
    cycles_run = 0
    while active.any():
        cycles_run += 1
        live = active[row_d]
        sel = row[live & ((rr["flags"][row] & R.RR_EXISTS) != 0)]  # 1. every child ready
        rr["ready_replicas"][sel] = rr["replicas"][sel]
        ds_out, _, rro = oracle.sweep_ds(dsc, roles, rr)  # 2.
        changed = np.zeros(n_ds, bool)
        gone = live & ~row_new & (((ds_out["drained_revs"][row_d] >> row_r.astype(np.uint32)) & 1) == 1)  # 3.
        changed[row_d[gone]] = True
        rr["flags"][row[gone]] &= ~np.uint32(R.RR_EXISTS)
        init = active & ((ds_out["flags"] & R.DOUT_INIT) != 0)  # 4.
        changed |= init
        dsc["flags"][init] |= np.uint32(R.DS_HAS_NEW_REVISION)
        sel = row[live & init[row_d] & ~row_new & ((rr["flags"][row] & R.RR_EXISTS) != 0)]
        rr["initial_replicas"][sel] = rr["replicas"][sel]
        v = rro[row]  # 5.
        f = rr["flags"][row]
        ex = (f & R.RR_EXISTS) != 0
        upd = live & (v >= 0) & ex & ((rr["replicas"][row] != v) | ((f & R.RR_REPLICAS_NIL) != 0))
        make = live & (v >= 0) & ~ex & row_new
        rr["replicas"][row[upd]] = v[upd]
        rr["flags"][row[upd]] &= ~np.uint32(R.RR_REPLICAS_NIL)
        rr["replicas"][row[make]] = v[make]
        rr["initial_replicas"][row[make]] = -1
        rr["ready_replicas"][row[make]] = 0
        rr["flags"][row[make]] = np.uint32(R.RR_EXISTS) | (rank[row_d[make]] << np.uint32(R.RR_TS_SHIFT))
        changed[row_d[upd | make]] = True
        stopped |= active & ~changed
        active &= changed
        cycles[active] += 1
        nold, nnew = _counts(rr, row, row_j, row_new, n_j)
        ra = active[role_d]
        step_d = np.zeros(n_ds, bool)
        step_d[role_d[ra & ((nold != old) | (nnew != new))]] = True
        peak = np.where(ra, np.maximum(peak, old + nnew), peak)
        floor = np.where(ra, np.minimum(floor, nold + new), floor)
        js = np.nonzero(step_d[role_d])[0]
        if steps and len(js):
            records.append((js, n_steps[role_d[js]], nold[js], nnew[js]))
        n_steps[step_d] += 1
        old = np.where(ra, nold, old)
        new = np.where(ra, nnew, new)
        active &= cycles < cap

    left = np.zeros(n_ds, bool)
    left[role_d[(old != 0) | ((role_i < S[role_d]) & (new != target))]] = True
    done = rolling & stopped & ~left
    flags = np.where(rolling, R.DSF_ROLLING, 0) | np.where(waiting, R.DSF_WAITING, 0)
    flags |= np.where(done, R.DSF_DONE, 0) | np.where(rolling & ~done, R.DSF_UNFINISHED, 0)
    fc["flags"][ok] = flags[ok]
    fc["cycles"] = cycles
    fc["n_steps"] = n_steps
    fr["peak_replicas"][role_idx] = _clamp(peak)
    fr["floor_available"][role_idx] = _clamp(floor)
    fr["final_old"][role_idx] = _clamp(old)
    fr["final_new"][role_idx] = _clamp(new)
    rows_of = np.where(ok, n_steps * n, 0)
    base = np.cumsum(rows_of) - rows_of
    fc["step_base"] = np.minimum(base, 0xFFFFFFFF)
    needed = int(rows_of.sum())
    traj, written = None, 0
    if steps:
        capacity = needed if step_capacity is None else int(step_capacity)
        trunc = (rows_of > 0) & (base + rows_of > capacity)
        fc["flags"][trunc] |= np.uint32(R.DSF_TRUNCATED)
        written = int(rows_of[~trunc].sum())
        traj = np.zeros(written, R.DS_ROLE_OUT)
        for js, sidx, o, nw in records:
            d = role_d[js]
            keep = ~trunc[d]
            pos = base[d[keep]] + sidx[keep] * n[d[keep]] + role_i[js[keep]]
            traj["next_old"][pos] = _clamp(o[keep])
            traj["next_new"][pos] = _clamp(nw[keep])
    return {"ds": fc, "roles": fr, "steps": traj, "n_steps_written": written, "n_steps_needed": needed,
            "cycles_run": cycles_run}


def trajectory(res, ds, d):
    """DS d's trajectory as a list of steps, each a list of (old, new) per role."""
    c = res["ds"][d]
    n = int(ds["n_roles"][d])
    rows = res["steps"][int(c["step_base"]): int(c["step_base"]) + int(c["n_steps"]) * n]
    return [[(int(rows[s * n + i]["next_old"]), int(rows[s * n + i]["next_new"])) for i in range(n)]
            for s in range(int(c["n_steps"]))]
