"""CPU reference of the LeaderWorkerSet rollout what-if (include/lwse.h, "rollout what-if").

Proposal i (resident row L_i, proposed row P_i) is answered by the C oracle's sweep of the resident tables
with row L_i replaced by P_i (group_base / group_count kept from the resident row): ``now[i]`` is that
sweep's LWS row L_i, and the forecast is ``lws_forecast_ref.lws_forecast`` of the replaced row over that
sweep's group results.  Proposals for distinct rows interact only through a group row that lies in one
proposal's range and is owned by another's row (a sweep's LWS row reads only its own range, and a group
row reads only its owner), so the proposals are swept in layers, each holding at most one proposal per row
and no two such rows: a query with one proposal per object of disjoint ranges is one sweep.  The
trajectory offsets are then composed over the proposals in query order with the contract of
``lwse_lws_forecast_out``.
"""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import records as R
from lws_forecast_ref import lws_forecast


def foreign_owners(lws, groups, rows):
    """Row → the other rows that own group rows inside its range (ranges outside the table hold none)."""
    out = {}
    for r in np.unique(np.asarray(rows)).tolist():
        b, c = int(lws["group_base"][r]), int(lws["group_count"][r])
        if c and b + c <= len(groups):
            own = groups["lws_index"][b: b + c]
            f = set(np.unique(own[own != r]).tolist())
            if f:
                out[r] = f
    return out


def layers(rows, foreign=None):
    """Proposal indices grouped so that no layer names a row twice, nor a row and an owner of group rows
    inside its range (a foreign-owned row must keep its resident result)."""
    foreign = foreign or {}
    out: list = []  # [proposals, rows, rows whose results a proposal of the layer reads]
    for i, r in enumerate(np.asarray(rows).tolist()):
        f = foreign.get(r, set())
        for lay in out:
            if r not in lay[1] and r not in lay[2] and not (lay[1] & f):
                break
        else:
            lay = [[], set(), set()]
            out.append(lay)
        lay[0].append(i)
        lay[1].add(r)
        lay[2] |= f
    return [lay[0] for lay in out]


def replaced(lws, rows, recs, idx):
    """The resident rows with the proposals ``idx`` put in place (their ranges from the resident rows)."""
    t = lws.copy()
    for i in idx:
        r = int(rows[i])
        rec = recs[i].copy()
        rec["group_base"], rec["group_count"] = lws["group_base"][r], lws["group_count"][r]
        t[r] = rec
    return t


def rollout_whatif(t, rows, recs, steps=True, step_capacity=None, threads=8):
    """→ dict as ``Engine.resident_rollout_whatif`` over the tables ``t`` (an ``encoder.LwsTables`` or
    ``synth`` world: lws, groups, pod_state, pod_ident, nodes, flags)."""
    rows = np.asarray(rows, dtype=np.int64)
    n = len(rows)
    now = np.zeros(n, R.LWS_OUT)
    fc = np.zeros(n, R.LWS_FORECAST)
    traj: list = [None] * n
    for idx in layers(rows, foreign_owners(t.lws, t.groups, rows)):
        lws2 = replaced(t.lws, rows, recs, idx)
        lo, go, _ = oracle.sweep_lws(lws2, t.groups, t.pod_state, t.pod_ident, t.nodes, flags=t.flags, threads=threads)
        sel = rows[idx]
        now[idx] = lo[sel]
        f = lws_forecast(lws2[sel], go)
        for j, i in enumerate(idx):
            fc[i] = f["lws"][j]
            b, k = int(f["lws"][j]["step_base"]), int(f["lws"][j]["n_steps"])
            traj[i] = f["steps"][b: b + k]
    # the trajectory layout over the proposals (lwse_lws_forecast_out)
    counts = fc["n_steps"].astype(np.int64)
    needed = int(counts.sum())
    cap = needed if (steps and step_capacity is None) else int(step_capacity or 0)
    out_steps = np.zeros(cap if steps else 0, R.LWS_FORECAST_STEP)
    base = written = 0
    for i in range(n):
        k = int(counts[i])
        fc[i]["step_base"] = min(base, 0xFFFFFFFF)
        if steps and k:
            if base + k > cap:
                fc[i]["flags"] |= R.LWSF_TRUNCATED
            else:
                out_steps[base: base + k] = traj[i]
                written += k
        base += k
    return {"now": now, "lws": fc, "steps": out_steps[:written] if steps else None, "n_steps_written": written,
            "n_steps_needed": needed}
