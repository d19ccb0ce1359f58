"""CPU reference of the LeaderWorkerSet rolling-update forecast (include/lwse.h, "rolling-update forecast").

Every object is replayed at once over private tables: each object gets C group rows, built so that the
C oracle's group pass gives its flag bytes, and every cycle is ``oracle.sweep_lws`` over all of them
(group pass and LWS pass).  An apply rewrites the group rows the way an ideal StatefulSet controller and
kubelet leave them: groups at or past the new replicas are gone, the others run and are ready, those at
or past the partition (and those already at the new revision) carry the object's revision.  The engine
states the same rule on flag bytes; the reference checks that the group pass gives exactly those bytes.
Objects that stop keep their rows (so their results) while the others go on.  Output layout and values
are those of ``Engine.lws_forecast``.
"""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import records as R

_MASK = 0x1F


def _rows_from_bytes(b, owner, lws):
    """Group rows whose group pass gives flag bytes ``b`` (slot owners ``owner`` index ``lws``)."""
    b = b.astype(np.uint32)
    c, cr, cu = (b & R.GOUT_COUNTED) != 0, (b & R.GOUT_COND_READY) != 0, (b & R.GOUT_COND_UPDATED) != 0
    sr, su = (b & R.GOUT_STATE_READY) != 0, (b & R.GOUT_STATE_UPDATED) != 0
    # COUNTED pins the ready / updated predicates to COND_*; the STATE_* bits then need the name match
    assert not np.any(~c & (cr | cu)), "COND_* without COUNTED"
    assert not np.any(c & (sr | su) & ((sr != cr) | (su != cu))), "flag byte no group row gives"
    ready = np.where(c, cr, sr)
    upd = np.where(c, cu, su)
    nm = sr | su
    g = np.zeros(len(b), R.GROUP_REC)
    f = np.zeros(len(b), np.uint32)
    f |= np.where(c, np.uint32(R.GRP_POD_PRESENT | R.GRP_WSTS_FOUND), np.uint32(0))
    f |= np.where(nm, np.uint32(R.GRP_POD_NAME_MATCH | R.GRP_WSTS_LABEL_NAME_MATCH), np.uint32(0))
    f |= np.where(ready, np.uint32(R.GRP_POD_RUNNING | R.GRP_POD_READY | R.GRP_WSTS_REV_SETTLED), np.uint32(0))
    g["flags"] = f
    rev = lws["rev_hash"][owner]
    g["leader_rev_hash"] = np.where(upd, rev, ~rev)
    g["wsts_rev_hash"] = g["leader_rev_hash"]
    w = np.maximum(lws["size"][owner].astype(np.int64) - 1, 0).astype(np.int32)
    g["wsts_spec_replicas"] = w
    g["wsts_avail_replicas"] = w
    g["leader_node"] = R.NONE
    g["lws_index"] = owner
    return g


def _scaled_surge(lws):
    lib = oracle.lib()
    out = np.zeros(len(lws), np.int64)
    for i in range(len(lws)):
        out[i] = lib.lwso_scaled_value(int(lws["max_surge"][i]), int(bool(lws["flags"][i] & R.LWS_SURGE_IS_PERCENT)),
                                       int(lws["replicas"][i]), 1)
    return out


def lws_forecast(lws, group_out, steps=True, step_capacity=None):
    """→ dict as ``Engine.lws_forecast``: lws, steps (or None), n_steps_written, n_steps_needed."""
    n = len(lws)
    fc = np.zeros(n, R.LWS_FORECAST)
    gb, gc = lws["group_base"].astype(np.int64), lws["group_count"].astype(np.int64)
    Rr = lws["replicas"].astype(np.int64)
    bad = gb + gc > len(group_out)
    surge = np.maximum(np.minimum(_scaled_surge(lws), Rr), 0)
    C = np.maximum(gc, np.maximum(np.maximum(lws["sts_replicas"].astype(np.int64), Rr + surge), 0))
    over = ~bad & (C > R.LWS_FORECAST_MAX_SLOTS)
    fc["flags"][bad] = R.LWSF_BAD_TABLE
    fc["flags"][over] = R.LWSF_NOT_FORECAST
    ok = ~bad & ~over
    cnt = np.where(ok, C, 0)
    off = np.cumsum(cnt) - cnt
    owner = np.repeat(np.arange(n), cnt)
    idx = np.arange(len(owner)) - off[owner]

    pl = lws.copy()
    pl["group_base"] = np.where(ok, off, 0)
    pl["group_count"] = cnt
    src = gb[owner] + idx
    inside = idx < gc[owner]
    b0 = np.zeros(len(owner), np.uint32)
    b0[inside] = group_out["flags"][src[inside]] & _MASK
    pg = _rows_from_bytes(b0, owner, pl)
    pst = np.zeros(1, R.POD_STATE)
    pid = np.zeros(1, R.POD_IDENT)

    def sweep():
        lo, go, _ = oracle.sweep_lws(pl, pg, pst, pid)
        return lo, (go["flags"] & _MASK).astype(np.uint32)

    lo, b = sweep()
    assert np.array_equal(b, b0), "the group rows do not give the flag bytes they were built from"
    lf = lo["flags"]
    not_fc = ok & ((lf & (R.LOUT_RUP_ERROR | R.LOUT_STATUS_ERROR | R.LOUT_IRREGULAR)) != 0)
    fc["flags"][not_fc] = R.LWSF_NOT_FORECAST
    run = ok & ~not_fc
    cond = (lf & R.LOUT_COND_MASK) >> R.LOUT_COND_SHIFT
    flags = np.where(run & (cond == R.COND_UPDATE_IN_PROGRESS), R.LWSF_ROLLING, 0).astype(np.uint32)
    peak = np.where((lws["flags"] & R.LWS_STS_EXISTS) != 0, lws["sts_replicas"].astype(np.int64), 0)
    floor = lo["ready_replicas"].astype(np.int64)
    cap = np.minimum(2 * C + 8, R.LWS_FORECAST_MAX_CYCLES)
    n_steps = np.zeros(n, np.int64)
    stopped = np.zeros(n, bool)
    active = run.copy()
    records = []  # per cycle: (objects, their step index, their rows)
    first = True
    while active.any():
        p2, n2 = lo["sts_partition"].astype(np.int64), lo["sts_replicas"].astype(np.int64)
        active &= n2 <= C  # the slots cannot hold n': UNFINISHED
        peak = np.where(active, np.maximum(peak, n2), peak)
        act = active[owner]
        in_n = idx < n2[owner]
        ge_p = idx >= p2[owner]
        cu = (b & R.GOUT_COND_UPDATED) != 0
        keep = in_n & ((b & R.GOUT_COUNTED) != 0) & ((b & R.GOUT_COND_READY) != 0) & ~(ge_p & ~cu)
        kept = np.bincount(owner[act & keep], minlength=n)
        floor = np.where(active, np.minimum(floor, kept), floor)
        if first:
            gained = act & in_n & (((b & R.GOUT_STATE_READY) == 0) | ((b & R.GOUT_COND_READY) == 0))
            flags[np.unique(owner[gained])] |= np.uint32(R.LWSF_WAITING)
            first = False
        nb = np.where(in_n, 0x0D, 0) | np.where(in_n & (ge_p | cu), 0x12, 0)
        changed = np.zeros(n, bool)
        changed[owner[act & (nb != b)]] = True
        nflags = (pl["flags"] | np.uint32(R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID)) & ~np.uint32(R.LWS_UPDATED)
        changed |= ((nflags != pl["flags"]) | (pl["sts_replicas"] != n2) | (pl["sts_partition"] != p2)
                    | (pl["sts_replicas_annotation"] != pl["replicas"]))
        changed &= active
        stopped |= active & ~changed
        active = changed
        if not active.any():
            break
        # the apply: the row takes what the controller writes, the groups what the StatefulSet makes of it
        pl["flags"][active] = nflags[active]
        pl["sts_replicas"][active] = n2[active]
        pl["sts_partition"][active] = p2[active]
        pl["sts_replicas_annotation"][active] = pl["replicas"][active]
        sel = np.nonzero(active[owner])[0]
        pg[sel] = _rows_from_bytes(nb[sel], owner[sel], pl)
        lo, b = sweep()
        assert np.array_equal(b[sel], nb[sel].astype(np.uint32)), "the group pass disagrees with the byte rule"
        objs = np.nonzero(active)[0]
        if steps:
            rows = np.zeros(len(objs), R.LWS_FORECAST_STEP)
            rows["partition"] = lo["sts_partition"][objs]
            rows["sts_replicas"] = lo["sts_replicas"][objs]
            rows["ready_replicas"] = lo["ready_replicas"][objs]
            rows["updated_replicas"] = lo["updated_replicas"][objs]
            records.append((objs, n_steps[objs].copy(), rows))
        n_steps[active] += 1
        active &= n_steps < cap

    fp, fr = lo["sts_partition"].astype(np.int64), lo["sts_replicas"].astype(np.int64)
    flags |= np.where(run & ~stopped, R.LWSF_UNFINISHED, 0).astype(np.uint32)
    flags |= np.where(run & stopped & ((lo["flags"] & R.LOUT_UPDATE_DONE) != 0), R.LWSF_DONE, 0).astype(np.uint32)
    flags |= np.where(run & stopped & (fp > 0) & (fp == lws["partition"]), R.LWSF_HELD, 0).astype(np.uint32)
    fc["flags"][run] = flags[run]
    fc["cycles"][run] = n_steps[run]
    fc["n_steps"][run] = n_steps[run]
    fc["peak_sts_replicas"][run] = peak[run]
    fc["floor_ready"][run] = floor[run]
    fc["final_partition"][run] = fp[run]
    fc["final_replicas"][run] = fr[run]
    rows_of = np.where(run, n_steps, 0)
    base = np.cumsum(rows_of) - rows_of
    fc["step_base"] = np.minimum(base, 0xFFFFFFFF)
    needed = int(rows_of.sum())
    traj, written = None, 0
    if steps:
        capacity = needed if step_capacity is None else int(step_capacity)
        trunc = (rows_of > 0) & (base + rows_of > capacity)
        fc["flags"][trunc] |= np.uint32(R.LWSF_TRUNCATED)
        written = int(rows_of[~trunc].sum())
        traj = np.zeros(written, R.LWS_FORECAST_STEP)
        for objs, sidx, rows in records:
            keep = ~trunc[objs]
            traj[base[objs[keep]] + sidx[keep]] = rows[keep]
    return {"lws": fc, "steps": traj, "n_steps_written": written, "n_steps_needed": needed}


def trajectory(res, i):
    """Object i's trajectory rows as (partition, sts_replicas, ready, updated) tuples."""
    c = res["lws"][i]
    rows = res["steps"][int(c["step_base"]): int(c["step_base"]) + int(c["n_steps"])]
    return [tuple(int(v) for v in r) for r in rows]
