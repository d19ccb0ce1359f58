"""CPU reference of the DS rollout what-if (include/lwse.h, "DS rollout what-if").

``proposed`` builds every proposal's rows P_i as the definition states them, proposal i at DS row i with its role
rows at DS_MAX_ROLES * i and its revision-role and link rows after those of the proposals before it.  ``now`` is
``oracle.sweep_ds`` over those rows as the linked DS tick reads them (``ds_link_world.linked_revroles``), and the
forecast is ``ds_forecast_ref.ds_forecast`` over the same rows."""
from __future__ import annotations

import numpy as np

import oracle
from ds_forecast_ref import ds_forecast
from ds_link_world import linked_revroles, none_links
from lws_b200 import records as R

M = R.DS_MAX_ROLES


def _aligned(chunks, dtype):
    out = R.aligned_empty(sum(len(c) for c in chunks), dtype)
    if len(out):
        out[:] = np.concatenate(chunks)
    return out


def proposed(ds, roles, revroles, links, proposals, q_roles=None):
    """→ (ds, roles, revroles, links, bad): the proposed tables, and which proposals are BAD_TABLE.  A BAD
    proposal's DS row keeps the resident fields with rev_base = NONE, beyond every table, so that the sweep and
    the forecast report it BAD_TABLE; it has no rows."""
    n = len(proposals)
    P = R.aligned_empty(n, R.DS_REC)
    Pr = R.aligned_empty(n * M, R.DS_ROLE_REC)
    rr, lk = [], []
    bad = np.zeros(n, bool)
    off = 0
    for i, p in enumerate(proposals):
        d = ds[int(p["ds"])].copy()
        nr, S, V = int(d["n_roles"]), int(d["n_spec_roles"]), int(d["n_old_revs"])
        rb, vb, f = int(d["role_base"]), int(d["rev_base"]), int(d["flags"])
        ok = (nr <= M and S <= nr and V <= R.DS_MAX_OLD_REVS and rb + nr <= len(roles)
              and vb + (V + 1) * nr <= len(revroles))
        retire = ok and bool(p["flags"] & R.DSP_NEW_REVISION) and bool(f & R.DS_HAS_NEW_REVISION)
        d["role_base"] = i * M
        if not ok or V + retire > R.DS_MAX_OLD_REVS:
            bad[i] = True
            d["rev_base"] = R.NONE
            P[i] = d
            continue
        Pr[i * M: i * M + nr] = q_roles[i * M: i * M + nr] if p["flags"] & R.DSP_ROLES else roles[rb: rb + nr]
        rows, lrows = [revroles[vb: vb + (V + 1) * nr]], [links[vb: vb + (V + 1) * nr]]
        if retire:  # the target revision becomes old revision V; the new revision has no child yet
            absent = R.aligned_empty(nr, R.DS_REVROLE_REC)
            absent["initial_replicas"] = -1
            rows.append(absent)
            lrows.append(none_links(nr))
            d["n_old_revs"] = V + 1
            d["flags"] = f & ~R.DS_HAS_NEW_REVISION
        d["rev_base"] = off
        off += (V + 1 + retire) * nr
        P[i] = d
        rr += rows
        lk += lrows
    return P, Pr, _aligned(rr, R.DS_REVROLE_REC), _aligned(lk, R.DS_LINK), bad


def ds_rollout_whatif(ds, roles, revroles, links, proposals, q_roles=None, lws=None, lws_out=None, steps=True,
                      step_capacity=None):
    """→ dict as ``Engine.resident_ds_rollout_whatif``.  ``links``: the resident link table (None: no link rows);
    ``lws`` / ``lws_out``: the resident LWS table and its results when the engine's DS rows are linked and its LWS
    rows swept, else None (every row uses its own ready count)."""
    if links is None:
        links = none_links(len(revroles))
    P, Pr, Prr, Pl, bad = proposed(ds, roles, revroles, links, proposals, q_roles)
    read, _, _ = linked_revroles(Prr, Pl, lws, lws_out)
    now, now_roles, _ = oracle.sweep_ds(P, Pr, read)
    out = ds_forecast(P, Pr, Prr, steps=steps, step_capacity=step_capacity)
    del out["cycles_run"]
    out["now"], out["now_roles"], out["bad"] = now, now_roles, bad
    return out


def trajectory_of(res, i, n):
    """Proposal i's trajectory (n roles) as a list of steps, each a list of (old, new) per role."""
    c = res["ds"][i]
    rows = res["steps"][int(c["step_base"]): int(c["step_base"]) + int(c["n_steps"]) * n]
    return [[(int(rows[s * n + j]["next_old"]), int(rows[s * n + j]["next_new"])) for j in range(n)]
            for s in range(int(c["n_steps"]))]
