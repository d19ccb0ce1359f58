"""The DS rollout what-if (lwse_resident_ds_rollout_whatif) on a linked world with C4-sized DS tables: 50 000
DisaggregatedSets of 2 roles (1-3 old revisions, tests/ds_drain_ref.py's ds_drain_world, built as
profiles/microbench/ds_drain.py builds it) whose revision-role rows link to child LeaderWorkerSets:

  - the call time (wall clock around a call that returns once the answer is in host memory) and the device time
    (CUDA events on the what-if stream, LWSE_WHATIF_TIMING=1; they include the host synchronisation that sizes
    the gathered tables) of one proposal, of a template bump of every DS with and without the trajectory, and of
    a grid of 16 rollout settings x 1 000 DS;
  - the per-kernel times of a torch.profiler run of its own;
  - lwse_ds_resident_forecast on the same world, for comparison;
  - whether each answer equals the reference (tests/ds_rollout_whatif_ref.py).

The card's name and power limit are read in the same call.

    python profiles/microbench/ds_rollout_whatif.py --out /tmp/ds_rollout_whatif.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

os.environ.setdefault("LWSE_WHATIF_TIMING", "1")  # (read by the engine at its first what-if)

from ds_tick import gpu_info  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from place_whatif import event_device_us, kernel_profile, timed  # noqa: E402

M = R.DS_MAX_ROLES


def grid_query(w, n_ds=1000):
    """16 settings (maxSurge {0, 1, 2, 25%} x maxUnavailable {0, 1, 2, 50%}) with a new template on n_ds DS."""
    grid = [(s, u) for s in (0, 1, 2, 25) for u in (0, 1, 2, 50)]
    props = np.zeros(len(grid) * n_ds, R.DS_PROPOSAL)
    props["ds"] = np.tile(np.arange(n_ds), len(grid))
    props["flags"] = R.DSP_NEW_REVISION | R.DSP_ROLES
    q = R.aligned_empty(len(props) * M, R.DS_ROLE_REC)
    for g, (s, u) in enumerate(grid):
        for d in range(n_ds):
            i, rb, nr = g * n_ds + d, int(w.ds["role_base"][d]), min(int(w.ds["n_roles"][d]), M)
            rows = w.roles[rb: rb + nr].copy()
            spec = (rows["flags"] & R.ROLE_IN_SPEC) != 0
            rows["max_surge"] = np.where(spec, s, rows["max_surge"])
            rows["max_unavailable"] = np.where(spec, u, rows["max_unavailable"])
            pct = (R.ROLE_SURGE_IS_PERCENT if s == 25 else 0) | (R.ROLE_UNAVAIL_IS_PERCENT if u == 50 else 0)
            keep = rows["flags"] & ~np.uint32(R.ROLE_SURGE_IS_PERCENT | R.ROLE_UNAVAIL_IS_PERCENT | R.ROLE_SURGE_INVALID
                                               | R.ROLE_UNAVAIL_INVALID)
            rows["flags"] = np.where(spec, keep | R.ROLE_HAS_ROLLING_CONFIG | pct, rows["flags"])
            q[i * M: i * M + nr] = rows
    return props, q


def measure(eng, w, args):
    from ds_rollout_whatif_ref import ds_rollout_whatif

    eng.upload_nodes(w.nodes, w.n_domains)
    eng.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    eng.resident_tick(eng.make_tick((), w.flags))
    eng.ds_resident_load(w.ds, w.roles, w.revroles)
    eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
    out = {"ds": len(w.ds), "revision_role_rows": len(w.revroles), "lws": len(w.lws)}
    bump = np.zeros(len(w.ds), R.DS_PROPOSAL)
    bump["ds"] = np.arange(len(w.ds))
    bump["flags"] = R.DSP_NEW_REVISION
    summ = eng.resident_ds_rollout_whatif(bump, steps=False)
    need = int(summ["n_steps_needed"])
    # the single proposal: the first DS whose bump starts a rollout with steps, so that the call pays the
    # trajectory pass and its copy as an admission check of a template edit does
    first = int(np.flatnonzero(summ["ds"]["n_steps"] > 0)[0])
    gp, gq = grid_query(w)
    gneed = int(eng.resident_ds_rollout_whatif(gp, gq, steps=False)["n_steps_needed"])
    queries = {"one_proposal": (bump[first: first + 1], None, True, None),
               "bump_every_ds": (bump, None, True, need),
               "bump_every_ds_summaries": (bump, None, False, None),
               "grid_16x1000": (gp, gq, True, gneed)}
    for name, (props, q, steps, cap) in queries.items():
        call = lambda: eng.resident_ds_rollout_whatif(props, q, steps=steps, step_capacity=cap)
        for _ in range(3):
            call()
        got = call()
        ref = ds_rollout_whatif(w.ds, w.roles, w.revroles, w.links, props, q, lws=w.lws, lws_out=w.base[0],
                                steps=steps, step_capacity=cap)
        equal = all(got[k].tobytes() == ref[k].tobytes() for k in ("now", "now_roles", "ds", "roles"))
        equal &= (got["steps"] is None) == (ref["steps"] is None)
        equal &= got["steps"] is None or got["steps"].tobytes() == ref["steps"].tobytes()
        out[name] = {"proposals": len(props), "trajectory_rows": int(got["n_steps_written"]),
                     **({"ds_row": int(props["ds"][0])} if len(props) == 1 else {}),
                     "call": timed(call, args.calls, args.repeats),
                     "device": event_device_us(eng, call, args.calls * args.repeats),
                     "kernels": kernel_profile(call), "equal_to_reference": bool(equal)}
    fneed = int(eng.ds_resident_forecast(steps=False)["n_steps_needed"])
    for name, steps, cap in (("ds_resident_forecast", True, fneed), ("ds_resident_forecast_summaries", False, None)):
        call = lambda: eng.ds_resident_forecast(steps=steps, step_capacity=cap)
        for _ in range(3):
            call()
        out[name] = {"call": timed(call, args.calls, args.repeats), "kernels": kernel_profile(call)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--n-ds", type=int, default=50_000)
    ap.add_argument("--nodes", type=int, default=2048)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from ds_drain_ref import ds_drain_world

    out = {"config": {"calls": args.calls, "repeats": args.repeats, **gpu_info()}}
    eng = Engine(0)
    w = ds_drain_world(n_ds=args.n_ds, n_nodes=args.nodes, seed=23, nodes_per_domain=16, roles=(2,))
    out["C4"] = measure(eng, w, args)
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
