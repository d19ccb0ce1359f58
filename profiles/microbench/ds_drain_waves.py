"""The DS drain waves plan (lwse_resident_ds_drain_waves) on the DS drain's C4-sized world (profiles/microbench/
ds_drain.py: 50 000 DisaggregatedSets of 2 roles linked to child LeaderWorkerSets on 2 048 nodes in 128 domains),
and the same world with every child at maxUnavailable 100 % (every LWS floor 0, so the DS caps decide), with every
node and every domain ordered by drain cost, cap 64, for three constraint masks — LWS floor only, the
default (LWS floor, DS service, DS old service) and all four:

  - the call time (wall clock around a call that returns once the answer is in host memory) and the device time
    from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1);
  - the plan kernel's time per key (torch.profiler);
  - once per scope, the host first-fit over the set forms (one resident_drain_budget and one resident_ds_drain per
    probe), timed once, and whether it gives the same waves.

The card's name and power limit are read in the same call.

    python profiles/microbench/ds_drain_waves.py --out /tmp/ds_drain_waves.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

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

MASKS = {"lws_floor": R.DSW_LWS_FLOOR, "default": R.DSW_LWS_FLOOR | R.DSW_DS_SERVICE | R.DSW_DS_OLD_SERVICE,
         "all": R.DSW_ALL}


def host_first_fit(eng, scope, ids, constraints, limit_s):
    """First-fit over the engine's set forms, one probe per key and open wave; stops after limit_s seconds."""
    t0 = time.perf_counter()
    waves, status = [], []

    def trig(ks):
        b = eng.resident_drain_budget(**{scope: ks})
        d = eng.resident_ds_drain(**{scope: ks})
        return ((R.DSW_LWS_FLOOR if b["n_breached"] else 0) | (R.DSW_DS_SERVICE if d["n_service_lost"] else 0)
                | (R.DSW_DS_OLD_SERVICE if d["n_old_service_lost"] else 0) | (R.DSW_DS_STALL if d["n_stalled"] else 0))

    done = 0
    for k in (int(x) for x in ids):
        if time.perf_counter() - t0 > limit_s:
            break
        done += 1
        if trig([k]) & constraints:
            status.append(-1)
            continue
        for v, W in enumerate(waves):
            if not trig(W + [k]) & constraints:
                W.append(k)
                status.append(v)
                break
        else:
            if len(waves) < 64:
                waves.append([k])
                status.append(len(waves) - 1)
            else:
                status.append(-2)
    return {"seconds": time.perf_counter() - t0, "keys_done": done, "keys": len(ids), "status": status}


def measure(eng, w, args):
    eng.upload_nodes(w.nodes, w.n_domains)
    eng.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    eng.resident_tick(eng.make_tick((), w.flags))
    eng.ds_resident_load(w.ds, w.roles, w.revroles)
    eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
    out = {"ds": len(w.ds), "lws": len(w.lws), "groups": len(w.groups), "nodes": len(w.nodes), "domains": w.n_domains}
    for scope in ("nodes", "domains"):
        cost = eng.resident_drain_budget_cost(scope)
        c = cost
        ids = np.lexsort((np.arange(len(c)), c["groups_restarted"], -c["min_margin"].astype(np.int64)))
        for mname, mask in MASKS.items():
            call = lambda: eng.resident_ds_drain_waves(**{scope: ids}, constraints=mask)
            for _ in range(2):
                call()
            got = call()
            prof = kernel_profile(call)
            plan_us = sum(v for k, v in prof.get("per_call", {}).items() if "plan_capped" in k)
            out[f"{scope}_{mname}"] = {
                "keys": len(ids), "call": timed(call, args.calls, args.repeats),
                "device": event_device_us(eng, call, args.calls * args.repeats), "kernels": prof,
                "plan_us_per_key": (plan_us / len(ids)) if plan_us else None,
                **{k: int(got[k]) for k in R.DS_DRAIN_WAVES_TOTALS},
                "wave0_ds_service_lost": int(got["waves"]["ds_service_lost"][0]) if len(got["waves"]) else 0,
                "wave0_ds_stalled": int(got["waves"]["ds_stalled"][0]) if len(got["waves"]) else 0}
        got = eng.resident_ds_drain_waves(**{scope: ids})
        ff = host_first_fit(eng, scope, ids, MASKS["default"], args.host_limit)
        st = [int(k["wave"]) if k["status"] == R.DRAINW_PLANNED else (-1 if k["status"] == R.DRAINW_BREACHES_ALONE else -2)
              for k in got["keys"][: ff["keys_done"]]]
        out[f"{scope}_host_first_fit_default"] = {"seconds": ff["seconds"], "keys_done": ff["keys_done"],
                                                  "keys": ff["keys"], "same_plan": st == ff["status"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--n-ds", type=int, default=50_000)
    ap.add_argument("--nodes", type=int, default=2048)
    ap.add_argument("--host-limit", type=float, default=60.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from ds_drain_ref import ds_drain_world

    out = {"config": {"calls": args.calls, "repeats": args.repeats, "host_limit_s": args.host_limit, **gpu_info()}}
    eng = Engine(0)
    w = ds_drain_world(n_ds=args.n_ds, n_nodes=args.nodes, seed=23, nodes_per_domain=16, roles=(2,))
    out["C4"] = measure(eng, w, args)
    # the same world with every child at maxUnavailable 100 %: every LWS floor is 0, so the DS caps decide
    from ds_drain_waves_ref import slack_world

    w = slack_world(mu=(100, True), n_ds=args.n_ds, n_nodes=args.nodes, seed=23, nodes_per_domain=16, roles=(2,))
    out["C4_mu100"] = measure(eng, w, args)
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
