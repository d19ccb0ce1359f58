"""The rollout what-if of LeaderWorkerSets (lwse_resident_rollout_whatif) at C3 and C5, next to the
resident forecast (lwse_resident_forecast) of the same tables in the same process:

  - one template-edit proposal (the latency of an interactive query);
  - one template-edit proposal per object, with the trajectory rows and with summaries only;
  - 16 rollout settings ((maxUnavailable, maxSurge) in 0..3, each with a template edit) for each of the
    first 1 000 objects: 16 000 proposals;
  - the wall clock around a call that returns once the answer is in host memory (median and spread over
    windows), and device time per kernel from torch.profiler CUDA activity records of a run of its own;
  - whether the engine's bytes equal the CPU reference (tests/rollout_whatif_ref.py).

The card's name and power limit are read in the same call.

    python profiles/microbench/rollout_whatif.py --out /tmp/rollout_whatif.json
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

from ds_tick import gpu_info  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200 import synth  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from lws_forecast import timed  # noqa: E402


def template_edit(lws, rows):
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = lws[rows]
    recs["rev_hash"] ^= np.uint64(0x5DEECE66D)
    recs["flags"] |= np.uint32(R.LWS_UPDATED)
    return recs


def settings_grid(lws, n_objects):
    rows = np.repeat(np.arange(n_objects, dtype=np.uint32), 16)
    recs = template_edit(lws, rows)
    mu, ms = np.tile(np.repeat(np.arange(4), 4), n_objects), np.tile(np.tile(np.arange(4), 4), n_objects)
    recs["max_unavailable"], recs["max_surge"] = mu, ms
    recs["flags"] &= ~np.uint32(R.LWS_SURGE_IS_PERCENT | R.LWS_UNAVAIL_IS_PERCENT | R.LWS_INTSTR_INVALID)
    return rows, recs


def device_us(eng, call, n_prof=10):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            call()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            n = ev.name
            key = ("gather" if "rollout_whatif_gather" in n else "restore" if "rollout_whatif_restore" in n else
                   "layout_scan" if "WhatifLayoutOp" in n else
                   "forecast_kernel<write>" if "lws_forecast_kernel" in n and "true>" in n else
                   "forecast_kernel<summary>" if "lws_forecast_kernel" in n else
                   "slots" if "forecast_slots_kernel" in n else
                   "slot_scan" if "scan_" in n and "SlotLayoutOp" in n else
                   "step_scan" if "scan_" in n and "StepLayoutOp" in n else
                   "pod_scan" if "pod_scan" in n else "group_pass" if "group_" in n else
                   "lws_pass" if "lws_sweep_kernel" in n else "memcpy" if "emcpy" in n else
                   "memset" if "emset" in n else n[:40])
            per[key] = per.get(key, 0.0) + ev.device_time_total
    per = {k: v / n_prof for k, v in per.items()}
    return {"per_call": per, "total": float(sum(per.values()))}


def one_config(eng, name, calls, repeats):
    from rollout_whatif_ref import rollout_whatif

    t = synth.make(name)
    out = {"lws": len(t.lws), "groups": len(t.groups), "pods": len(t.pod_state)}
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_tick(eng.make_tick((), t.flags))
    all_rows = np.arange(len(t.lws), dtype=np.uint32)
    queries = {
        "one_proposal": (all_rows[:1], template_edit(t.lws, all_rows[:1]), True),
        "fleet_with_trajectory": (all_rows, template_edit(t.lws, all_rows), True),
        "fleet_summaries_only": (all_rows, template_edit(t.lws, all_rows), False),
        "settings_16x1000": (*settings_grid(t.lws, min(1000, len(t.lws))), True),
    }
    fc_cap = int(eng.resident_forecast(steps=False)["n_steps_needed"])
    base = {
        "forecast_with_trajectory": lambda: eng.resident_forecast(steps=True, step_capacity=fc_cap),
        "forecast_summaries_only": lambda: eng.resident_forecast(steps=False),
    }
    for key, (rows, recs, steps) in queries.items():
        first = eng.resident_rollout_whatif(rows, recs, steps=steps)
        cap = int(first["n_steps_needed"]) if steps else None
        call = (lambda rows=rows, recs=recs, steps=steps, cap=cap:
                eng.resident_rollout_whatif(rows, recs, steps=steps, step_capacity=cap))
        for _ in range(3):
            call()
        n = calls if len(rows) > 1 else calls * 10
        ref = rollout_whatif(t, rows, recs, steps=steps)
        equal = (ref["now"].tobytes() == first["now"].tobytes() and ref["lws"].tobytes() == first["lws"].tobytes()
                 and (not steps or ref["steps"].tobytes() == first["steps"].tobytes()))
        out[key] = {"proposals": len(rows), "trajectory_rows": int(first["n_steps_needed"]),
                    "call": timed(call, n, repeats), "device_us": device_us(eng, call), "equal_to_reference": bool(equal)}
    for key, call in base.items():
        for _ in range(3):
            call()
        out[key] = {"call": timed(call, calls, repeats), "device_us": device_us(eng, call)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    out = {"config": {"calls": args.calls, "repeats": args.repeats, **gpu_info()}}
    for name in ("C3", "C5"):
        out[name] = one_config(eng, name, args.calls, args.repeats)
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
