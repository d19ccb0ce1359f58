"""The rolling-update forecast of LeaderWorkerSets (lwse_resident_forecast) at C3 and C5: 100 000 objects.

  - the call (wall clock around a call that returns once the forecast is in host memory), with the
    trajectory rows and with summaries only, over the resident tables after one tick;
  - device time per kernel from torch.profiler CUDA activity records of a run of its own (slot pass, slot
    scan, summary pass, step scan, trajectory pass, copies; each scan is three launches);
  - cycle and step counts of the forecast;
  - whether the engine's bytes equal the CPU reference (tests/lws_forecast_ref.py) on the same rows, and
    the reference's time (numpy over the C oracle's sweep, every object of the table swept in each
    batched cycle; not a serial replay of one object at a time).

The card's name and power limit are read in the same call.

    python profiles/microbench/lws_forecast.py --out /tmp/lws_forecast.json
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

from ds_tick import gpu_info  # noqa: E402
from lws_b200 import synth  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402


def timed(fn, calls, repeats):
    lat = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        lat.append((time.perf_counter() - t0) / calls * 1e6)
    return {"us": lat, "us_median": float(np.median(lat)), "us_spread": [min(lat), max(lat)]}


def one_config(eng, name, calls, repeats):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lws_forecast_ref import lws_forecast

    t = synth.make(name)
    out = {"lws": len(t.lws), "groups": len(t.groups), "pods": len(t.pod_state)}
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_tick(eng.make_tick((), t.flags))
    first = eng.resident_forecast(steps=True)
    cap = int(first["n_steps_needed"])
    for _ in range(3):
        eng.resident_forecast(steps=True, step_capacity=cap)
        eng.resident_forecast(steps=False)
    out["call_with_trajectory"] = timed(lambda: eng.resident_forecast(steps=True, step_capacity=cap), calls, repeats)
    out["call_summaries_only"] = timed(lambda: eng.resident_forecast(steps=False), calls, repeats)
    for steps in (True, False):
        n_prof = 10
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                eng.resident_forecast(steps=steps, step_capacity=cap)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                n = ev.name
                key = ("forecast_kernel<write>" if "lws_forecast_kernel" in n and "true>" in n else
                       "forecast_kernel<summary>" if "lws_forecast_kernel" in n else
                       "slots" if "forecast_slots_kernel" in n else
                       "slot_scan" if "scan_" in n and "SlotLayoutOp" in n else
                       "step_scan" if "scan_" in n and "StepLayoutOp" in n else "memcpy" if "emcpy" in n else
                       "memset" if "emset" in n else n[:40])
                per[key] = per.get(key, 0.0) + ev.device_time_total
        per = {k: v / n_prof for k, v in per.items()}
        out["device_us_with_trajectory" if steps else "device_us_summaries_only"] = {
            "per_call": per, "total": float(sum(per.values()))}
    fc = first["lws"]
    stp = fc["n_steps"].astype(np.int64)
    out["forecast"] = {
        "rolling": int(((fc["flags"] & 1) != 0).sum()), "waiting": int(((fc["flags"] & 2) != 0).sum()),
        "done": int(((fc["flags"] & 4) != 0).sum()), "unfinished": int(((fc["flags"] & 8) != 0).sum()),
        "held": int(((fc["flags"] & 32) != 0).sum()), "not_forecast": int(((fc["flags"] & 128) != 0).sum()),
        "steps_max": int(stp.max()), "steps_mean": float(stp.mean()),
        "steps_p50_p90_p99": [float(np.percentile(stp, p)) for p in (50, 90, 99)], "trajectory_rows": cap,
    }
    go = eng.resident_outputs()[1]
    t0 = time.perf_counter()
    ref = lws_forecast(t.lws, go)
    out["cpu_reference_s"] = time.perf_counter() - t0
    out["equal_to_reference"] = bool(ref["lws"].tobytes() == first["lws"].tobytes()
                                     and ref["steps"].tobytes() == first["steps"].tobytes())
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
