"""The rollout forecast (lwse_ds_resident_forecast) at C4: 50 000 DisaggregatedSets, 2 roles.

  - the call (wall clock around a call that returns once the forecast is in host memory), with the
    trajectory rows and with summaries only;
  - device time per kernel from torch.profiler CUDA activity records of a run of its own (summary pass,
    scan, trajectory pass, copies);
  - cycle and step counts of the forecast;
  - the CPU reference of the same forecast in the same process, and whether the engine's bytes equal it.
    It is tests/ds_forecast_ref.py: numpy over the C oracle's sweep, one thread, every DS of the table
    swept in each of its batched cycles (DS that have stopped included).  It is not a serial replay of
    one DS at a time.

The card's name and power limit are read in the same call.

    python profiles/microbench/ds_forecast.py --out /tmp/ds_forecast.json
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


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from ds_forecast_ref import ds_forecast

    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    d = synth.make_ds(50_000, (2,))
    out = {"config": {"ds": len(d.ds), "roles": len(d.roles), "revroles": len(d.revroles), "calls": args.calls,
                      "repeats": args.repeats, **gpu_info()}}
    eng.ds_resident_load(d.ds, d.roles, d.revroles)
    eng.ds_resident_tick()
    first = eng.ds_resident_forecast(steps=True)
    cap = int(first["n_steps_needed"])
    for _ in range(3):
        eng.ds_resident_forecast(steps=True, step_capacity=cap)
        eng.ds_resident_forecast(steps=False)
    out["call_with_trajectory"] = timed(lambda: eng.ds_resident_forecast(steps=True, step_capacity=cap),
                                        args.calls, args.repeats)
    out["call_summaries_only"] = timed(lambda: eng.ds_resident_forecast(steps=False), args.calls, args.repeats)
    for steps in (True, False):
        n_prof = 10
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                eng.ds_resident_forecast(steps=steps, step_capacity=cap)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                name = ev.name
                # (torch.profiler reports demangled names: "void lwse::ds_forecast_kernel<true>(...)")
                key = ("forecast_kernel<write>" if "ds_forecast_kernel<true>" in name else
                       "forecast_kernel<summary>" if "ds_forecast_kernel<false>" in name else
                       "scan" if "scan" in name else "memcpy" if "emcpy" in name else
                       "memset" if "emset" in name else name[:40])
                per[key] = per.get(key, 0.0) + ev.device_time_total
        per = {k: v / n_prof for k, v in per.items()}
        out["device_us_with_trajectory" if steps else "device_us_summaries_only"] = {
            "per_call": per, "total": float(sum(per.values()))}
    fc = first["ds"]
    cyc = fc["cycles"].astype(np.int64)
    stp = fc["n_steps"].astype(np.int64)
    out["forecast"] = {
        "rolling": int(((fc["flags"] & 1) != 0).sum()), "done": int(((fc["flags"] & 4) != 0).sum()),
        "unfinished": int(((fc["flags"] & 8) != 0).sum()),
        "cycles_max": int(cyc.max()), "cycles_mean": float(cyc.mean()),
        "cycles_p50_p90_p99": [float(np.percentile(cyc, p)) for p in (50, 90, 99)],
        "steps_max": int(stp.max()), "steps_mean": float(stp.mean()), "trajectory_rows": cap,
    }
    # the CPU reference, one thread, same process
    t0 = time.perf_counter()
    ref = ds_forecast(d.ds, d.roles, d.revroles)
    out["cpu_reference_s"] = time.perf_counter() - t0
    out["cpu_reference_replay_cycles"] = int(ref["cycles_run"])
    out["equal_to_reference"] = bool(ref["ds"].tobytes() == first["ds"].tobytes()
                                     and ref["roles"].tobytes() == first["roles"].tobytes()
                                     and ref["steps"].tobytes() == first["steps"].tobytes())
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
