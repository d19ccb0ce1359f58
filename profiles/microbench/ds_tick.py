"""The DS tick (lwse_ds_resident_tick) at C4 and its effect on the pipelined LeaderWorkerSet tick.

  (1) C4 (50 000 DisaggregatedSets, 2 roles) at 0.1 %, 1 % and 10 % revision-role churn per tick
      (status updates of child LeaderWorkerSets: readyReplicas, sometimes replicas): the lone call
      (wall clock around a call that returns once its results are in pinned memory) and the device
      time of its kernels (torch.profiler CUDA activity records of a run of its own: scatter, sweep,
      copies), plus the number of DS listed per tick.  For comparison the stateless
      lwse_sweep_ds_host of the same tables (all three tables up, all three down).
  (2) C3 pipelined LeaderWorkerSet ticks at 1 % churn (two in flight), with and without a C4 DS tick
      at 1 % churn issued between each submit and wait, alternating window by window in one process.

The card's name and power limit are read in the same call; the DS mirrors are checked against the
oracle at the end of every churn level.

    python profiles/microbench/ds_tick.py --out /tmp/ds_tick.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from lws_b200 import churn, synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402

CHURN = (0.001, 0.01, 0.1)


def revrole_sets(rr: np.ndarray, frac: float, n_sets: int, seed: int) -> list:
    """[(rows, values)] status updates of `frac` of the revision-role rows per tick."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_sets):
        rows = np.unique(rng.choice(len(rr), size=max(1, int(len(rr) * frac)), replace=False)).astype(np.uint32)
        v = R.aligned_empty(len(rows), R.DS_REVROLE_REC)
        v[:] = rr[rows]
        v["ready_replicas"] = rng.integers(0, 33, size=len(rows))
        scale = rng.random(len(rows)) < 0.2
        v["replicas"] = np.where(scale, rng.integers(0, 33, size=len(rows)), v["replicas"])
        out.append((rows, v))
    return out


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def ds_level(eng, d, frac, steps, repeats):
    import oracle
    import torch
    from torch.profiler import ProfilerActivity, profile

    sets = revrole_sets(d.revroles, frac, 8, seed=int(frac * 1e4) + 1)
    rr = d.revroles.copy()
    eng.ds_resident_load(d.ds, d.roles, rr)
    eng.ds_resident_tick()
    i = 0
    lat, listed = [], []
    for _ in range(repeats):
        for _ in range(8):  # warm-up of the window
            rows, v = sets[i % 8]
            eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
            i += 1
        t0 = time.perf_counter()
        for _ in range(steps):
            rows, v = sets[i % 8]
            res = eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
            listed.append(res["n_changed"])
            i += 1
        lat.append((time.perf_counter() - t0) / steps * 1e6)
    for k in range(i):  # the host mirror of the i ticks, outside the timed loops
        rr[sets[k % 8][0]] = sets[k % 8][1]
    want = oracle.sweep_ds(d.ds, d.roles, rr)
    ok = all(res[n].tobytes() == w.tobytes() for n, w in zip(("ds_out", "role_out", "revrole_out"), want))
    # device time: the kernels and copies of 50 ticks in a profiled run of their own
    n_prof = 50
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            rows, v = sets[i % 8]
            eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
            i += 1
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            key = "ds_sweep_kernel" if "ds_sweep_kernel" in ev.name else ("scatter" if "scatter" in ev.name else
                                                                        ("memcpy" if "emcpy" in ev.name else ev.name[:40]))
            per[key] = per.get(key, 0.0) + ev.device_time_total
    per = {k: v / n_prof for k, v in per.items()}
    return {"call_us": lat, "call_us_median": float(np.median(lat)), "call_us_spread": [min(lat), max(lat)],
            "device_us_per_tick": per, "device_us_total": float(sum(per.values())),
            "rows_patched": int(len(sets[0][0])), "ds_listed_median": float(np.median(listed)),
            "mirrors_equal_oracle": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    d = synth.make_ds(50_000, (2,))
    out = {"config": {"ds": len(d.ds), "roles": len(d.roles), "revroles": len(d.revroles), "steps": args.steps,
                      "repeats": args.repeats, **gpu_info()}}
    # (1) the DS tick alone
    for frac in CHURN:
        out[f"ds_tick_churn_{frac:g}"] = ds_level(eng, d, frac, args.steps, args.repeats)
    host_out = (R.aligned_empty(len(d.ds), R.DS_OUT), R.aligned_empty(len(d.roles), R.DS_ROLE_OUT),
                R.aligned_empty(len(d.revroles), R.DS_REVROLE_OUT))
    for _ in range(5):
        eng.sweep_ds_host(d.ds, d.roles, d.revroles, out=host_out)
    stateless = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        for _ in range(20):
            eng.sweep_ds_host(d.ds, d.roles, d.revroles, out=host_out)
        stateless.append((time.perf_counter() - t0) / 20 * 1e6)
    out["stateless_sweep_ds_host_us_median"] = float(np.median(stateless))
    # (2) C3 pipelined LWS ticks with and without a DS tick between submit and wait
    t = synth.make("C3", 1.0, seed=synth.SEED)
    eng.upload_nodes(t.nodes, t.n_domains)
    flags = t.flags | R.TICK_PLACE
    reqs = t.place_requests()
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), flags))
    plan = churn.make_plan(t, reqs, eng.resident_place_outputs(), 0.01, 0.01)
    ticks = churn.ArenaPlan(eng, plan, flags).ticks
    ds_sets = revrole_sets(d.revroles, 0.01, 8, seed=77)
    eng.ds_resident_load(d.ds, d.roles, d.revroles)
    eng.ds_resident_tick()
    state = {"i": 0, "j": 0}

    def window(n, with_ds):
        eng.resident_tick_submit(ticks[state["i"] % len(ticks)])
        state["i"] += 1
        t0 = time.perf_counter()
        for _ in range(n):
            eng.resident_tick_submit(ticks[state["i"] % len(ticks)])
            state["i"] += 1
            if with_ds:
                rows, v = ds_sets[state["j"] % 8]
                eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
                state["j"] += 1
            eng.resident_tick_wait()
        dt = (time.perf_counter() - t0) / n
        eng.resident_tick_wait()
        return dt * 1e6

    res = {"lws_only_us": [], "lws_with_ds_tick_us": []}
    for _ in range(args.repeats):
        for name, with_ds in (("lws_only_us", False), ("lws_with_ds_tick_us", True)):
            window(8, with_ds)
            res[name].append(window(args.steps, with_ds))
    for name in list(res):
        res[name + "_median"] = float(np.median(res[name]))
    res["graph_on_steady_ticks"] = eng.resident_tick_info()["graph"]
    out["c3_pipelined_lws_tick"] = res
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
