"""The drain waves plan (lwse_resident_drain_waves) at C3 (10 000 nodes, 625 domains) and on the breach world of
tests/drain_budget_ref.py at 20 000 objects on 2 048 nodes, for both scopes, every key ordered by drain cost
(largest drain_budget_cost min_margin first) and max_waves 64:

  - the call time (wall clock around a call that returns once the plan is in host memory);
  - the device time from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1: behind the snapshot event, and
    after the last kernel; it includes the call's two sizing synchronisations);
  - the per-kernel times of a torch.profiler run of its own, and the plan kernel's time per key;
  - the number of waves and of keys per status, and whether the answer equals the reference
    (tests/drain_waves_ref.py, plan_fast);
  - the host-side first-fit the call replaces — each key against the set form alone, then against each open wave
    with one lwse_resident_drain_budget call — timed the same way once, and whether it plans the same.

The card's name and power limit are read in the same call.

    python profiles/microbench/drain_waves.py --out /tmp/drain_waves.json
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
from lws_b200 import synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from place_whatif import event_device_us, kernel_profile, timed  # noqa: E402


def host_first_fit(eng, scope, ids):
    """The plan from set-form calls alone: (wave per key, or -1 / -2 for breaches alone / no wave; calls made)."""
    waves, out, calls = [], [], 0
    for k in ids.tolist():
        calls += 1
        if eng.resident_drain_budget(**{scope: [k]})["n_breached"]:
            out.append(-1)
            continue
        for w, W in enumerate(waves):
            calls += 1
            if eng.resident_drain_budget(**{scope: W + [k]})["n_breached"] == 0:
                W.append(k)
                out.append(w)
                break
        else:
            if len(waves) < R.DRAIN_WAVES_MAX:
                waves.append([k])
                out.append(len(waves) - 1)
            else:
                out.append(-2)
    return np.asarray(out), calls


def measure(eng, t, args):
    import oracle
    from drain_waves_ref import orders, plan_fast

    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_tick(eng.make_tick((), t.flags))
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.flags & R.SWEEP_GANG, threads=16)[:2]
    out = {"nodes": len(t.nodes), "domains": t.n_domains, "lws": len(t.lws), "groups": len(t.groups),
           "pods": len(t.pod_state)}
    for scope in ("nodes", "domains"):
        cost = eng.resident_drain_budget_cost(scope)
        ids = orders(np.arange(len(cost)), cost)["by_cost"]
        call = lambda: eng.resident_drain_waves(**{scope: ids})
        for _ in range(3):
            call()
        got = call()
        keys, waves, tot = plan_fast(t.lws, base[0], t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, base[1], ids,
                                     scope == "domains")
        equal = (got["keys"].tobytes() == keys.tobytes() and got["waves"].tobytes() == waves.tobytes()
                 and {k: got[k] for k in R.DRAIN_WAVES_TOTALS} == tot)
        kern = kernel_profile(call)
        plan_us = next((v for k, v in kern["per_call"].items() if "drain_waves_plan_kernel" in k), None)
        t0 = time.perf_counter()
        host_plan, host_calls = host_first_fit(eng, scope, ids)
        host_s = time.perf_counter() - t0
        dev_plan = np.where(got["keys"]["status"] == R.DRAINW_PLANNED, got["keys"]["wave"].astype(np.int64),
                            np.where(got["keys"]["status"] == R.DRAINW_BREACHES_ALONE, -1, -2))
        out[scope] = {"keys": len(ids), "call": timed(call, args.calls, args.repeats),
                      "device": event_device_us(eng, call, args.calls * args.repeats), "kernels": kern,
                      "plan_kernel_us_per_key": plan_us / len(ids) if plan_us is not None and len(ids) else None,
                      **{k: int(got[k]) for k in R.DRAIN_WAVES_TOTALS}, "equal_to_reference": bool(equal),
                      "host_first_fit": {"s": host_s, "set_form_calls": host_calls,
                                         "same_plan": bool(np.array_equal(host_plan, dev_plan))}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from drain_budget_ref import budget_world

    out = {"config": {"calls": args.calls, "repeats": args.repeats, **gpu_info()}}
    eng = Engine(0)
    out["C3"] = measure(eng, synth.make("C3", 1.0, seed=synth.SEED), args)
    out["breach"] = measure(eng, budget_world(n_lws=20_000, n_nodes=2048, seed=17), args)
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
