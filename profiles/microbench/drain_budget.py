"""The drain budget (lwse_resident_drain_budget*) at C3 (10 000 nodes, 625 domains) and on the breach world of
tests/drain_budget_ref.py at 20 000 objects on 2 048 nodes (floors that bind):

  - the call time (wall clock around a call that returns once the rows are in host memory) of the set form for
    one node, one domain and 1 % of the nodes, and of the per-key form for all nodes and all domains;
  - the device time of each call from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1: behind the
    snapshot event, and after the last kernel; for the per-key form this includes the host synchronisation
    that sizes the table);
  - the per-kernel times of a torch.profiler run of its own;
  - whether each answer equals the reference (tests/drain_budget_ref.py; the set form against the spec oracle).

The card's name and power limit are read in the same call.

    python profiles/microbench/drain_budget.py --out /tmp/drain_budget.json
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
from lws_b200 import synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from place_whatif import event_device_us, kernel_profile, timed  # noqa: E402


def measure(eng, t, args):
    import oracle
    from drain_budget_ref import domain_nodes, drain_budget_cost_ref, drain_budget_ref

    fl = t.flags & R.SWEEP_GANG
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_tick(eng.make_tick((), t.flags))
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl, threads=16)[:2]
    rng = np.random.default_rng(3)
    dom = int(rng.integers(0, t.n_domains))
    out = {"nodes": len(t.nodes), "domains": t.n_domains, "lws": len(t.lws), "groups": len(t.groups),
           "pods": len(t.pod_state)}
    sets = {"one_node": ({"nodes": [int(rng.integers(0, len(t.nodes)))]}, None),
            "one_domain": ({"domains": [dom]}, domain_nodes(t.nodes, t.n_domains, [dom])),
            "nodes_1pct": ({"nodes": rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False)}, None)}
    for name, (kw, d) in sets.items():
        d = kw["nodes"] if d is None else d
        call = lambda: eng.resident_drain_budget(**kw)
        for _ in range(3):
            call()
        got = call()
        rows, ref = drain_budget_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, d, fl, base=base)
        o = np.argsort(got["rows"]["lws"], kind="stable")
        equal = got["rows"][o].tobytes() == rows.tobytes() and all(got[k] == ref[k] for k in R.DRAIN_BUDGET_TOTALS)
        out[name] = {"call": timed(call, args.calls, args.repeats),
                     "device": event_device_us(eng, call, args.calls * args.repeats),
                     "kernels": kernel_profile(call), **{k: int(got[k]) for k in R.DRAIN_BUDGET_TOTALS},
                     "equal_to_reference": bool(equal)}
    for scope in ("nodes", "domains"):
        call = lambda: eng.resident_drain_budget_cost(scope)
        for _ in range(3):
            call()
        got = call()
        ref = drain_budget_cost_ref(t.lws, base[0], t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, base[1],
                                    scope == "domains")
        out["cost_" + scope] = {"call": timed(call, args.calls, args.repeats),
                                "device": event_device_us(eng, call, args.calls * args.repeats),
                                "kernels": kernel_profile(call),
                                "lws_touched": int(got["lws_touched"].sum()), "lws_breached": int(got["lws_breached"].sum()),
                                "lws_loses_available": int(got["lws_loses_available"].sum()),
                                "equal_to_reference": bool(got.tobytes() == ref.tobytes())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
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
