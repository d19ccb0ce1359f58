"""The DS drain (lwse_resident_ds_drain*) on a world with C4-sized DS tables: 50 000 DisaggregatedSets of 2 roles
(1-3 old revisions, tests/ds_drain_ref.py's ds_drain_world) whose revision-role rows link to child LeaderWorkerSets
of 2-8 pod groups bound to 2 048 nodes in 16-node domains:

  - the call time (wall clock around a call that returns once the rows are in host memory) of the set form for
    one node, one domain, 1 % of the nodes, every node and every domain, and of the per-key form for all nodes and
    all domains;
  - the device time of each call from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1; for the per-key
    form this includes the two host synchronisations that size the tables);
  - the per-kernel times of a torch.profiler run of its own;
  - the drain budget (lwse_resident_drain_budget*) on the same world, one domain and per key, for comparison;
  - whether each answer equals the reference (tests/ds_drain_ref.py).

The card's name and power limit are read in the same call.

    python profiles/microbench/ds_drain.py --out /tmp/ds_drain.json
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


def measure(eng, w, args):
    from ds_drain_ref import TOTALS, ds_drain_cost_ref, ds_drain_domains_ref, ds_drain_ref

    eng.upload_nodes(w.nodes, w.n_domains)
    eng.resident_load(w.lws, w.groups, w.pod_state, w.pod_ident)
    eng.resident_tick(eng.make_tick((), w.flags))
    eng.ds_resident_load(w.ds, w.roles, w.revroles)
    eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, w.links, True)])
    res = eng.resident_outputs()
    assert res[0].tobytes() == w.base[0].tobytes() and res[1].tobytes() == w.base[1].tobytes()
    rng = np.random.default_rng(3)
    dom = int(rng.integers(0, w.n_domains))
    out = {"ds": len(w.ds), "revision_role_rows": len(w.revroles), "lws": len(w.lws), "groups": len(w.groups),
           "pods": len(w.pod_state), "nodes": len(w.nodes), "domains": w.n_domains,
           "rows_linked": int(eng.resident_ds_drain(nodes=[])["rows_linked"])}
    sets = {"one_node": {"nodes": [int(rng.integers(0, len(w.nodes)))]},
            "one_domain": {"domains": [dom]},
            "nodes_1pct": {"nodes": rng.choice(len(w.nodes), size=len(w.nodes) // 100, replace=False)},
            "every_node": {"nodes": np.arange(len(w.nodes))},
            "every_domain": {"domains": np.arange(w.n_domains)}}
    for name, kw in sets.items():
        call = lambda: eng.resident_ds_drain(**kw)
        for _ in range(3):
            call()
        got = call()
        ref = (ds_drain_domains_ref(w, list(kw["domains"])) if "domains" in kw else ds_drain_ref(w, list(kw["nodes"])))
        o = np.argsort(got["rows"]["ds"], kind="stable")
        equal = got["rows"][o].tobytes() == ref[0].tobytes() and all(got[k] == ref[1][k] for k in TOTALS)
        out[name] = {"call": timed(call, args.calls, args.repeats),
                     "device": event_device_us(eng, call, args.calls * args.repeats),
                     "kernels": kernel_profile(call), **{k: int(got[k]) for k in TOTALS},
                     "equal_to_reference": bool(equal)}
    for scope in ("nodes", "domains"):
        call = lambda: eng.resident_ds_drain_cost(scope)
        for _ in range(3):
            call()
        got = call()
        ref = ds_drain_cost_ref(w, scope == "domains")
        out["cost_" + scope] = {"call": timed(call, args.calls, args.repeats),
                                "device": event_device_us(eng, call, args.calls * args.repeats),
                                "kernels": kernel_profile(call),
                                **{f: int(got[f].sum()) for f in ("ds_touched", "ds_service_lost", "ds_old_service_lost",
                                                                  "ds_stalled", "rows_touched", "rows_zeroed")},
                                "equal_to_reference": bool(got.tobytes() == ref.tobytes())}
    # the LeaderWorkerSet drain budget on the same world
    for name, call in (("budget_one_domain", lambda: eng.resident_drain_budget(domains=[dom])),
                       ("budget_cost_nodes", lambda: eng.resident_drain_budget_cost("nodes")),
                       ("budget_cost_domains", lambda: eng.resident_drain_budget_cost("domains"))):
        for _ in range(3):
            call()
        out[name] = {"call": timed(call, args.calls, args.repeats),
                     "device": event_device_us(eng, call, args.calls * args.repeats)}
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
