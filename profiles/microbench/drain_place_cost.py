"""The drain placement (lwse_resident_drain_place_cost) at C3 (10 000 nodes, 625 domains, 98 072 requests), both
scopes:

  - the call time (wall clock around a call that returns once the rows are in host memory);
  - the device time from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1: behind the snapshot event, and
    after the last kernel; it includes the call's three host synchronisations);
  - the per-kernel times of a torch.profiler run of its own;
  - the namespaces solved (items) and the unpinned rows over all keys;
  - in the same process, the three-call composition (drain what-if → unpin → place what-if) looped over every
    domain and over every node (or a seeded sample, --node-sample; the count is recorded), and whether its rows
    equal the call's.

The card's name and power limit are read in the same call.

    python profiles/microbench/drain_place_cost.py   # writes profiles/h100_drain_place_cost.json
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_drain_place_cost.json"))
    ap.add_argument("--node-sample", type=int, default=0, help="node keys the composition loop runs (0: all)")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from test_gpu_drain_place_cost import composition

    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    res = {"gpu_info": gpu_info(), "nodes": len(t.nodes), "domains": t.n_domains, "requests": len(reqs),
           "namespaces": t.n_namespaces}
    d = t.nodes["domain_id"].astype(np.int64)
    rng = np.random.default_rng(11)
    for scope in ("domains", "nodes"):
        call = lambda: eng.resident_drain_place_cost(scope)
        for _ in range(3):
            got = call()
        r = {"call": timed(call, 5, args.repeats), "device_us": event_device_us(eng, call, 10),
             "items": int(got["namespaces_solved"].sum()), "unpinned": int(got["unpinned"].sum()),
             "stranded": int(got["stranded"].sum()), "keys_with_stranded": int((got["stranded"] > 0).sum())}
        if scope == "domains":
            keys = list(range(t.n_domains))
        elif args.node_sample:
            keys = sorted(rng.choice(len(t.nodes), size=args.node_sample, replace=False).tolist())
        else:
            keys = list(range(len(t.nodes)))
        t0 = time.perf_counter()
        same = 0
        for k in keys:
            drained = np.array([k]) if scope == "nodes" else np.flatnonzero(d == k)
            want = composition(eng, t, reqs, drained)
            row = got[k].copy()
            row["namespaces_solved"] = 0
            same += int(row.tobytes() == want.tobytes())
        loop = time.perf_counter() - t0
        r["composition"] = {"keys": len(keys), "seconds": loop, "us_per_key": loop / len(keys) * 1e6,
                            "rows_equal": same}
        r["kernels"] = kernel_profile(call, 5)
        res[scope] = r
        print(scope, json.dumps({k: v for k, v in r.items() if k != "kernels"}), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
