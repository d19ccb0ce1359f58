"""The drain what-if (lwse_resident_drain_whatif) and the drain cost of every node (lwse_resident_drain_cost) at
C3 (10 000 nodes, 98 072 groups, 6.3 M pods).

  - the call time (wall clock around a call that returns once the rows are in host memory) of the cost of
    every node, and of the what-if for one node, one domain and 1 % of the nodes;
  - the device time of each call from CUDA events on the what-if stream (the engine records them with
    LWSE_WHATIF_TIMING=1: behind the snapshot event, and after the last kernel — the copies back to the host
    not included);
  - the per-kernel times of a torch.profiler run of its own, and the cost kernel's achieved bytes/s against
    its algorithmic bytes (16 B of identity + 1 B of state per pod, 64 + 16 B of group row and owner prefix
    and 16 B of baseline group result per group);
  - the device time of a tick (1 % pod-state patches, sweep and round) with and without a drain what-if of
    one domain between its submit and its wait, alternating the two modes in one session;
  - whether the cost rows equal the numpy restatement (tests/drain_ref.py) and each what-if the spec oracle.

The card's name and power limit are read in the same call.

    python profiles/microbench/drain_whatif.py --out /tmp/drain_whatif.json
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import oracle
    from drain_ref import drain_cost_ref, drain_whatif_ref

    t = synth.make("C3", 1.0, seed=synth.SEED)
    fl = t.flags & R.SWEEP_GANG
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(t.place_requests(), t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    rng = np.random.default_rng(3)
    n_pods, n_groups = len(t.pod_state), len(t.groups)
    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, fl, threads=16)[:2]
    dom = int(rng.integers(0, t.n_domains))
    sets = {"one_node": [int(rng.integers(0, len(t.nodes)))],
            "one_domain": np.flatnonzero(t.nodes["domain_id"] == dom).tolist(),
            "nodes_1pct": rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False).tolist()}
    out = {"config": {"calls": args.calls, "repeats": args.repeats, "ticks": args.ticks, "nodes": len(t.nodes),
                      "groups": n_groups, "pods": n_pods, **gpu_info()}}

    for _ in range(3):
        eng.resident_drain_cost()
    cost = eng.resident_drain_cost()
    prof = kernel_profile(lambda: eng.resident_drain_cost())
    k_us = next(v for k, v in prof["per_call"].items() if "drain_cost_kernel" in k)
    alg = 17 * n_pods + 96 * n_groups
    out["drain_cost"] = {"call": timed(lambda: eng.resident_drain_cost(), args.calls, args.repeats),
                         "device": event_device_us(eng, lambda: eng.resident_drain_cost(), args.calls * args.repeats),
                         "kernels": prof, "algorithmic_bytes": alg, "kernel_us": k_us,
                         "achieved_bytes_per_s": alg / (k_us * 1e-6),
                         "groups_restarted_total": int(cost["groups_restarted"].sum()),
                         "equal_to_reference": bool(cost.tobytes() == drain_cost_ref(
                             t.lws, t.groups, t.pod_state, t.pod_ident, len(t.nodes), base[1]).tobytes())}
    for name, d in sets.items():
        for _ in range(3):
            eng.resident_drain_whatif(d)
        got = eng.resident_drain_whatif(d)
        ref = drain_whatif_ref(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, d, fl, base=base)
        o = np.argsort(got["rows"], kind="stable")
        equal = (np.array_equal(got["rows"][o], ref["rows"]) and got["after"][o].tobytes() == ref["after"].tobytes()
                 and all(got[k] == ref[k] for k in R.DRAIN_WHATIF))
        out[name] = {"call": timed(lambda: eng.resident_drain_whatif(d), args.calls, args.repeats),
                     "device": event_device_us(eng, lambda: eng.resident_drain_whatif(d), args.calls * args.repeats),
                     "kernels": kernel_profile(lambda: eng.resident_drain_whatif(d)),
                     "nodes": len(d), **{k: int(got[k]) for k in R.DRAIN_WHATIF}, "equal_to_reference": bool(equal)}

    es = torch.cuda.ExternalStream(eng.stream)

    def tick_device_us(tick, between=None, n=args.ticks):
        lat = []
        for _ in range(n):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(es)
            eng.resident_tick_submit(tick)
            b.record(es)
            if between is not None:
                between()
            eng.resident_tick_wait()
            torch.cuda.synchronize()
            lat.append(a.elapsed_time(b) * 1e3)
        return lat

    rows = np.sort(rng.choice(n_pods, size=n_pods // 100, replace=False)).astype(np.uint32)
    tick = eng.make_tick([(R.TABLE_POD_STATE, rows, t.pod_state[rows].copy())], t.flags | R.TICK_PLACE)  # (own values: steady)
    d = sets["one_domain"]
    modes = {"without_whatif": [], "with_whatif": []}
    tick_device_us(tick, n=5)
    for _ in range(4):
        for mode in ("without_whatif", "with_whatif"):
            modes[mode] += tick_device_us(tick, (lambda: eng.resident_drain_whatif(d)) if mode == "with_whatif" else None)
    out["tick_device_us"] = {k: {"us_median": float(np.median(v)), "us_spread": [min(v), max(v)], "n": len(v)}
                             for k, v in modes.items()}
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
