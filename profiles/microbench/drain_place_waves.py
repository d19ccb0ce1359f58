"""The drain placement waves plan (lwse_resident_drain_place_waves) at C3 (10 000 nodes, 625 domains), keys ordered
by drain cost (largest drain_budget_cost min_margin first, then fewest groups restarted), max_waves 8 and 64, with
the default constraints (LWS floor and stranded) and with the LWS floor alone, both scopes (by nodes: the first
``--node-keys`` keys):

  - the call time (wall clock around a call that returns once the plan is in host memory) and the device time from
    CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1, including the call's sizing synchronisations);
  - the device time per key of the step graph: (the call's device time - a call with no key) / keys;
  - the items solved: the sum of namespaces_solved over the waves' final probes, and the waves and statuses;
  - the host first-fit the call replaces, each probe the engine's three-call composition (drain what-if, unpin,
    place what-if) plus the set-form drain budget, over the first ``--host-keys`` keys: the time per probe and the
    probes made, and whether it plans those keys the same.

The card's name and power limit are read in the same call.

    python profiles/microbench/drain_place_waves.py --out /tmp/drain_place_waves.json
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
from place_whatif import event_device_us  # noqa: E402

DEFAULT = R.DPW_LWS_FLOOR | R.DPW_STRANDED


def composition(eng, t, reqs, drained):
    """(stranded, bumped, breached) of the engine's set forms over a node set."""
    from test_gpu_drain_place_cost import composition as comp

    row = comp(eng, t, reqs, drained)
    return int(row["stranded"]), int(row["bumped"]), int(eng.resident_drain_budget(nodes=drained)["n_breached"])


def host_first_fit(eng, t, reqs, ids, by_domain, constraints, max_waves):
    d = t.nodes["domain_id"].astype(np.int64)
    nodes_of = (lambda k: np.flatnonzero(d == k)) if by_domain else (lambda k: np.array([k]))
    waves, out, probes = [], [], 0

    def bad(keys):
        nonlocal probes
        probes += 1
        s, b, br = composition(eng, t, reqs, np.concatenate([nodes_of(k) for k in keys]))
        return ((constraints & R.DPW_LWS_FLOOR and br) or (constraints & R.DPW_STRANDED and s)
                or (constraints & R.DPW_BUMPED and b))

    t0 = time.perf_counter()
    for k in ids:
        if bad([k]):
            out.append(R.NONE)
            continue
        for w, W in enumerate(waves):
            if not bad(W + [k]):
                W.append(k)
                out.append(w)
                break
        else:
            if len(waves) < max_waves:
                waves.append([k])
                out.append(len(waves) - 1)
            else:
                out.append(R.NONE)
    dt = time.perf_counter() - t0
    return out, probes, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--node-keys", type=int, default=2000)
    ap.add_argument("--host-keys", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    res = {"config": "C3", "gpu": gpu_info(), "runs": []}
    for scope in ("domains", "nodes"):
        cost = eng.resident_drain_budget_cost(scope)
        ids = np.arange(len(cost))
        ids = ids[np.lexsort((ids, cost["groups_restarted"], -cost["min_margin"].astype(np.int64)))]
        if scope == "nodes":
            ids = ids[: a.node_keys]
        call = lambda ks, cap, cons: eng.resident_drain_place_waves(max_waves=cap, constraints=cons, **{scope: ks})
        for cap in (8, 64):
            for name, cons in (("default", DEFAULT), ("lws_floor", R.DPW_LWS_FLOOR)):
                got = call(ids, cap, cons)  # (warm-up)
                wall = []
                for _ in range(a.repeats):
                    t0 = time.perf_counter()
                    call(ids, cap, cons)
                    wall.append((time.perf_counter() - t0) * 1e3)
                dev = event_device_us(eng, lambda: call(ids, cap, cons), a.repeats)
                empty = event_device_us(eng, lambda: call(ids[:0], cap, cons), a.repeats)
                dmed, emed = float(np.median(dev["us"])), float(np.median(empty["us"]))
                res["runs"].append({
                    "scope": scope, "keys": int(len(ids)), "max_waves": cap, "constraints": name,
                    "call_ms_median": float(np.median(wall)), "call_ms": wall,
                    "device_us_median": dmed, "device_us_no_keys_median": emed,
                    "step_us_per_key": (dmed - emed) / max(len(ids), 1),
                    "items_solved_in_final_probes": int(got["waves"]["namespaces_solved"].sum()),
                    "n_waves": int(got["n_waves"]), "n_planned": int(got["n_planned"]),
                    "n_breaches_alone": int(got["n_breaches_alone"]), "n_no_wave": int(got["n_no_wave"])})
                print(json.dumps(res["runs"][-1]), flush=True)
        hk = ids[: a.host_keys]
        got = call(hk, 64, DEFAULT)
        out, probes, dt = host_first_fit(eng, t, reqs, [int(k) for k in hk], scope == "domains", DEFAULT, 64)
        planned = [int(w) if s == R.DRAINW_PLANNED else R.NONE for w, s in zip(got["keys"]["wave"], got["keys"]["status"])]
        res["runs"].append({"scope": scope, "host_first_fit_keys": int(len(hk)), "probes": probes,
                            "host_ms": dt * 1e3, "host_ms_per_probe": dt * 1e3 / max(probes, 1),
                            "same_plan": planned == out})
        print(json.dumps(res["runs"][-1]), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
