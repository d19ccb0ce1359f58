"""The placement what-if (lwse_resident_place_whatif) at C3 (10 000 nodes, 625 domains, 98 072 requests).

  - five queries: (a) a new 16-group LeaderWorkerSet in one namespace, (b) a scale-up of one object by 4
    groups, (c) a cordon of one domain, (d) a cordon of 1 % of the nodes, (e) 1 % of the request rows patched;
  - per query the call (wall clock around a call that returns once the rows are in host memory); the device
    time of a call from CUDA events on the what-if stream (the engine records them with LWSE_WHATIF_TIMING=1:
    behind the snapshot event, and after the diff kernel — the copies back to the host not included; the
    gaps while the host enqueues are); and the per-kernel times of a torch.profiler run of its own;
  - for comparison, the device time of a tick that runs the full placement round alone (no sweep, no
    patches), from CUDA events on the engine's stream around the tick;
  - the device time of a tick (1 % node capacity patches, sweep and round) with and without a what-if (a)
    issued between its submit and its wait, alternating the two modes in one session;
  - whether each query's rows equal the spec reference (tests/test_place_whatif.py).

The card's name and power limit are read in the same call.

    python profiles/microbench/place_whatif.py --out /tmp/place_whatif.json
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
from lws_b200 import informer, synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402


def timed(fn, calls, repeats):
    lat = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        lat.append((time.perf_counter() - t0) / calls * 1e6)
    return {"us": lat, "us_median": float(np.median(lat)), "us_spread": [min(lat), max(lat)]}


def event_device_us(eng, fn, n):
    """Device time of each call on the what-if stream (the engine's CUDA events)."""
    import ctypes as C

    from lws_b200.engine import lib

    f = lib().lwse_debug_whatif_device_us
    f.argtypes, f.restype = [C.c_void_p, C.POINTER(C.c_float)], C.c_int
    lat = []
    for _ in range(n):
        fn()
        us = C.c_float()
        assert f(eng._h, C.byref(us)) == 0
        lat.append(float(us.value))
    return {"us": lat, "us_median": float(np.median(lat)), "us_spread": [min(lat), max(lat)]}


def kernel_profile(fn, n=10):
    """Mean device time per kernel / copy of a call (torch.profiler CUDA activity records)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    per = {}
    for _ in range(n):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        evs = [ev for ev in prof.events() if ev.device_type.name == "CUDA"]
        for ev in evs:
            n_ = ev.name
            key = ("memcpy" if "emcpy" in n_ else "memset" if "emset" in n_ else n_.split("(")[0].replace("void ", "")[:60])
            per[key] = per.get(key, 0.0) + ev.device_time_total / n
    return {"per_call": per, "total": float(sum(per.values()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from test_place_whatif import whatif_ref

    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    occ = R.occupancy_of(t.pod_ident, len(t.nodes))
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    rng = np.random.default_rng(3)
    n_ns = t.n_namespaces
    big_ns = int(np.argmax(np.bincount(reqs["ns"].astype(np.int64), minlength=n_ns)))

    def extra(n, ns):
        x = R.aligned_empty(n, R.PLACE_REQ)
        x["priority"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
        x["group_key"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64)
        x["group"], x["ns"], x["size"], x["leader_node"] = np.arange(n), ns, 4, R.NONE
        return x

    def node_seg(rows, edit):
        rows = np.unique(np.asarray(rows, dtype=np.uint32))
        vals = R.aligned_empty(len(rows), R.NODE_REC)
        vals[:] = t.nodes[rows]
        edit(vals)
        return (R.TABLE_NODES, rows, vals)

    def cordon(v):
        v["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)

    excl = np.flatnonzero((t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY) != 0)
    obj = int(excl[0])
    scale = informer.IncrementalEncoder._whatif_requests(
        int(t.lws["uid_hash"][obj]), int(t.lws["size"][obj]), int(t.ns_of_lws[obj]),
        range(int(t.lws["replicas"][obj]), int(t.lws["replicas"][obj]) + 4))
    live = np.flatnonzero(reqs["size"] >= 1)
    rows_e = np.sort(rng.choice(live, size=len(reqs) // 100, replace=False)).astype(np.uint32)
    vals_e = R.aligned_empty(len(rows_e), R.PLACE_REQ)
    vals_e[:] = reqs[rows_e]
    vals_e["leader_node"] = R.NONE
    vals_e["size"] += 1
    d = int(t.nodes["domain_id"][0])
    q = {
        "a_new_lws_16_groups": ([], extra(16, big_ns)),
        "b_scale_up_4_groups": ([], scale),
        "c_cordon_one_domain": ([node_seg(np.flatnonzero(t.nodes["domain_id"] == d), cordon)], None),
        "d_cordon_1pct_nodes": ([node_seg(rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False), cordon)], None),
        "e_requests_1pct": ([(R.TABLE_PLACE_REQS, rows_e, vals_e)], None),
    }
    out = {"config": {"calls": args.calls, "repeats": args.repeats, "ticks": args.ticks, "nodes": len(t.nodes),
                      "domains": t.n_domains, "requests": len(reqs), "namespaces": n_ns, **gpu_info()}}
    for name, (segs, x) in q.items():
        for _ in range(3):
            eng.resident_place_whatif(segs, x)
        got = eng.resident_place_whatif(segs, x)
        ref = whatif_ref(t.nodes, occ, t.n_domains, reqs, segs, x, n_ns=n_ns)
        order = np.argsort(got["rows"], kind="stable")
        equal = (np.array_equal(got["rows"][order], ref["rows"]) and got["after"][order].tobytes() == ref["after"].tobytes()
                 and got["extra_out"].tobytes() == ref["extra_out"].tobytes())
        out[name] = {"call": timed(lambda: eng.resident_place_whatif(segs, x), args.calls, args.repeats),
                     "device": event_device_us(eng, lambda: eng.resident_place_whatif(segs, x), args.calls * args.repeats),
                     "kernels": kernel_profile(lambda: eng.resident_place_whatif(segs, x)),
                     "n_changed": got["n_changed"], "namespaces_solved": got["namespaces_solved"], "form": got["form"],
                     "equal_to_reference": bool(equal)}

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

    round_only = eng.make_tick((), R.TICK_PLACE | R.TICK_NO_SWEEP)
    tick_device_us(round_only, n=5)
    lat = tick_device_us(round_only)
    out["tick_round_only_device_us"] = {"us_median": float(np.median(lat)), "us_spread": [min(lat), max(lat)]}
    rows = np.sort(rng.choice(len(t.nodes), size=len(t.nodes) // 100, replace=False)).astype(np.uint32)
    vals = R.aligned_empty(len(rows), R.NODE_REC)
    vals[:] = t.nodes[rows]
    tick = eng.make_tick([(R.TABLE_NODES, rows, vals)], t.flags | R.TICK_PLACE)  # (values rewritten with their own: a steady tick)
    wa_segs, wa_x = q["a_new_lws_16_groups"]
    modes = {"without_whatif": [], "with_whatif": []}
    tick_device_us(tick, n=5)
    for rep in range(4):
        for mode in ("without_whatif", "with_whatif"):
            modes[mode] += tick_device_us(tick, (lambda: eng.resident_place_whatif(wa_segs, wa_x)) if mode == "with_whatif" else None)
    out["tick_device_us"] = {k: {"us_median": float(np.median(v)), "us_spread": [min(v), max(v)], "n": len(v)} for k, v in modes.items()}
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
