"""The scale headroom (lwse_resident_scale_headroom) at C3 (10 000 nodes, 625 domains, 100 000 exclusive objects of one
group in 200 namespaces), asked for every exclusive object in its own namespace, with no ceiling and with the ceiling
replicas + 8:

  - the call (wall clock around a call that returns once the answer is in host memory) and its device time (CUDA
    events on the what-if stream, LWSE_WHATIF_TIMING=1: behind the snapshot event and after the finish kernel);
  - the per-kernel times of a torch.profiler run of its own;
  - the rounds and the entries per flag;
  - the alternative a caller has without the call: a host-driven bisection over the same bounds, one
    lwse_resident_rollout_place call with the scale-only proposals P(mid) of every entry still searching per round
    (the r0 probe from the resident rows first); its answers are asserted equal to the call's.

The card's name and power limit are read in the same run.

    python profiles/microbench/scale_headroom.py   # writes profiles/h100_scale_headroom.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

os.environ["LWSE_WHATIF_TIMING"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from ds_tick import gpu_info  # noqa: E402
from lws_b200 import synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from place_whatif import event_device_us, kernel_profile, timed  # noqa: E402


def host_bounds(t, rows, ceil):
    """hi = min(c + 1, R_pig) (at least r0 + 1) and whether the ceiling bounds it, per entry, from the tables."""
    lws, gflags, nd = t.lws, t.groups["flags"], int(t.n_domains)
    hi = np.zeros(len(rows), np.int64)
    by_ceil = np.zeros(len(rows), bool)
    for j, r in enumerate(rows.tolist()):
        gb, gc, r0 = int(lws["group_base"][r]), int(lws["group_count"][r]), int(lws["replicas"][r])
        miss = np.flatnonzero((gflags[gb: gb + gc] & R.GRP_POD_PRESENT) == 0)
        pig = int(miss[nd]) + 1 if len(miss) > nd else gc + (nd + 1 - len(miss))
        c = -1 if ceil is None else int(ceil[j])
        by_ceil[j] = 0 <= c and c + 1 <= pig
        hi[j] = max(c + 1 if by_ceil[j] else pig, r0 + 1)
    return hi, by_ceil


def host_bisection(eng, t, rows, ns, ceil, mask, settled):
    """max_replicas per settled entry from one resident_rollout_place call per round → (H, rounds)."""
    trig = lambda o: ((o["stranded"] > 0) & bool(mask & R.RPW_STRANDED)) | (
        ((o["own_lost"] > 0) | (o["bumped"] > 0)) & bool(mask & R.RPW_BUMPED))
    idx = np.flatnonzero(settled)
    r0 = t.lws["replicas"][rows[idx]].astype(np.int64)
    hi, by_ceil = host_bounds(t, rows[idx], None if ceil is None else ceil[idx])
    lo = r0.copy()
    blocked = trig(eng.resident_rollout_place(rows[idx], ns[idx])["rows"])
    probed = np.zeros(len(idx), bool)
    rounds = 0
    while True:
        bis = ~blocked & (hi - lo > 1)
        fin = ~blocked & (hi - lo == 1) & ~by_ceil & ~probed
        act = np.flatnonzero(bis | fin)
        if not len(act):
            break
        mid = np.where(bis[act], lo[act] + (hi[act] - lo[act]) // 2, hi[act])
        recs = R.aligned_empty(len(act), R.LWS_REC)
        recs[:] = t.lws[rows[idx[act]]]
        recs["replicas"] = mid
        bad = trig(eng.resident_rollout_place(rows[idx[act]], ns[idx[act]], recs)["rows"])
        hi[act] = np.where(bad, mid, hi[act])
        probed[act] |= bad
        lo[act] = np.where(bad, lo[act], mid)
        rounds += 1
    return np.where(blocked, -1, lo), rounds


def run(eng, t, with_ceiling, repeats):
    rows = np.flatnonzero(t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY).astype(np.uint32)
    ns = t.ns_of_lws[rows].astype(np.uint32)
    ceil = (t.lws["replicas"][rows] + 8).astype(np.int32) if with_ceiling else None
    mask = R.RPW_STRANDED
    call = lambda: eng.resident_scale_headroom(rows, ns, ceil, mask)
    got = call()
    out = got["rows"]
    flags = {name: int(((out["flags"] & b) != 0).sum()) for b, name in R.SHR_NAMES.items()}
    settled = (out["flags"] & R.SHR_SOLVED) != 0
    t0 = time.perf_counter()
    h, host_rounds = host_bisection(eng, t, rows, ns, ceil, mask, settled)
    host_s = time.perf_counter() - t0
    assert h.tolist() == out["max_replicas"][settled].astype(np.int64).tolist(), "host bisection disagrees"
    host = timed(lambda: host_bisection(eng, t, rows, ns, ceil, mask, settled), 1, max(2, repeats // 2))
    res = {"objects": int(len(rows)), "ceiling": "replicas + 8" if with_ceiling else None, "rounds": int(got["rounds"]),
           "entries_per_flag": flags, "headroom_sum": int(got["headroom"]),
           "max_replicas_minus_r0_hist": np.bincount(
               (out["max_replicas"][settled & ((out["flags"] & R.SHR_BLOCKED) == 0)] -
                out["replicas"][settled & ((out["flags"] & R.SHR_BLOCKED) == 0)]).astype(np.int64)).tolist(),
           "call": timed(call, 2, repeats), "device": event_device_us(eng, call, 2 * repeats),
           "kernels": kernel_profile(call, 5),
           "host_bisection": {"rounds": host_rounds, "first_run_us": host_s * 1e6, **host}}
    res["speedup_vs_host_bisection"] = res["host_bisection"]["us_median"] / res["call"]["us_median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_scale_headroom.json"))
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    eng = Engine(0)
    t = synth.make("C3", 1.0, seed=synth.SEED)
    reqs = t.place_requests()
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    res = {"gpu_info": gpu_info(), "world": {"nodes": int(len(t.nodes)), "domains": int(t.n_domains),
                                             "requests": int(len(reqs)), "namespaces": int(t.n_namespaces)}}
    for name, wc in (("C3_no_ceiling", False), ("C3_ceiling_replicas_plus_8", True)):
        r = run(eng, t, wc, args.repeats)
        res[name] = r
        print(name, json.dumps({k: v for k, v in r.items() if k != "kernels"}), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
