"""The rollout placement (lwse_resident_rollout_place) at C3 (100 000 objects, all exclusive, 10 000 nodes, 625
domains), resident rows, and at a C3-shaped world of 25 000 objects with 4 groups and maxSurge 2, asked with a
template bump on every object:

  - the call time (wall clock around a call that returns once the rows are in host memory);
  - the device time from CUDA events on the what-if stream (LWSE_WHATIF_TIMING=1; it includes the call's host
    synchronisations);
  - the per-kernel times of a torch.profiler run of its own;
  - the entries solved, the surge and stranded rows;
  - in the same process, the host composition (the forecast → the informer's extra rows → resident_place_whatif,
    one what-if per entry with extra rows) over every such entry, or a seeded sample (--sample; the count is
    recorded, and the per-entry cost is what the loop measured), and how many of its rows equal the call's.

The card's name and power limit are read in the same call.

    python profiles/microbench/rollout_place.py   # writes profiles/h100_rollout_place.json
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

COLS = ["surge", "placed", "stranded", "own_lost", "bumped", "n_changed", "n_lost", "n_moved", "n_gained", "n_placed",
        "n_unschedulable", "n_conflict", "namespaces_solved"]


def surge_world():
    """C3's nodes, domains, namespaces and group count, as 25 000 objects of 4 groups with maxSurge 2: a template
    bump then rolls each object with two surge groups (C3's objects have one group each, and maxSurge is clamped
    to replicas, so a bump of C3 itself adds none)."""
    p = synth.profile("C3", 1.0)
    p.name = "C3-r4-surge2"
    p.n_lws = 25_000
    p.replicas_choices = (4,)
    p.max_surge = ((2, False),)
    return synth.make(p, 1.0, seed=synth.SEED)


def run(eng, t, bump, sample, repeats, rng):
    from test_gpu_rollout_place import _REQS, composition

    reqs = t.place_requests()
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    rows = np.arange(len(t.lws), dtype=np.uint32)
    ns = t.ns_of_lws.astype(np.uint32)
    recs = None
    if bump:
        recs = R.aligned_empty(len(rows), R.LWS_REC)
        recs[:] = t.lws
        recs["rev_hash"] ^= np.uint64(0x5DEECE66D)
        recs["flags"] |= np.uint32(R.LWS_UPDATED)
    call = lambda: eng.resident_rollout_place(rows, ns, recs)
    for _ in range(3):
        got = call()
    out = got["rows"]
    r = {"objects": len(rows), "requests": len(reqs), "call": timed(call, 3, repeats),
         "device_us": event_device_us(eng, call, 5), "solved": int(got["n_solved"]), "surge_rows": int(got["n_surge"]),
         "stranded_rows": int(got["n_stranded"]), "entries_that_strand": int(got["n_strands"]),
         "entries_with_extra_rows": int((out["surge"] > 0).sum())}
    sel = np.flatnonzero(out["surge"] > 0)
    if sample and len(sel) > sample:
        sel = np.sort(rng.choice(sel, size=sample, replace=False))
    _REQS[id(eng)] = reqs
    t0 = time.perf_counter()
    want = composition(eng, t.lws, t.groups, rows[sel], ns[sel], None if recs is None else recs[sel])
    loop = time.perf_counter() - t0
    same = sum(all(out[i][c] == want[j][c] for c in COLS) for j, i in enumerate(sel.tolist()))
    r["composition"] = {"entries": int(len(sel)), "seconds": loop, "us_per_entry": loop / max(len(sel), 1) * 1e6,
                        "rows_equal": int(same)}
    r["kernels"] = kernel_profile(call, 3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_rollout_place.json"))
    ap.add_argument("--sample", type=int, default=2000, help="entries the composition loop runs (0: all)")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    rng = np.random.default_rng(11)
    eng = Engine(0)
    res = {"gpu_info": gpu_info()}
    for name, make, bump in (("C3_resident", lambda: synth.make("C3", 1.0, seed=synth.SEED), False),
                             ("C3_r4_surge2_template_bump", surge_world, True)):
        r = run(eng, make(), bump, args.sample, args.repeats, rng)
        res[name] = r
        print(name, json.dumps({k: v for k, v in r.items() if k != "kernels"}), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
