"""The rollout placement waves (lwse_resident_rollout_place_waves), asked with a template bump on every exclusive
object:

  - C3 itself (100 000 objects of one group, 200 namespaces; a bump of C3 adds no group, so this is the setup and
    the rounds over keys without extra rows);
  - the C3-shaped world of profiles/microbench/rollout_place.py (25 000 objects of 4 groups, maxSurge 2);
  - the worst case R = n: the first 2 000 objects of that world, every entry in namespace 0, so that the rounds
    run one key at a time.

For each: the call time of the plan (wall clock around a call that returns once the answer is in host memory), the
call time of its setup alone (lwse_resident_rollout_place on the same query), the rounds R, the waves and the key
totals.  The card's name and power limit are read in the same call.

    python profiles/microbench/rollout_place_waves.py   # writes profiles/h100_rollout_place_waves.json
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

from ds_tick import gpu_info  # noqa: E402
from lws_b200 import synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402
from place_whatif import timed  # noqa: E402
from rollout_place import surge_world  # noqa: E402


def run(eng, t, n_keys, one_ns, repeats):
    reqs = t.place_requests()
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    rows = np.flatnonzero(t.lws["flags"] & R.LWS_EXCLUSIVE_TOPOLOGY)[:n_keys].astype(np.uint32)
    ns = np.zeros(len(rows), np.uint32) if one_ns else t.ns_of_lws[rows].astype(np.uint32)
    recs = R.aligned_empty(len(rows), R.LWS_REC)
    recs[:] = t.lws[rows]
    recs["rev_hash"] ^= np.uint64(0x5DEECE66D)
    recs["flags"] |= np.uint32(R.LWS_UPDATED)
    plan = lambda: eng.resident_rollout_place_waves(rows, ns, recs, constraints=R.RPW_ALL)
    setup = lambda: eng.resident_rollout_place(rows, ns, recs)
    got = plan()
    alone = setup()["rows"]
    solved = (alone["flags"] & R.RPL_SOLVED) != 0
    part = got["keys"]["status"] != R.ROLLW_NOT_SOLVED
    part &= got["keys"]["status"] != R.ROLLW_TRIGGERS_ALONE
    per_ns = np.bincount(ns[part].astype(np.int64)) if part.any() else np.zeros(1, np.int64)
    return {"objects": int(len(rows)), "requests": int(len(reqs)), "one_namespace": bool(one_ns),
            "rounds_R": int(per_ns.max()), "solved": int(solved.sum()), "surge_rows": int(alone["surge"][solved].sum()),
            "n_waves": int(got["n_waves"]), **{k: int(got[k]) for k in R.ROLLOUT_WAVES_TOTALS if k != "n_waves"},
            "wave_keys": got["waves"]["n_keys"].tolist(), "wave_surge": got["waves"]["surge"].tolist(),
            "plan_call": timed(plan, 2, repeats), "setup_call": timed(setup, 2, repeats)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_rollout_place_waves.json"))
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    eng = Engine(0)
    res = {"gpu_info": gpu_info()}
    for name, make, n_keys, one_ns in (("C3_template_bump", lambda: synth.make("C3", 1.0, seed=synth.SEED), None, False),
                                       ("C3_r4_surge2_template_bump", surge_world, None, False),
                                       ("C3_r4_surge2_one_namespace_2000", surge_world, 2000, True)):
        r = run(eng, make(), n_keys, one_ns, args.repeats)
        res[name] = r
        print(name, json.dumps(r), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
