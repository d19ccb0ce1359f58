"""C3 resident tick at 1 % churn on a request table grouped by namespace and on the same table made
ungrouped (1 % of the requests moved to tail rows, two namespaces interleaved — what creating and
deleting LeaderWorkerSets in place leaves behind).  The two alternate in one process.  Per case: the
synchronous tick (lwse_resident_tick, wall clock around a call
that returns after the device finished) and the pipelined tick (two in flight, as bench.py's headline).
Every case's final placement rows are checked against the spec oracle.

    python profiles/microbench/lifecycle_tick.py --out /tmp/lifecycle_tick.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from lws_b200 import churn, synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402


def ungroup(reqs):
    from test_gpu_lifecycle import ungroup as f

    return f(reqs)


class Case:
    def __init__(self, eng, t, reqs, flags):
        self.eng, self.t, self.reqs, self.flags = eng, t, reqs, flags
        eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        eng.resident_place_load(reqs, t.n_namespaces)
        eng.resident_tick(eng.make_tick((), flags))
        place = eng.resident_place_outputs()
        self.plan = churn.make_plan(t, reqs, place, 0.01, 0.01)
        self.i = 0

    def load(self):  # every timing window starts from the loaded tables, with whole plan cycles
        self.eng.resident_load(self.t.lws, self.t.groups, self.t.pod_state, self.t.pod_ident)
        self.eng.resident_place_load(self.reqs, self.t.n_namespaces)
        self.ap = churn.ArenaPlan(self.eng, self.plan, self.flags)
        self.eng.resident_tick(self.eng.make_tick((), self.flags))
        self.i = 0

    def serial(self, n):
        t0 = time.perf_counter()
        for _ in range(n):
            self.eng.resident_tick(self.ap.ticks[self.i % len(self.ap.ticks)])
            self.i += 1
        return (time.perf_counter() - t0) / n

    def pipelined(self, n):
        t0 = time.perf_counter()
        self.eng.resident_tick_submit(self.ap.ticks[self.i % len(self.ap.ticks)])
        self.i += 1
        for _ in range(n - 1):
            self.eng.resident_tick_submit(self.ap.ticks[self.i % len(self.ap.ticks)])
            self.i += 1
            self.eng.resident_tick_wait()
        self.eng.resident_tick_wait()
        return (time.perf_counter() - t0) / n

    def check(self):
        import oracle

        m = self.reqs.copy()
        pst, grp = self.t.pod_state.copy(), self.t.groups.copy()
        for k in range(self.i):
            churn.apply_to_mirror(self.plan[k % len(self.plan)], pst, grp, m)
        occ = R.occupancy_of(self.t.pod_ident, len(self.t.nodes))
        want = oracle.place(self.t.nodes, occ, self.t.n_domains, self.t.n_namespaces, m, threads=16)
        return self.eng.resident_place_outputs().tobytes() == want.tobytes()


def measure(cases: dict, steps: int, repeats: int) -> dict:
    out = {name: {"serial_ms": [], "pipelined_ms": [], "info": None} for name in cases}
    for rep in range(repeats):
        for name, c in cases.items():  # alternating, window by window
            c.load()
            c.serial(8)
            out[name]["serial_ms"].append(c.serial(steps) * 1e3)
            c.pipelined(8)
            out[name]["pipelined_ms"].append(c.pipelined(steps) * 1e3)
            out[name]["info"] = c.eng.resident_tick_info()
            if rep == repeats - 1:  # (before the next case loads its tables)
                out[name]["placement_equals_spec_oracle"] = c.check()
    for name in cases:
        for k in ("serial_ms", "pipelined_ms"):
            v = out[name][k]
            out[name][k + "_median"] = float(np.median(v))
    return out


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    t = synth.make("C3", 1.0, seed=synth.SEED)
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    flags = t.flags | R.TICK_PLACE
    reqs = t.place_requests()
    cases = {"grouped": Case(eng, t, reqs, flags), "ungrouped": Case(eng, t, ungroup(reqs), flags)}
    res = measure(cases, args.steps, args.repeats)
    res["config"] = {"workload": "C3", "scale": 1.0, "churn_pods": 0.01, "churn_reqs": 0.01, "steps": args.steps,
                     "repeats": args.repeats, "n_requests": int(len(reqs)), **gpu_info()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
