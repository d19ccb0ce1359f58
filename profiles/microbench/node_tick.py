"""C3 resident tick at 1 % churn (pod rows and placement requests) with node events, four cases alternating
window by window in one process:

  (a) no node events;
  (b) 100 node capacity patches per tick (LWSE_TABLE_NODES segment; the node index is kept);
  (c) (b) plus 4 cordons / uncordons per tick: every tick's round rebuilds the node index on the device;
  (d) the events of (c) applied the way they had to be before node patches: lwse_upload_nodes of the whole
      node table between ticks (it drains the ticks in flight, drops the tick graphs and rebuilds the index).

Per case: the synchronous tick (lwse_resident_tick, wall clock around a call that returns after the device
finished) and the pipelined tick (two in flight; in (d) every upload drains the tick before it).  Every case's
final placement rows and group rows are checked against the oracle on the same rows; the card's name and
power limit are read in the same call.

    python profiles/microbench/node_tick.py --out /tmp/node_tick.json
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

import numpy as np  # noqa: E402

from lws_b200 import churn, synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402

N_CAPACITY = 100  # capacity patches per tick
N_CORDON = 4      # cordons / uncordons per tick (cases c, d)


def node_sets(nodes: np.ndarray, n_sets: int, cordons: bool, seed: int) -> list:
    """[(rows, values)] per tick; a cycle of the sets leaves every node schedulable as it started (a tick
    cordons N_CORDON nodes and the next one uncordons them), capacities are drawn anew."""
    rng = np.random.default_rng(seed)
    cur = nodes.copy()
    out = []
    cordoned = None
    sched = np.flatnonzero(cur["flags"] & R.NODE_SCHEDULABLE)
    for k in range(n_sets):
        rows = set(rng.choice(len(cur), size=N_CAPACITY, replace=False).tolist())
        vals = {r: cur[r].copy() for r in rows}
        for r in rows:
            vals[r]["capacity"] = int(rng.integers(0, 16))
        if cordons:
            if cordoned is None:
                cordoned = rng.choice(sched, size=N_CORDON, replace=False).tolist()
                flip = lambda v: v & ~np.uint16(R.NODE_SCHEDULABLE)  # noqa: E731
            else:
                flip = lambda v: v | np.uint16(R.NODE_SCHEDULABLE)  # noqa: E731
            for r in cordoned:
                v = vals.setdefault(r, cur[r].copy())
                v["flags"] = flip(v["flags"])
            cordoned = None if k % 2 else cordoned
        order = sorted(vals)
        rr = np.array(order, dtype=np.uint32)
        vv = R.aligned_empty(len(order), R.NODE_REC)
        for i, r in enumerate(order):
            vv[i] = vals[r]
        cur[rr] = vv
        out.append((rr, vv))
    assert n_sets % 2 == 0
    return out


class Case:
    def __init__(self, name, eng, t, reqs, flags, plan, nodes_k, upload):
        self.name, self.eng, self.t, self.reqs, self.flags = name, eng, t, reqs, flags
        self.plan, self.nodes_k, self.upload = plan, nodes_k, upload
        self.cur = R.aligned_empty(len(t.nodes), R.NODE_REC)  # case d: the node table it uploads

    def load(self):  # every timing window starts from the loaded tables, with whole plan cycles
        e, t = self.eng, self.t
        e.upload_nodes(t.nodes, t.n_domains)
        e.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
        e.resident_place_load(self.reqs, t.n_namespaces)
        self.ticks = self._arena_ticks()
        e.resident_tick(e.make_tick((), self.flags))
        self.cur[:] = t.nodes
        self.i = 0

    def _arena_ticks(self):
        """The churn plan's segments, plus (cases b, c) the node segment of the same tick, in the arena."""
        n_ticks = len(self.nodes_k) if self.nodes_k else len(self.plan)  # (a multiple of the plan's length)
        arrays = []
        for k in range(n_ticks):
            ps = self.plan[k % len(self.plan)]
            a = [ps.pod_rows, ps.pod_vals, ps.req_rows, ps.req_vals, ps.grp_rows, ps.grp_vals]
            if self.nodes_k and not self.upload:
                a += list(self.nodes_k[k % len(self.nodes_k)])
            arrays.append(a)
        need = 4096 + sum(((x.nbytes + 255) // 256 + 1) * 256 for a in arrays for x in a)
        arena = self.eng.resident_arena(need)
        cursor = 0

        def put(x):
            nonlocal cursor
            off = (cursor + 255) // 256 * 256
            view = arena[off: off + x.nbytes].view(x.dtype)
            view[...] = x
            cursor = off + x.nbytes
            return view

        ticks = []
        for k in range(n_ticks):
            ps = self.plan[k % len(self.plan)]
            segs = [(R.TABLE_POD_STATE, put(ps.pod_rows), put(ps.pod_vals))]
            if len(ps.grp_rows):
                segs.append((R.TABLE_GROUPS, put(ps.grp_rows), put(ps.grp_vals)))
            if len(ps.req_rows):
                segs.append((R.TABLE_PLACE_REQS, put(ps.req_rows), put(ps.req_vals)))
            if self.nodes_k and not self.upload:
                rr, vv = self.nodes_k[k % len(self.nodes_k)]
                segs.append((R.TABLE_NODES, put(rr), put(vv)))
            ticks.append(self.eng.make_tick(segs, self.flags))
        return ticks

    def _before(self):  # case d: the node events of this tick, by a whole-table upload
        if self.upload:
            rr, vv = self.nodes_k[self.i % len(self.nodes_k)]
            self.cur[rr] = vv
            self.eng.upload_nodes(self.cur, self.t.n_domains)

    def serial(self, n):
        t0 = time.perf_counter()
        for _ in range(n):
            self._before()
            self.eng.resident_tick(self.ticks[self.i % len(self.ticks)])
            self.i += 1
        return (time.perf_counter() - t0) / n

    def pipelined(self, n):
        t0 = time.perf_counter()
        in_flight = 0
        for _ in range(n):
            self._before()
            if self.upload:
                in_flight = 0  # (the upload drained the tick in flight)
            if in_flight == 2:
                self.eng.resident_tick_wait()
                in_flight -= 1
            self.eng.resident_tick_submit(self.ticks[self.i % len(self.ticks)])
            self.i += 1
            in_flight += 1
        for _ in range(in_flight):
            self.eng.resident_tick_wait()
        return (time.perf_counter() - t0) / n

    def check(self) -> bool:
        import oracle

        t = self.t
        m = self.reqs.copy()
        pst, grp = t.pod_state.copy(), t.groups.copy()
        nodes = t.nodes.copy()
        for k in range(self.i):
            churn.apply_to_mirror(self.plan[k % len(self.plan)], pst, grp, m)
            if self.nodes_k:
                rr, vv = self.nodes_k[k % len(self.nodes_k)]
                nodes[rr] = vv
        occ = R.occupancy_of(t.pod_ident, len(t.nodes))
        want_p = oracle.place(nodes, occ, t.n_domains, t.n_namespaces, m, threads=16)
        _, want_g, _ = oracle.sweep_lws(t.lws, grp, pst, t.pod_ident, nodes, flags=t.flags, threads=16)
        return (self.eng.resident_place_outputs().tobytes() == want_p.tobytes()
                and self.eng.resident_outputs()[1].tobytes() == want_g.tobytes())


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    t = synth.make("C3", 1.0, seed=synth.SEED)
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    flags = t.flags | R.TICK_PLACE
    reqs = t.place_requests()
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), flags))
    plan = churn.make_plan(t, reqs, eng.resident_place_outputs(), 0.01, 0.01)
    n_sets = len(plan) if len(plan) % 2 == 0 else 2 * len(plan)
    cap_only = node_sets(t.nodes, n_sets, False, 5)
    cordon = node_sets(t.nodes, n_sets, True, 5)
    cases = {
        "a_no_node_events": Case("a", eng, t, reqs, flags, plan, None, False),
        "b_capacity_patches": Case("b", eng, t, reqs, flags, plan, cap_only, False),
        "c_capacity_and_cordon_patches": Case("c", eng, t, reqs, flags, plan, cordon, False),
        "d_upload_nodes_between_ticks": Case("d", eng, t, reqs, flags, plan, cordon, True),
    }
    out = {name: {"serial_ms": [], "pipelined_ms": []} for name in cases}
    for rep in range(args.repeats):
        for name, c in cases.items():  # alternating, window by window
            c.load()
            c.serial(8)
            out[name]["serial_ms"].append(c.serial(args.steps) * 1e3)
            c.pipelined(8)
            out[name]["pipelined_ms"].append(c.pipelined(args.steps) * 1e3)
            out[name]["tick_info"] = eng.resident_tick_info()
            out[name]["node_info"] = eng.resident_node_info()
            if rep == args.repeats - 1:  # (before the next case loads its tables)
                out[name]["rows_equal_oracle"] = c.check()
    for name in cases:
        for k in ("serial_ms", "pipelined_ms"):
            v = out[name][k]
            out[name][k + "_median"] = float(np.median(v))
            out[name][k + "_spread"] = [float(min(v)), float(max(v))]
    out["config"] = {"workload": "C3", "scale": 1.0, "churn_pods": 0.01, "churn_reqs": 0.01, "capacity_patches": N_CAPACITY,
                     "cordons": N_CORDON, "steps": args.steps, "repeats": args.repeats, "n_nodes": int(len(t.nodes)),
                     **gpu_info()}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
