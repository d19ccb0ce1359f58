"""The linked DS tick (revision-role rows linked to resident child LeaderWorkerSets) against the unlinked
one, at C4, and its effect on the pipelined LeaderWorkerSet tick.

  (1) C4 (50 000 DisaggregatedSets, 2 roles), every existing revision-role row linked to a resident
      size-1 child LeaderWorkerSet, at 0.1 %, 1 % and 10 % revision-role churn per tick: the lone call
      (wall clock around a call that returns once its results are in pinned memory) and the device time
      of its kernels (torch.profiler CUDA activity records of a run of their own), unlinked and linked
      windows alternating in one process.  The linked sweep gathers the link row, the LWS row's uid word
      and the result row's ready and flags words for every revision-role row.
  (2) C3 pipelined LeaderWorkerSet ticks at 1 % churn (two in flight): alone, with an unlinked C4 DS tick
      between each submit and wait, and with a linked one (its rows linked to C3 LWS rows, so it waits
      for the LWS tick just submitted), alternating window by window.

The card's name and power limit are read in the same call; the linked DS mirrors are checked against
the oracle (ready counts substituted by the link rule) at the end of every churn level.

    python profiles/microbench/ds_link_tick.py --out /tmp/ds_link_tick.json
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

from ds_tick import gpu_info, revrole_sets  # noqa: E402
from lws_b200 import churn, synth  # noqa: E402
from lws_b200 import records as R  # noqa: E402
from lws_b200.engine import Engine  # noqa: E402

CHURN = (0.001, 0.01, 0.1)


def device_us(eng, sets, i, n_prof=50):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            rows, v = sets[i % len(sets)]
            eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
            i += 1
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            key = "ds_sweep_kernel" if "ds_sweep_kernel" in ev.name else ("scatter" if "scatter" in ev.name else
                                                                        ("memcpy" if "emcpy" in ev.name else ev.name[:40]))
            per[key] = per.get(key, 0.0) + ev.device_time_total
    return {k: v / n_prof for k, v in per.items()}, i


def ds_level(eng, d, links, lws, lws_out, frac, steps, repeats):
    import oracle
    from ds_link_world import linked_revroles

    sets = revrole_sets(d.revroles, frac, 8, seed=int(frac * 1e4) + 1)
    out = {}
    for linked in (False, True):
        out["linked" if linked else "unlinked"] = {"call_us": []}
    i = 0
    for _ in range(repeats):
        for linked in (False, True):
            eng.ds_resident_load(d.ds, d.roles, d.revroles)
            eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)] if linked else [])
            rr = d.revroles.copy()
            i = 0
            for _ in range(8):
                rows, v = sets[i % 8]
                eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
                i += 1
            t0 = time.perf_counter()
            for _ in range(steps):
                rows, v = sets[i % 8]
                res = eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
                i += 1
            out["linked" if linked else "unlinked"]["call_us"].append((time.perf_counter() - t0) / steps * 1e6)
            if linked:
                info = eng.ds_resident_tick_info()
                for k in range(i):
                    rr[sets[k % 8][0]] = sets[k % 8][1]
                sub, took, fell = linked_revroles(rr, links, lws, lws_out)
                want = oracle.sweep_ds(d.ds, d.roles, sub)
                ok = all(res[n].tobytes() == w.tobytes() for n, w in zip(("ds_out", "role_out", "revrole_out"), want))
                out["linked"]["mirrors_equal_oracle"] = bool(ok) and out["linked"].get("mirrors_equal_oracle", True)
                out["linked"]["rows_from_lws"], out["linked"]["rows_fallback"] = info["rows_from_lws"], info["rows_fallback"]
                assert (info["rows_from_lws"], info["rows_fallback"]) == (took, fell)
    for linked in (False, True):
        r = out["linked" if linked else "unlinked"]
        eng.ds_resident_load(d.ds, d.roles, d.revroles)
        eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, links, True)] if linked else [])
        r["device_us_per_tick"], _ = device_us(eng, sets, 0)
        r["device_us_total"] = float(sum(r["device_us_per_tick"].values()))
        r["call_us_median"] = float(np.median(r["call_us"]))
        r["call_us_spread"] = [min(r["call_us"]), max(r["call_us"])]
    out["rows_patched"] = int(len(sets[0][0]))
    return out


def main():
    import oracle

    from ds_link_world import child_lws_tables, none_links

    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    d = synth.make_ds(50_000, (2,))
    out = {"config": {"ds": len(d.ds), "roles": len(d.roles), "revroles": len(d.revroles), "steps": args.steps,
                      "repeats": args.repeats, **gpu_info()}}
    # (1) C4 alone, every existing revision-role row linked to a size-1 child
    lws, groups, pst, pid, links = child_lws_tables(d.revroles, np.random.default_rng(5))
    eng.resident_load(lws, groups, pst, pid)
    eng.resident_tick(eng.make_tick(()))
    lws_out = oracle.sweep_lws(lws, groups, pst, pid)[0]
    out["config"]["child_lws"] = len(lws)
    out["config"]["linked_rows"] = int((links["lws_row"] != R.NONE).sum())
    for frac in CHURN:
        out[f"ds_tick_churn_{frac:g}"] = ds_level(eng, d, links, lws, lws_out, frac, args.steps, args.repeats)
    # (2) C3 pipelined LWS ticks: alone, with an unlinked DS tick, with a linked one between submit and wait
    t = synth.make("C3", 1.0, seed=synth.SEED)
    eng.upload_nodes(t.nodes, t.n_domains)
    flags = t.flags | R.TICK_PLACE
    reqs = t.place_requests()
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(reqs, t.n_namespaces)
    eng.resident_tick(eng.make_tick((), flags))
    plan = churn.make_plan(t, reqs, eng.resident_place_outputs(), 0.01, 0.01)
    ticks = churn.ArenaPlan(eng, plan, flags).ticks
    ds_sets = revrole_sets(d.revroles, 0.01, 8, seed=77)
    rng = np.random.default_rng(9)
    c3_links = none_links(len(d.revroles))
    ex = np.flatnonzero(d.revroles["flags"] & R.RR_EXISTS)
    at = rng.integers(0, len(t.lws), size=len(ex))
    c3_links["lws_row"][ex] = at
    c3_links["lws_uid_hash"][ex] = t.lws["uid_hash"][at]
    state = {"i": 0, "j": 0}

    def window(n, ds_mode):
        if ds_mode:
            eng.ds_resident_load(d.ds, d.roles, d.revroles)
            eng.ds_resident_tick([(R.TABLE_DS_LINKS, 0, c3_links, True)] if ds_mode == "linked" else [])
        eng.resident_tick_submit(ticks[state["i"] % len(ticks)])
        state["i"] += 1
        t0 = time.perf_counter()
        for _ in range(n):
            eng.resident_tick_submit(ticks[state["i"] % len(ticks)])
            state["i"] += 1
            if ds_mode:
                rows, v = ds_sets[state["j"] % 8]
                eng.ds_resident_tick([(R.TABLE_DS_REVROLES, rows, v)])
                state["j"] += 1
            eng.resident_tick_wait()
        dt = (time.perf_counter() - t0) / n
        eng.resident_tick_wait()
        return dt * 1e6

    modes = (("lws_only_us", None), ("lws_with_ds_tick_us", "unlinked"), ("lws_with_linked_ds_tick_us", "linked"))
    res = {name: [] for name, _ in modes}
    graphs = {}
    for _ in range(args.repeats):
        for name, mode in modes:
            window(8, mode)
            res[name].append(window(args.steps, mode))
            graphs[name] = eng.resident_tick_info()["graph"]
    for name in list(res):
        res[name + "_median"] = float(np.median(res[name]))
    res["graph_on_steady_ticks"] = graphs
    res["linked_rows_from_lws"] = eng.ds_resident_tick_info()["rows_from_lws"]
    out["c3_pipelined_lws_tick"] = res
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
