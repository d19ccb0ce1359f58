"""The placement explanation (lwse_resident_place_explain) at C3 (10 000 nodes, 625 domains, 98 072 requests).

  - four queries: (a) every row of the baseline that is not PLACED, listed (none at C3); (b) every row of the
    baseline, by mask; (c) every row of the what-if round with the nodes of one topology domain cordoned; (d) the
    what-if round with every domain from 24 on cordoned, every UNSCHEDULABLE or CONFLICT row;
  - per query the call (wall clock around a call that returns once the rows are in host memory), the device time
    of a call from CUDA events on the what-if stream (the engine records them with LWSE_WHATIF_TIMING=1: behind
    the snapshot event and after the explain kernel, the copies back not included), and the per-kernel times of
    a torch.profiler run of its own;
  - whether (a) and (d) equal the reference (tests/place_explain_ref.py) and the certificate holds on (b) and (c).

The card's name and power limit are read in the same call.

    python profiles/microbench/place_explain.py --out /tmp/place_explain.json
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

ALL = R.PLACE_PLACED | R.PLACE_PINNED | R.PLACE_CONFLICT | R.PLACE_UNSCHEDULABLE


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from place_explain_ref import certificate, cordon_seg, explain_ref
    from rollout_place_ref import world_of

    t = synth.make("C3", 1.0, seed=synth.SEED)
    w = world_of(t)
    eng = Engine(0)
    eng.upload_nodes(t.nodes, t.n_domains)
    eng.resident_load(t.lws, t.groups, t.pod_state, t.pod_ident)
    eng.resident_place_load(w.reqs, w.n_ns)
    eng.resident_tick(eng.make_tick((), t.flags | R.TICK_PLACE))
    base = eng.resident_place_outputs().copy()
    not_placed = np.flatnonzero((base["flags"] & R.PLACE_PLACED) == 0).astype(np.uint32)
    dom = int(np.bincount(t.nodes["domain_id"][t.nodes["domain_id"] < t.n_domains].astype(np.int64)).argmax())
    seg = cordon_seg(w.nodes, np.flatnonzero(w.nodes["domain_id"] == dom), cordon=True)
    queries = {
        "not_placed_listed": dict(rows=not_placed),
        "every_row_by_mask": dict(mask=ALL),
        "whatif_one_domain_cordoned_every_row": dict(segs=[seg], mask=ALL),
        "whatif_domains_24_up_cordoned": dict(segs=[cordon_seg(w.nodes, np.flatnonzero(w.nodes["domain_id"] >= 24), True)]),
    }
    torch.cuda.init()
    res = {"gpu": gpu_info(), "world": {"nodes": len(t.nodes), "domains": int(t.n_domains), "requests": len(w.reqs),
                                        "namespaces": int(w.n_ns), "cordoned_domain": dom}, "queries": {}}
    for name, kw in queries.items():
        fn = lambda kw=kw: eng.resident_place_explain(**kw)
        got = fn()
        for _ in range(3):
            fn()
        r = {"n_explained": int(got["n_explained"]), "classes": got["classes"], "flags": got["flags"],
             "call": timed(fn, args.calls, args.repeats), "device": event_device_us(eng, fn, args.calls * args.repeats),
             "kernels": kernel_profile(fn)}
        if kw.get("mask") == ALL:
            want = explain_ref(w, rows=[], segs=kw.get("segs", ()))
            r["certificate_violations"] = len(certificate({**want, "all_rows": got["rows"]}, w.n_ns, w.n_domains))
        else:
            want = explain_ref(w, **kw)
            r["equals_reference"] = bool(got["rows"].tobytes() == want["rows"].tobytes() and got["classes"] == want["classes"]
                                         and got["flags"] == want["flags"])
        res["queries"][name] = r
        print(name, r["n_explained"], f"call {r['call']['us_median']:.0f} us, device {r['device']['us_median']:.0f} us",
              {k: v for k, v in r.items() if k in ("equals_reference", "certificate_violations")}, flush=True)
    eng.close()
    out = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(out)
    else:
        print(out)


if __name__ == "__main__":
    main()
