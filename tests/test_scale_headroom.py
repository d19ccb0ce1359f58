"""Scale headroom (lwse_resident_scale_headroom) without a GPU: the device's bisection against the literal definition
(every R solved over every namespace) on seeded fuzz worlds and the edge worlds, each edge on its side, the wrong
statements caught, the settled claim against the forecast reference, the informer helpers and the records."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from lws_b200 import records as R
from rollout_place_ref import fuzz_world
from rollout_whatif_ref import rollout_whatif
from scale_headroom_ref import edge_queries, extra_groups, fuzz_query, headroom_world, scale_headroom_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASKS = (R.RPW_STRANDED, R.RPW_ALL)


@pytest.fixture(scope="module")
def worlds():
    return {fa: headroom_world(fa) for fa in (False, True)}


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("mask", MASKS)
def test_bisection_equals_the_definition_on_fuzz_worlds(seed, mask):
    w = fuzz_world(seed)
    rows, ns, ceil = fuzz_query(w, seed)
    for c in (None, ceil):
        a = scale_headroom_ref(w, rows, ns, c, mask)
        b = scale_headroom_ref(w, rows, ns, c, mask, mode="literal")
        assert a["rows"].tobytes() == b["rows"].tobytes()
        assert a["n_solved"] > 0


@pytest.mark.parametrize("fit_all", [False, True])
@pytest.mark.parametrize("mask", MASKS)
def test_bisection_equals_the_definition_on_the_edge_worlds(worlds, fit_all, mask):
    w, rows = worlds[fit_all]
    rr, nn, cc, _ = edge_queries(w, rows)
    for c in (None, cc):
        a = scale_headroom_ref(w, rr, nn, c, mask)
        b = scale_headroom_ref(w, rr, nn, c, mask, mode="literal")
        assert a["rows"].tobytes() == b["rows"].tobytes()


def _by_label(w, rows, mask, fit_all=False):
    rr, nn, cc, labels = edge_queries(w, rows)
    return dict(zip(labels, scale_headroom_ref(w, rr, nn, cc, mask)["rows"]))


def test_each_edge_lands_on_its_side(worlds):
    w, rows = worlds[False]
    s = _by_label(w, rows, R.RPW_STRANDED)
    b = _by_label(w, rows, R.RPW_ALL)
    # three fitting domains in the empty namespace: r0 + 3, the fourth group strands; a second object alike
    for k in ("k_fits", "k_fits_other", "ceiling_above_h"):
        assert (s[k]["max_replicas"], s[k]["probe"], s[k]["stranded"]) == (6, 7, 1) and s[k]["flags"] & R.SHR_STRANDS
    # ceilings: clean (the same row again), equal to r0 and below r0
    assert (s["k_fits_twice_ceiling"]["max_replicas"], s["k_fits_twice_ceiling"]["flags"]) == (4, R.SHR_SOLVED | R.SHR_AT_CEILING)
    for k in ("ceiling_at_r0", "ceiling_below_r0"):
        assert s[k]["max_replicas"] == 3 and s[k]["flags"] == R.SHR_SOLVED | R.SHR_AT_CEILING and s[k]["surge"] == 0
    # headroom 0: the object's own namespace has no free domain
    assert (s["headroom_0"]["max_replicas"], s["headroom_0"]["replicas"]) == (3, 3)
    # three holders: bumping them is allowed under STRANDED alone, not with BUMPED
    assert s["holders"]["max_replicas"] == 6 and b["holders"]["max_replicas"] == 3
    assert b["holders"]["bumped"] == 1 and b["holders"]["flags"] & R.SHR_BUMPS
    # a missing leader below group_count is extra at r0: one domain less; in the crowded namespace r0 is BLOCKED
    assert s["missing_leader"]["max_replicas"] == 5
    assert s["blocked"]["flags"] & R.SHR_BLOCKED and s["blocked"]["max_replicas"] == -1 and s["blocked"]["probe"] == 3
    # group rows in [r0, group_count): a present group 2 is free, a missing one is extra
    assert s["below_gc_present"]["max_replicas"] == 6 and s["below_gc_missing"]["max_replicas"] == 5
    # the object's own unpinned rows hold the fitting domains: with BUMPED, r0 + 1 takes one of them (own_lost)
    assert b["own_A"]["max_replicas"] == 3 and b["own_A"]["own_lost"] == 1 and b["own_A"]["bumped"] == 0
    assert s["own_A"]["max_replicas"] > 3
    for k, f in (("updated", R.SHR_NOT_SETTLED), ("rolling", R.SHR_NOT_SETTLED), ("held", R.SHR_NOT_SETTLED),
                 ("scaling", R.SHR_NOT_SETTLED), ("uf", R.SHR_NOT_SETTLED), ("not_exclusive", R.SHR_NOT_EXCLUSIVE)):
        assert s[k]["flags"] == f and (s[k]["max_replicas"], s[k]["probe"]) == (-1, -1), k
    assert s["not_forecast"]["flags"] & R.SHR_NOT_FORECAST
    # every domain fits: the bisection ends at R_pig - 1 = r0 + n_domains, and the final round probes R_pig
    wf, rf = worlds[True]
    f = _by_label(wf, rf, R.RPW_STRANDED)["k_fits"]
    assert (f["max_replicas"], f["probe"], f["surge"], f["stranded"]) == (3 + wf.n_domains, 4 + wf.n_domains, wf.n_domains + 1, 1)
    assert not f["flags"] & R.SHR_AT_CEILING


def test_one_solve_at_the_bound_is_wrong_on_the_priority_world(worlds):
    """E(C) strands a group that E(g + 1) places: the first stranded group of the bound's solve is not H + 1."""
    w, rows = worlds[False]
    r = rows["A"]
    a = scale_headroom_ref(w, [r], [2])["rows"][0]
    x = scale_headroom_ref(w, [r], [2], variant="bound_once")["rows"][0]
    assert a["max_replicas"] == 6 and x["max_replicas"] != a["max_replicas"]


def test_no_settled_check_disagrees_with_the_rollout_placement(worlds):
    """Answering the held and mid-rollout objects as if settled gives rows that the rollout placement of P(R) (the
    rollout what-if's forecast) contradicts."""
    w, rows = worlds[False]
    wrong = 0
    for k in ("held", "rolling", "updated"):
        r = rows[{"held": "S3", "rolling": "S2", "updated": "S1"}[k]]
        x = scale_headroom_ref(w, [r], [2], variant="no_settled")["rows"][0]
        assert x["flags"] & R.SHR_SOLVED
        h = int(x["max_replicas"])
        rec = R.aligned_empty(2, R.LWS_REC)
        rec[:] = w.lws[r]
        rec["replicas"] = [max(h, 0), h + 1]
        fc = rollout_whatif(w, [r, r], rec, steps=False)["lws"]
        wrong += int(any(int(fc["peak_sts_replicas"][j]) != int(rec["replicas"][j]) for j in range(2)))
    assert wrong > 0


def test_bumped_without_own_lost_is_wrong(worlds):
    w, rows = worlds[False]
    a = scale_headroom_ref(w, [rows["A"]], [5], constraints=R.RPW_ALL)["rows"][0]
    x = scale_headroom_ref(w, [rows["A"]], [5], constraints=R.RPW_ALL, variant="bumped_no_own")["rows"][0]
    assert a["own_lost"] > 0 and a["bumped"] == 0 and x["max_replicas"] > a["max_replicas"]


@pytest.mark.parametrize("world", ["edge", "fuzz"])
def test_settled_rows_forecast_peak_r(worlds, world):
    """The claim that makes E(R) the rollout placement's E of P(R): on every SOLVED entry, for every R in
    [r0, min(C_i, r0 + 16)], the rollout what-if's forecast of the scale-only edit has peak R."""
    if world == "edge":
        w, rows = worlds[False]
        rr, nn, cc, _ = edge_queries(w, rows)
    else:
        w = fuzz_world(2)
        rr = np.arange(len(w.lws), dtype=np.uint32)
        nn, cc = np.full(len(rr), 2, np.uint32), None
    out = scale_headroom_ref(w, rr, nn, cc)["rows"]
    q = []
    for i in np.flatnonzero((out["flags"] & R.SHR_SOLVED) != 0):
        r0 = int(out["replicas"][i])
        top = max(int(out["probe"][i]), int(out["max_replicas"][i]))
        q += [(int(rr[i]), R_) for R_ in range(r0, min(top, r0 + 16) + 1)]
    assert len(q) > 20
    recs = R.aligned_empty(len(q), R.LWS_REC)
    for j, (r, R_) in enumerate(q):
        recs[j] = w.lws[r]
        recs[j]["replicas"] = R_
    fc = rollout_whatif(w, [r for r, _ in q], recs, steps=False)["lws"]
    assert fc["peak_sts_replicas"].tolist() == [R_ for _, R_ in q]


def test_extra_rows_are_a_prefix():
    w = fuzz_world(1)
    for r in range(0, len(w.lws), 7):
        gs = [extra_groups(w, r, R_) for R_ in range(0, 12)]
        assert all(gs[k] == gs[k + 1][: len(gs[k])] for k in range(len(gs) - 1))


def test_informer_query_and_report():
    from informer_world import make_world

    from lws_b200 import informer

    items, cluster = make_world(3, n_lws=14, n_nodes=28)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    keys = sorted(k for k, sl in enc.slots.items() if int(enc.lws["flags"][sl.lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY)
    rows, ns, ceil = enc.scale_headroom_query(ceilings={keys[0]: 9})
    assert rows.tolist() == [enc.slots[k].lws_row for k in keys] and ceil.tolist() == [9] + [-1] * (len(keys) - 1)
    assert ns.tolist() == [enc.ns_ids[k[0]] for k in keys]
    out = np.zeros(len(rows), R.SCALE_HEADROOM)
    out["flags"] = R.SHR_SOLVED | R.SHR_STRANDS
    out["replicas"], out["max_replicas"] = 2, 5
    out["flags"][0] = R.SHR_SOLVED | R.SHR_AT_CEILING
    out["flags"][-1] = R.SHR_NOT_SETTLED
    out["max_replicas"][-1] = -1
    rep = enc.scale_headroom_report({"rows": out, "lws_rows": rows})
    assert (rep[0]["namespace"], rep[0]["name"], rep[0]["limit"], rep[0]["headroom"]) == (*keys[0], "ceiling", 3)
    assert rep[1]["limit"] == "strands" and rep[1]["max_replicas"] == 5
    assert rep[-1]["headroom"] is None and rep[-1]["flags"] == ["not_settled"]


def test_records_match_the_header():
    h = open(os.path.join(ROOT, "include", "lwse.h")).read()
    s = h[h.index("typedef struct lwse_scale_headroom {"):]
    s = s[: s.index("} lwse_scale_headroom;")]
    assert tuple(re.findall(r"^\s+u?int32_t (\w+);", s, re.M)) == R.SCALE_HEADROOM.names
    bits = re.findall(r"#define LWSE_SHR_(\w+) \(1u << (\d+)\)", h)
    assert len(bits) == len(R.SHR_NAMES)
    for name, bit in bits:
        assert getattr(R, "SHR_" + name) == 1 << int(bit)


def test_struct_layout_against_gcc():
    """sizeof and offsetof of the two new structs, compiled by gcc against lwse.h, equal the numpy / ctypes mirrors."""
    import ctypes as C

    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/lwse.h"', "int main(){"]
    lines.append('printf("%zu\\n", sizeof(lwse_scale_headroom));')
    for f in R.SCALE_HEADROOM.names:
        lines.append(f'printf("%zu\\n", offsetof(lwse_scale_headroom, {f}));')
    lines.append('printf("%zu\\n", sizeof(lwse_scale_headroom_query));')
    qf = [f for f, _ in R.ScaleHeadroomQuery._fields_]
    for f in qf:
        lines.append(f'printf("%zu\\n", offsetof(lwse_scale_headroom_query, {f}));')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [R.SCALE_HEADROOM.itemsize] + [R.SCALE_HEADROOM.fields[f][1] for f in R.SCALE_HEADROOM.names]
    want += [C.sizeof(R.ScaleHeadroomQuery)] + [getattr(R.ScaleHeadroomQuery, f).offset for f in qf]
    assert got == want


def test_guards_in_the_sources():
    src = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_engine.cu")).read()
    body = src[src.index("LWSE_API int lwse_resident_scale_headroom("):]
    body = body[: body.index("\n}\n")]
    assert "e->xch_world > 0 || e->rn_reqs >= (1u << 24)" in body
    assert re.search(r"\(uint64_t\)nr \+ max_extra >= \(1ull << 24\)\) return LWSE_ERR_UNSUPPORTED", body)
    assert body.index("max_extra >= (1ull << 24)") < body.index("memcpy(q->out")
