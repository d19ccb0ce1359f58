"""Placement explanation (lwse_resident_place_explain) without a GPU: the reference of tests/place_explain_ref.py on
the edge world (each case on its side), the serial-order certificate on fuzz worlds and at C3 (baseline and what-if
rounds), the wrong statements it tells apart, the report helper on an informer world and the records against lwse.h
and gcc."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from lws_b200 import records as R
from place_explain_ref import (TIE, certificate, cordon_seg, edge_world, explain_ref, extra_reqs, fuzz_world, hi_of,
                               round_of)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = R.PLACE_PLACED | R.PLACE_PINNED | R.PLACE_CONFLICT | R.PLACE_UNSCHEDULABLE


@pytest.fixture(scope="module")
def edge():
    w, rows = edge_world()
    ans = explain_ref(w, rows=list(range(len(w.reqs))))
    return w, rows, {int(e["row"]): e for e in ans["all_rows"]}, ans


def test_edge_rows_land_on_their_side(edge):
    w, rows, e, ans = edge
    K, d1, d2 = TIE
    assert hi_of(K, d1) == hi_of(K, d2)
    x = lambda n: e[rows[n]]
    out = ans["round"]
    # the tie: T0 takes the lower domain, T1 the other; B's two blockers tie and the lower one is named
    assert int(out["domain_id"][rows["T0"]]) == d1 and int(x("T0")["best_domain"]) == d1 and int(x("T0")["n_held_later"]) == 1
    assert int(x("T1")["blocker_domain"]) == d1 and int(x("T1")["blocker_row"]) == rows["T0"]
    b = x("B")
    assert b["flags"] == R.PEX_EXCLUSIVE and int(b["n_held_earlier"]) == 2 and int(b["blocker_domain"]) == d1
    assert int(b["blocker_row"]) == int(np.flatnonzero((out["domain_id"] == d1) & (w.reqs["ns"] == 1))[0])
    # dom_free == s fits, s - 1 is the shortfall of 1; a cordoned node makes domain 3 too small, domain 4 has no
    # usable node: both would fit uncordoned
    f5 = x("F5")
    assert f5["flags"] == R.PEX_EXCLUSIVE | R.PEX_CORDONED and int(f5["n_fit_uncordoned"]) == 2
    assert (int(f5["shortfall"]), int(f5["shortfall_domain"])) == (1, 2)
    assert (int(f5["n_held_pinned"]), int(f5["n_held_earlier"]), int(f5["n_open"])) == (1, 3, 0)
    assert int(f5["n_no_usable"]) == 1 and int(f5["best_domain"]) == R.NONE
    # domain 1 (dom_free 5) is held by the pinned P1; P2 conflicts with it
    p2 = x("P2")
    assert p2["flags"] & R.PEX_CONFLICT and (int(p2["blocker_domain"]), int(p2["blocker_row"])) == (1, rows["P1"])
    assert x("P1")["flags"] & R.PEX_CONFLICT == 0 and int(x("P1")["n_own"]) == 1
    for n in ("NC_MISSING", "NC_UNLABELLED", "NC_RANGE"):
        assert x(n)["flags"] & R.PEX_NO_CLAIM
    for n in ("Z0", "ZN"):
        assert x(n)["flags"] & R.PEX_BAD_SIZE and int(x(n)["n_too_small"]) == 0
    # the occupancy above capacity counts 0, not negative: domain 5 has 8 free and fits
    assert int(out["domain_id"][rows["U3"]]) == 5 or 5 in [int(out["domain_id"][rows[n]]) for n in ("U1", "U2")]
    # a pinned leader on a cordoned node still holds its domain (own, though no node is usable)
    assert int(x("PC")["n_own"]) == 1 and int(x("PC")["n_no_usable"]) == 0
    # E1 sees the pinned holder as pinned, Q sees E1 as an earlier unpinned holder
    assert int(x("Q")["n_held_pinned"]) == 1 and int(x("Q")["n_held_earlier"]) == 1
    cap = x("CAP")
    assert cap["flags"] & R.PEX_CAPACITY and (int(cap["shortfall"]), int(cap["shortfall_domain"])) == (1, d1)
    assert x("NS")["flags"] == R.PEX_NO_NAMESPACE and sum(int(x("NS")[f]) for f in R.PLACE_EXPLAIN_CLASSES) == 0
    assert certificate(ans, w.n_ns, w.n_domains) == []


def test_totals_sum_the_rows(edge):
    w, rows, e, ans = edge
    got = ans["all_rows"]
    for f in R.PLACE_EXPLAIN_CLASSES:
        assert ans["classes"][f] == int(got[f].astype(np.int64).sum())
    assert ans["flags"]["capacity"] >= 1 and ans["flags"]["conflict"] == 1 and ans["flags"]["no_namespace"] == 1


def test_mask_selects_ascending_and_capacity_truncates(edge):
    w, rows, e, ans = edge
    m = explain_ref(w)
    sel = np.flatnonzero((m["round"]["flags"] & (R.PLACE_UNSCHEDULABLE | R.PLACE_CONFLICT)) != 0)
    assert m["rows"]["row"].tolist() == sel.tolist() and m["n_explained"] == len(sel) > 3
    c = explain_ref(w, capacity=3)
    assert c["n_explained"] == len(sel) and len(c["rows"]) == 3 and c["classes"] == m["classes"]


def test_whatif_rounds(edge):
    w, rows, e, ans = edge
    # uncordon domain 4 (a node-index rebuild): one more domain fits, and F5 places
    a = explain_ref(w, rows=[rows["F5"]], segs=[cordon_seg(w.nodes, [8, 9], cordon=False)])
    assert a["whatif"] and a["round"]["flags"][rows["F5"]] & R.PLACE_PLACED and int(a["rows"][0]["n_own"]) == 1
    assert int(a["rows"][0]["n_fit_uncordoned"]) == 1 and int(a["rows"][0]["n_no_usable"]) == 0
    # extra rows, one of them in a namespace the resident count does not have
    x = extra_reqs([(2, 5, 0), (4, 5, 0), (2, 9, 90)])
    b = explain_ref(w, rows=[len(w.reqs), len(w.reqs) + 1, len(w.reqs) + 2], extra=x, n_ns=5)
    assert b["round_rows"] == len(w.reqs) + 3 and certificate(b, 5, w.n_domains) == []
    assert b["rows"][1]["flags"] & R.PEX_NO_NAMESPACE == 0
    # extra rows only, on an empty request table
    empty = type(w)(**{**vars(w), "reqs": R.aligned_empty(0, R.PLACE_REQ)})
    c = explain_ref(empty, mask=ALL, extra=x[:2], n_ns=5)
    assert c["n_explained"] == 2 and all(int(r["n_open"]) + int(r["n_own"]) > 0 for r in c["rows"])


def test_general_form_domains(edge):
    """5 457 domains (beyond one CTA): the domains without nodes are no_usable; node 129 (domain 99) now counts."""
    w, rows, e, ans = edge
    big = type(w)(**{**vars(w), "n_domains": 5457})
    a = explain_ref(big, rows=[rows["F5"], rows["B"]])
    assert int(a["rows"][0]["n_no_usable"]) == int(e[rows["F5"]]["n_no_usable"]) + 5457 - 64 - 1
    assert certificate(a, w.n_ns, 5457) == []


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_certificate_on_fuzz_worlds(seed):
    w = fuzz_world(seed)
    a = explain_ref(w, mask=ALL)
    assert a["n_explained"] == len(w.reqs) and certificate(a, w.n_ns, w.n_domains) == []
    seg = cordon_seg(w.nodes, range(0, len(w.nodes), 7), cordon=True)
    b = explain_ref(w, mask=ALL, segs=[seg], extra=extra_reqs([(0, 3, 0), (1, 6, 1), (w.n_ns, 2, 0)]), n_ns=w.n_ns + 1)
    assert b["whatif"] and certificate(b, w.n_ns + 1, w.n_domains) == []
    for r in a["all_rows"]:
        if r["flags"] & R.PEX_NO_NAMESPACE == 0:
            assert sum(int(r[f]) for f in R.PLACE_EXPLAIN_CLASSES[:7]) == w.n_domains


def test_certificate_at_c3():
    from lws_b200 import synth
    from rollout_place_ref import world_of

    t = synth.make("C3", 1.0, seed=synth.SEED)
    w = world_of(t)
    a = explain_ref(w)  # every UNSCHEDULABLE and CONFLICT row: none in the C3 baseline
    placed = np.flatnonzero((a["round"]["flags"] & R.PLACE_PLACED) != 0)
    b = explain_ref(w, rows=placed[:: max(1, len(placed) // 1500)])
    assert certificate(b, w.n_ns, w.n_domains) == []
    # every domain from 24 on cordoned: thousands of rows strand, each EXCLUSIVE and CORDONED
    seg = cordon_seg(w.nodes, np.flatnonzero(w.nodes["domain_id"] >= 24), cordon=True)
    c = explain_ref(w, segs=[seg])
    assert c["n_explained"] > 1000 and certificate(c, w.n_ns, w.n_domains) == []
    assert c["flags"]["exclusive"] == c["flags"]["cordoned"] == c["n_explained"]


@pytest.mark.parametrize("variant", ["held_before_fit", "later_blocks", "capacity_not_free"])
def test_wrong_statements_give_other_rows(edge, variant):
    w, rows, e, ans = edge
    bad = explain_ref(w, rows=list(range(len(w.reqs))), variant=variant)
    assert bad["all_rows"].tobytes() != ans["all_rows"].tobytes()


def test_round_of_the_baseline_is_the_oracle(edge):
    w, rows, e, ans = edge
    base = round_of(w)
    same = round_of(w, n_ns=w.n_ns)
    assert not base[4] and not same[4] and base[2].tobytes() == same[2].tobytes()


def test_report_on_an_informer_world():
    from informer_world import make_world

    from lws_b200 import informer

    items, cluster = make_world(3, n_lws=14, n_nodes=28)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    reqs = enc.reqs[: enc.r_end]  # (the used rows; the table has spare rows beyond them)
    assert len(reqs) > 1
    g0 = enc.object_of_group_row(int(reqs["group"][0]))
    dom = sorted(enc._domain_ids.items(), key=lambda kv: kv[1])
    rows = np.zeros(3, R.PLACE_EXPLAIN)
    for f in ("best_domain", "blocker_domain", "blocker_row", "shortfall_domain"):
        rows[f] = R.NONE
    rows["row"] = [0, 0, len(reqs)]
    rows[0]["flags"] = R.PEX_EXCLUSIVE | R.PEX_CORDONED
    rows[0]["n_too_small"], rows[0]["n_fit_uncordoned"], rows[0]["n_no_usable"] = 2, 1, 0
    rows[0]["n_held_pinned"], rows[0]["n_held_earlier"] = 1, 1
    rows[0]["shortfall"], rows[0]["shortfall_domain"] = 2, dom[0][1]
    rows[0]["blocker_domain"], rows[0]["blocker_row"] = dom[-1][1], 0
    rows[1]["flags"] = R.PEX_NO_NAMESPACE
    rows[2]["n_open"] = 4
    result = {"rows": rows, "n_domains": 4, "round_rows": len(reqs) + 1}
    rep = enc.place_explain_report(result, extra_groups=[("ns-x", "new", 5)])
    # without extra_groups a row past the encoder's used request rows names no object, spare rows included
    assert len(enc.reqs) > enc.r_end
    spare = rows[2:].copy()
    spare["row"] = enc.r_end
    bare = enc.place_explain_report({**result, "rows": spare, "round_rows": len(enc.reqs) + 1})
    assert (bare[0]["namespace"], bare[0]["name"], bare[0]["group"]) == (None, None, None)
    assert (rep[0]["namespace"], rep[0]["name"], rep[0]["group"]) == g0
    assert rep[0]["message"] == (f"0/4 domains available: 2 too small, 0 without a usable node (1 of these would fit "
                                 f"with cordoned nodes), 2 held ahead in the namespace (1 pinned); 2 slots short in "
                                 f"{dom[0][0]}; would take {dom[-1][0]}, held by {g0[0]}/{g0[1]} group {g0[2]}")
    assert rep[0]["flags"] == ["exclusive", "cordoned"]
    assert rep[1]["message"] == "no such namespace"
    assert (rep[2]["namespace"], rep[2]["name"], rep[2]["group"]) == ("ns-x", "new", 5)
    assert rep[2]["message"].startswith("4/4 domains available")


def test_records_match_the_header():
    h = open(os.path.join(ROOT, "include", "lwse.h")).read()
    s = h[h.index("typedef struct lwse_place_explain_row {"):]
    s = s[: s.index("} lwse_place_explain_row;")]
    assert tuple(re.findall(r"^\s+u?int32_t (\w+);", s, re.M)) == R.PLACE_EXPLAIN.names
    bits = re.findall(r"#define LWSE_PEX_(\w+) \(1u << (\d+)\)", h)
    assert len(bits) == len(R.PEX_NAMES) == 7
    for name, bit in bits:
        assert getattr(R, "PEX_" + name) == 1 << int(bit)


def test_struct_layout_against_gcc():
    """sizeof and offsetof of the two new structs, compiled by gcc against lwse.h, equal the numpy / ctypes mirrors."""
    import ctypes as C

    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/lwse.h"', "int main(){"]
    lines.append('printf("%zu\\n", sizeof(lwse_place_explain_row));')
    for f in R.PLACE_EXPLAIN.names:
        lines.append(f'printf("%zu\\n", offsetof(lwse_place_explain_row, {f}));')
    lines.append('printf("%zu\\n", sizeof(lwse_place_explain_query));')
    qf = [f for f, _ in R.PlaceExplainQuery._fields_]
    for f in qf:
        lines.append(f'printf("%zu\\n", offsetof(lwse_place_explain_query, {f}));')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [R.PLACE_EXPLAIN.itemsize] + [R.PLACE_EXPLAIN.fields[f][1] for f in R.PLACE_EXPLAIN.names]
    want += [C.sizeof(R.PlaceExplainQuery)] + [getattr(R.PlaceExplainQuery, f).offset for f in qf]
    assert got == want
