"""Drain budget (lwse_resident_drain_budget*) without a GPU: the per-key form restated in numpy
(tests/drain_budget_ref.py) against the set form by its definition — the spec oracle's what-if of that node or of
that domain's nodes — on small worlds and on a world where floors bind; the floor at maxUnavailable's edges;
the verdict flags; nodes without a domain; the informer's helpers; the record layouts against lwse.h."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from drain_budget_ref import (budget_row_of_cost, budget_world, budgets, domain_nodes, drain_budget_cost_ref,
                              drain_budget_ref, min_margin_of, owners)
from drain_ref import special_tables
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def _world(name):
    """(lws, groups, pst, pid, nodes, n_domains, sweep flags)."""
    if name == "special":
        lws, groups, pst, pid, nodes = special_tables()
        nodes = nodes.copy()
        nodes["domain_id"][6] = R.NONE   # a node in no domain
        nodes["domain_id"][7] = 9        # a domain id beyond n_domains
        return lws, groups, pst, pid, nodes, 4, 0
    if name == "breach":
        t = budget_world(n_lws=160, n_nodes=48, seed=5)
        return t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags & R.SWEEP_GANG
    from test_drain_whatif import _lifecycle_world, _node_world

    enc = _node_world() if name == "node" else _lifecycle_world()
    lws, groups, pst, pid, _ = enc.full_tables()
    return lws, groups, pst, pid, enc.node_rec, enc.n_domains, 0


@functools.lru_cache(maxsize=None)
def _base(name):
    lws, groups, pst, pid, nodes, _, flags = _world(name)
    return oracle.sweep_lws(lws, groups, pst, pid, nodes, flags)[:2]


WORLDS = ["special", "node", "lifecycle", "breach"]


def check_key(row, rows, totals, where):
    for k, v in budget_row_of_cost(row).items():
        assert totals[k] == v, (where, k)
    assert int(row["min_margin"]) == min_margin_of(rows), where
    assert len(rows) == totals["n_touched"]


@pytest.mark.parametrize("by_domain", [False, True], ids=["nodes", "domains"])
@pytest.mark.parametrize("name", WORLDS)
def test_per_key_equals_the_set_form(name, by_domain):
    """Every per-node (per-domain) row == the set form of that node (of that domain's nodes)."""
    lws, groups, pst, pid, nodes, n_domains, flags = _world(name)
    base = _base(name)
    cost = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, n_domains, base[1], by_domain)
    assert len(cost) == (n_domains if by_domain else len(nodes))
    touched = 0
    for k in range(len(cost)):
        d = domain_nodes(nodes, n_domains, [k]) if by_domain else [k]
        rows, totals = drain_budget_ref(lws, groups, pst, pid, nodes, d, flags, base=base)
        check_key(cost[k], rows, totals, (name, k))
        touched += totals["n_touched"]
    if name != "special":  # (the special table's groups sit in no LWS range: they touch no object)
        assert touched > 0


def test_nodes_without_a_domain():
    """domain_id = NONE or >= n_domains: the node is in no domain row, and a domain drain never drains it."""
    lws, groups, pst, pid, nodes, n_domains, _ = _world("special")
    base = _base("special")
    assert list(domain_nodes(nodes, n_domains, range(n_domains))) == [0, 1, 2, 3, 4, 5]
    by_node = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, n_domains, base[1], False)
    by_dom = drain_budget_cost_ref(lws, base[0], groups, pst, pid, nodes, n_domains, base[1], True)
    assert by_dom["pods"].sum() == by_node["pods"][:6].sum() < by_node["pods"].sum()
    assert by_dom["leaders"].sum() == by_node["leaders"][:6].sum() < by_node["leaders"].sum()


def test_floor_at_max_unavailable_edges():
    """floor = max(0, replicas - mu), mu rounded down: 0, 1, replicas, above replicas, 33 % and 50 % of 3,
    0 % and 100 %; in the breach world every edge occurs."""
    cases = [(3, 0, False, 3), (3, 1, False, 2), (3, 3, False, 0), (3, 5, False, 0), (3, 33, True, 3),
             (3, 50, True, 2), (3, 100, True, 0), (3, 0, True, 3), (8, 25, True, 6), (4, 20, False, 0)]
    lws = R.aligned_empty(len(cases), R.LWS_REC)
    out = R.aligned_empty(len(cases), R.LWS_OUT)
    for i, (reps, mu, pct, _) in enumerate(cases):
        lws[i]["replicas"], lws[i]["max_unavailable"] = reps, mu
        lws[i]["flags"] = R.LWS_UNAVAIL_IS_PERCENT if pct else 0
    floor, *_ = budgets(lws, out, 0)
    assert floor.tolist() == [c[3] for c in cases]
    t_lws = _world("breach")[0]
    seen = {(int(r), int(m), bool(f & R.LWS_UNAVAIL_IS_PERCENT))
            for r, m, f in zip(t_lws["replicas"], t_lws["max_unavailable"], t_lws["flags"])}
    for reps, mu, pct, _ in [(3, 33, True, 0), (3, 50, True, 0), (3, 100, True, 0), (3, 0, True, 0), (4, 20, False, 0),
                             (3, 0, False, 0), (4, 1, False, 0)]:
        assert (reps, mu, pct) in seen


@pytest.mark.parametrize("bit", ["BAD_TABLE", "IRREGULAR", "RUP_ERROR", "STATUS_ERROR", "INTSTR_INVALID"])
def test_not_evaluated(bit):
    """Each excluding flag gives NOT_EVALUATED (floor 0) and counts in no total but n_touched."""
    lws, groups, pst, pid, nodes, n_domains, flags = _world("breach")
    lws_out, gout = _base("breach")
    lws_out = lws_out.copy()
    cost = drain_budget_cost_ref(lws, lws_out, groups, pst, pid, nodes, n_domains, gout, True)
    dom = int(np.argmax(cost["lws_breached"]))
    d = domain_nodes(nodes, n_domains, [dom])
    rows, _ = drain_budget_ref(lws, groups, pst, pid, nodes, d, flags, base=(lws_out, gout))
    victim = int(rows["lws"][np.flatnonzero(rows["flags"] & R.DRAINB_BREACHED)[0]])
    if bit == "INTSTR_INVALID":
        lws = lws.copy()
        lws["flags"][victim] |= R.LWS_INTSTR_INVALID
    else:
        lws_out["flags"][victim] |= getattr(R, "LOUT_" + bit)
    rows2, tot2 = drain_budget_ref(lws, groups, pst, pid, nodes, d, flags, base=(lws_out, gout))
    r = rows2[rows2["lws"] == victim]
    assert len(r) == 1 and r["flags"][0] == R.DRAINB_NOT_EVALUATED and r["floor"][0] == 0
    assert tot2["n_breached"] == int(((rows["flags"] & R.DRAINB_BREACHED) != 0).sum()) - 1
    cost2 = drain_budget_cost_ref(lws, lws_out, groups, pst, pid, nodes, n_domains, gout, True)
    check_key(cost2[dom], rows2, tot2, bit)


def test_verdicts_in_the_breach_world():
    """ALREADY_BELOW with and without a touch, BREACHED, LOSES_AVAILABLE only through groups below replicas."""
    lws, groups, pst, pid, nodes, n_domains, flags = _world("breach")
    lws_out, gout = _base("breach")
    floor, ready, evaluated, available, gb, _ = budgets(lws, lws_out, len(groups))
    below = evaluated & (ready < floor)
    assert below.sum() > 5
    seen = {"below_touched": 0, "below_untouched": 0, "breached": 0, "loses": 0}
    own = owners(lws, groups)
    for dom in range(n_domains):
        rows, tot = drain_budget_ref(lws, groups, pst, pid, nodes, domain_nodes(nodes, n_domains, [dom]), flags,
                                     base=(lws_out, gout))
        assert tot["n_already_below"] == int(below.sum())
        t = (rows["flags"] & R.DRAINB_ALREADY_BELOW) != 0
        seen["below_touched"] += int(t.sum())
        seen["below_untouched"] += int(below.sum()) - int(t.sum())
        seen["breached"] += tot["n_breached"]
        seen["loses"] += tot["n_loses_available"]
        wf_after = None
        for r in rows:
            L = int(r["lws"])
            if not available[L] or not evaluated[L] or r["ready_after"] == r["ready_before"]:
                continue
            if wf_after is None:
                from drain_ref import drain_whatif_ref

                wf_after = drain_whatif_ref(lws, groups, pst, pid, nodes, domain_nodes(nodes, n_domains, [dom]), flags,
                                            base=(lws_out, gout))["after_all"]
            g = np.flatnonzero(own == L)
            hit = ((gout["flags"][g] & (R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING)) == 0) & \
                  ((wf_after["flags"][g] & (R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING)) != 0) & \
                  ((gout["flags"][g] & R.GOUT_COND_READY) != 0)
            low = (g[hit] - gb[L]) < lws["replicas"][L]
            assert bool(r["flags"] & R.DRAINB_LOSES_AVAILABLE) == bool(low.any())
    for k in ("below_touched", "below_untouched", "breached", "loses"):
        assert seen[k] > 0, (k, seen)


def test_informer_helpers():
    from test_drain_whatif import _node_world

    enc = _node_world()
    vals = sorted(enc._domain_ids)[:2]
    ids = enc.whatif_drain_domains(vals + vals[:1])
    assert ids.dtype == np.uint32 and ids.tolist() == sorted({enc._domain_ids[v] for v in vals})
    with pytest.raises(KeyError):
        enc.whatif_drain_domains(["no-such-value"])
    row = next(iter(enc._lws_key))
    res = {"rows": np.zeros(2, R.DRAIN_BUDGET)}
    res["rows"]["lws"] = [row, len(enc.lws) - 1]
    res["rows"]["flags"][0] = R.DRAINB_BREACHED | R.DRAINB_LOSES_AVAILABLE
    rep = enc.drain_budget_report(res)
    assert (rep[0]["namespace"], rep[0]["name"]) == enc.object_of_lws_row(row)
    assert rep[0]["conditions"] == ["breached", "loses_available"] and rep[0]["lws"] == row
    assert enc.object_of_lws_row(len(enc.lws) - 1) is None or rep[1]["name"] is not None


def test_records_match_header():
    """Sizes and offsets of lwse_drain_budget, lwse_drain_budget_query and lwse_drain_budget_cost, via a
    gcc-compiled probe."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){"]
    for s, names in (("lwse_drain_budget", R.DRAIN_BUDGET.names), ("lwse_drain_budget_cost", R.DRAIN_BUDGET_COST.names),
                     ("lwse_drain_budget_query", [f for f, _ in R.DrainBudgetQuery._fields_])):
        lines.append(f'printf("{s} %zu\\n", sizeof({s}));')
        for f in names:
            lines.append(f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));')
    lines.append('printf("scopes %u %u\\n", LWSE_DRAIN_NODES, LWSE_DRAIN_DOMAINS);')
    lines.append('printf("flags %u %u %u %u\\n", LWSE_DRAINB_NOT_EVALUATED, LWSE_DRAINB_BREACHED, '
                 'LWSE_DRAINB_ALREADY_BELOW, LWSE_DRAINB_LOSES_AVAILABLE);')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = {l.split(" ", 1)[0]: l.split(" ", 1)[1] for l in out.strip().splitlines()}
    assert int(got["lwse_drain_budget"]) == R.DRAIN_BUDGET.itemsize == 32
    assert int(got["lwse_drain_budget_cost"]) == R.DRAIN_BUDGET_COST.itemsize == 48
    for f in R.DRAIN_BUDGET.names:
        assert int(got[f"lwse_drain_budget.{f}"]) == R.DRAIN_BUDGET.fields[f][1], f
    for f in R.DRAIN_BUDGET_COST.names:
        assert int(got[f"lwse_drain_budget_cost.{f}"]) == R.DRAIN_BUDGET_COST.fields[f][1], f
    assert R.DRAIN_BUDGET_COST.fields["pods_recreated"][1] == R.DRAIN_COST.fields["pods_recreated"][1]
    assert int(got["lwse_drain_budget_query"]) == C.sizeof(R.DrainBudgetQuery)
    for f, _ in R.DrainBudgetQuery._fields_:
        assert int(got[f"lwse_drain_budget_query.{f}"]) == getattr(R.DrainBudgetQuery, f).offset, f
    assert got["scopes"] == f"{R.DRAIN_NODES} {R.DRAIN_DOMAINS}"
    assert got["flags"] == (f"{R.DRAINB_NOT_EVALUATED} {R.DRAINB_BREACHED} {R.DRAINB_ALREADY_BELOW} "
                            f"{R.DRAINB_LOSES_AVAILABLE}")
