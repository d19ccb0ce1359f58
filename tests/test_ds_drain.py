"""The DS drain without a GPU (lwse.h, "DS drain"): the per-key restatement equals the set form for every node and
every domain of several worlds, the named cases of the definition one by one, the (DS, key) table sizes, the record
layouts against the header, and the informer's report."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ds_drain_ref import (COST_FIELDS, World, cost_row_of, ds_drain_cost_ref, ds_drain_domains_ref, ds_drain_ref,
                          ds_drain_world, index_entries, link_targets, overlap_worlds, single_row_world, table_slot,
                          table_slots, wrap_keys)
from ds_link_world import linked_revroles
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORLDS = {"w0": dict(n_ds=60, n_nodes=24, seed=3), "w1": dict(n_ds=80, n_nodes=32, seed=11),
          "w2": dict(n_ds=60, n_nodes=24, seed=29, nodes_per_domain=4), "w3": dict(n_ds=40, n_nodes=16, seed=41)}


@pytest.fixture(scope="module", params=sorted(WORLDS))
def world(request):
    return ds_drain_world(**WORLDS[request.param])


def test_world_covers_the_cases(world):
    """The world has every kind the definition names: links that take, each fall-back cause, a shared child,
    BAD_TABLE, ready and stable DS."""
    w = world
    L = link_targets(w.revroles, w.links, w.lws, w.base[0])
    rr, took, _ = linked_revroles(w.revroles, w.links, w.lws, w.base[0])
    assert took == int((L >= 0).sum()) > 0
    assert (rr["ready_replicas"] == np.where(L >= 0, w.base[0]["ready_replicas"][np.maximum(L, 0)],
                                             w.revroles["ready_replicas"])).all()
    ex = (w.revroles["flags"] & R.RR_EXISTS) != 0
    assert (ex & (w.links["lws_row"] == R.NONE)).any()
    assert (ex & (w.links["lws_row"] != R.NONE) & (w.links["lws_row"] >= len(w.lws))).any()
    taken = L[L >= 0]
    assert len(np.unique(taken)) < len(taken)  # two rows, one child
    import oracle

    out = oracle.sweep_ds(w.ds, w.roles, rr)[0]
    for bit in (R.DOUT_BAD_TABLE, R.DOUT_NEW_READY, R.DOUT_STABLE, R.DOUT_ROLLING):
        assert ((out["flags"] & bit) != 0).any(), bit


def test_per_key_equals_set_form(world):
    """Row k of the per-key restatement is the set form for D = {k}, for every node and every domain."""
    w = world
    for by_domain, n_keys, call in ((False, len(w.nodes), lambda k: ds_drain_ref(w, [k])),
                                    (True, w.n_domains, lambda k: ds_drain_domains_ref(w, [k]))):
        cost = ds_drain_cost_ref(w, by_domain)
        hits = 0
        for k in range(n_keys):
            _, totals, _, _ = call(k)
            want = cost_row_of(totals)
            assert {f: int(cost[f][k]) for f in COST_FIELDS} == want, (by_domain, k)
            hits += want["ds_touched"] > 0
        assert hits > 0


def test_verdicts_occur():
    """Across the worlds, every verdict occurs for some single node or domain."""
    seen = 0
    for kw in WORLDS.values():
        w = ds_drain_world(**kw)
        for k in range(w.n_domains):
            rows, _, _, _ = ds_drain_domains_ref(w, [k])
            for r in rows:
                seen |= int(r["flags"])
    for bit in (R.DSD_TOUCHED, R.DSD_SERVICE_LOST, R.DSD_OLD_SERVICE_LOST, R.DSD_STALLS, R.DSD_CHANGED):
        assert seen & bit, bit


# --------------------------------------------------------------------------------------------------
# named cases on a hand-made world
# --------------------------------------------------------------------------------------------------
def tiny(n_old=1, n_roles=2, n_spec=2, has_new=True):
    """One DS, every row existing, replicas 1 and ready 1, each row linked to its own child LWS (one group of two
    pods on node = row index), from a world whose LWS sweep the oracle runs.  → World."""
    from lws_b200 import synth

    n_rr = (n_old + 1) * n_roles
    p = synth.Profile("tiny", n_rr, size_choices=(2,), replicas_choices=(1,), n_nodes=n_rr, nodes_per_domain=2,
                      node_capacity=64, f_mid_update=0.0, p_group_ready=1.0, p_leader_unscheduled=0.0,
                      restart_policy_p=(0.0, 1.0, 0.0))
    t = synth.make(p, seed=5)
    # child L's pods all on node L
    low = np.uint32((1 << R.PODID_NODE_SHIFT) - 1)
    for g in range(len(t.groups)):
        L, pb, pc = int(t.groups["lws_index"][g]), int(t.groups["pod_base"][g]), int(t.groups["pod_count"][g])
        t.groups["leader_node"][g] = L
        t.pod_ident["place"][pb: pb + pc] = (t.pod_ident["place"][pb: pb + pc] & low) | np.uint32(L << R.PODID_NODE_SHIFT)
    import oracle

    base = oracle.sweep_lws(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.flags & R.SWEEP_GANG)[:2]
    ds = R.aligned_empty(1, R.DS_REC)
    ds[0] = (7, 0, n_roles, n_spec, 0, n_old, R.DS_HAS_NEW_REVISION if has_new else 0)
    roles = R.aligned_empty(n_roles, R.DS_ROLE_REC)
    roles[:] = (1, 1, 0, R.ROLE_IN_SPEC | R.ROLE_HAS_ROLLING_CONFIG)
    roles["flags"][n_spec:] = 0
    rr = R.aligned_empty(n_rr, R.DS_REVROLE_REC)
    rr[:] = (1, 1, 1, R.RR_EXISTS)
    rr["flags"] |= (np.arange(n_rr) // n_roles + 1).astype(np.uint32) << np.uint32(R.RR_TS_SHIFT)
    links = R.aligned_empty(n_rr, R.DS_LINK)
    links["lws_row"] = np.arange(n_rr)
    links["lws_uid_hash"] = t.lws["uid_hash"][:n_rr]
    links["reserved"] = 0
    return World(t.lws, t.groups, t.pod_state, t.pod_ident, t.nodes, t.n_domains, t.flags, ds, roles, rr, links, base)


def node_of_child(w, L):
    g = int(w.lws["group_base"][L])
    return int(w.pod_ident["place"][int(w.groups["pod_base"][g])] >> R.PODID_NODE_SHIFT)


def ready_children(w):
    return int((w.base[0]["ready_replicas"] >= 1).sum())


def test_tiny_world_is_ready():
    w = tiny()
    assert ready_children(w) == len(w.revroles)
    rows, totals, _, _ = ds_drain_ref(w, [])
    assert totals["n_touched"] == 0 and totals["rows_linked"] == len(w.revroles)


def test_new_revision_loses_service_and_stalls():
    w = tiny()
    L = 3  # the new revision's second spec role
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, L)])
    assert totals["n_touched"] == 1 and totals["rows_zeroed"] == 1
    f = int(rows["flags"][0])
    assert f & R.DSD_SERVICE_LOST and f & R.DSD_CHANGED
    assert int(rows["new_zeroed_roles"][0]) == 0b10 and int(rows["old_zeroed_roles"][0]) == 0
    assert bool(f & R.DSD_STALLS) == bool(rows["before"]["flags"][0] & R.DOUT_STABLE)


def test_old_revision_loses_service_while_target_keeps_it():
    w = tiny()
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, 0)])  # old revision 0, role 0
    f = int(rows["flags"][0])
    assert f & R.DSD_OLD_SERVICE_LOST and not f & R.DSD_SERVICE_LOST and not f & R.DSD_STALLS
    assert int(rows["old_zeroed_roles"][0]) == 1 and int(rows["new_zeroed_roles"][0]) == 0


@pytest.mark.parametrize("cause", ["none", "stale_uid", "past_table", "not_existing"])
def test_fall_back_rows_see_no_drain(cause):
    w = tiny()
    r = 3
    if cause == "none":
        w.links["lws_row"][r] = R.NONE
    elif cause == "stale_uid":
        w.links["lws_uid_hash"][r] ^= np.uint64(1)
    elif cause == "past_table":
        w.links["lws_row"][r] = len(w.lws)
    else:
        w.revroles["flags"][r] &= ~np.uint32(R.RR_EXISTS)
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, r)])
    assert totals["n_touched"] == 0 and totals["rows_linked"] == len(w.revroles) - 1


def test_excluded_lws_flags_fall_back():
    w = tiny()
    lws_out = w.base[0].copy()
    lws_out["flags"][3] |= R.LOUT_STATUS_ERROR
    w.base = (lws_out, w.base[1])
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, 3)])
    assert totals["n_touched"] == 0 and totals["rows_linked"] == len(w.revroles) - 1


def test_no_link_patch_touches_nothing():
    w = tiny()
    w.links["lws_row"] = R.NONE
    for n in range(len(w.nodes)):
        _, totals, _, _ = ds_drain_ref(w, [n])
        assert totals["n_touched"] == 0 and totals["rows_linked"] == 0


def test_two_rows_linked_to_one_child():
    w = tiny()
    w.links[2] = w.links[3]  # new revision, both roles → child 3
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, 3)])
    assert totals["rows_touched"] == 2 and totals["rows_zeroed"] == 2
    cost = ds_drain_cost_ref(w)
    assert int(cost["rows_touched"][node_of_child(w, 3)]) == 2


def test_removed_role_counts_rows_not_verdicts():
    w = tiny(n_roles=3, n_spec=2)
    r = 5  # new revision, removed role
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, r)])
    assert totals["rows_touched"] == 1 and totals["rows_zeroed"] == 1
    assert int(rows["flags"][0]) & ~(R.DSD_TOUCHED | R.DSD_CHANGED) == 0
    assert int(rows["new_zeroed_roles"][0]) == 0  # (a removed role serves nothing)


def test_not_rolling_never_stalls():
    w = tiny(n_old=0)
    for n in range(len(w.nodes)):
        rows, _, _, _ = ds_drain_ref(w, [n])
        assert not (rows["flags"] & R.DSD_STALLS).any()
        assert not (rows["before"]["flags"] & R.DOUT_ROLLING).any()


@pytest.mark.parametrize("ready,lost_expected_zeroed", [(1, True), (2, False)])
def test_ready_minus_lost_crossing_one(ready, lost_expected_zeroed):
    """A child with `ready` ready groups losing one: ready_after = ready - 1 crosses 1 only from 1."""
    w = tiny()
    lws_out = w.base[0].copy()
    lws_out["ready_replicas"][3] = ready
    w.base = (lws_out, w.base[1])
    rows, totals, _, _ = ds_drain_ref(w, [node_of_child(w, 3)])
    assert totals["rows_touched"] == 1 and (totals["rows_zeroed"] == 1) == lost_expected_zeroed
    assert bool(int(rows["flags"][0]) & R.DSD_SERVICE_LOST) == lost_expected_zeroed


# --------------------------------------------------------------------------------------------------
# (DS, key) table sizing and probing
# --------------------------------------------------------------------------------------------------
def test_table_sizes_at_128_and_129_pairs():
    assert table_slots(128) == 256 and table_slots(129) == 512
    assert table_slots(0) == 256


def test_probing_wraps():
    """Keys chosen so that two land on the last slot: the second probes to slot 0 (the probe is linear mod the
    size, as in table_add)."""
    mask = 255
    last = [k for k in range(1 << 20) if table_slot((k << 32) | 1, mask) == mask][:2]
    assert len(last) == 2
    taken = {}
    for k in last:
        h = table_slot((k << 32) | 1, mask)
        while h in taken:
            h = (h + 1) & mask
        taken[h] = k
    assert sorted(taken) == [0, mask]


@pytest.mark.parametrize("n_pairs", [128, 129])
def test_single_row_worlds_have_their_pair_count(n_pairs):
    """The worlds the device test builds (DS, key) tables from: every DS row gives one (row, node) pair, so the
    per-key form sizes its table for exactly n_pairs pairs (256 slots at 128, 512 at 129)."""
    w = single_row_world({d: d % 63 for d in range(n_pairs)})
    cost = ds_drain_cost_ref(w)
    assert int(cost["rows_touched"].sum()) == int(cost["ds_touched"].sum()) == n_pairs
    for k in (0, 5, 62):
        assert cost_row_of(ds_drain_ref(w, [k])[1]) == {f: int(cost[f][k]) for f in COST_FIELDS}


def test_wrap_world_homes_keys_on_the_last_slot():
    keys = wrap_keys()
    assert len(keys) == 128 and table_slots(len(keys)) == 256
    homed = [d for d, k in keys.items() if table_slot((d << 32) | k, 255) == 255]
    assert len(homed) >= 12  # 12 entries cannot all sit in slot 255: inserts wrap to slot 0 and on
    cost = ds_drain_cost_ref(single_row_world(keys))
    assert int(cost["ds_touched"].sum()) == 128


def test_overlapping_ranges_count_rows_once_per_ds():
    """Two DS over one revision-role range: the reverse index holds a linked row once per DS, more entries than the
    table has rows; a world with copies of the rows needs as many."""
    shared, copied = overlap_worlds(ds_drain_world(n_ds=60, n_nodes=24, seed=3), 200)
    assert index_entries(shared) == index_entries(copied) > len(shared.revroles)


def test_kernel_sources_match_the_sizing():
    src = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_engine.cu")).read()
    assert "uint64_t ds_slots = 256;" in src and "while (ds_slots < 2 * ds_pairs) ds_slots <<= 1;" in src
    ksrc = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_drain_kernels.cu")).read()
    assert "k *= 0xFF51AFD7ED558CCDull;" in ksrc and "t = table_slot(dk, p.table_mask);" in ksrc


# --------------------------------------------------------------------------------------------------
# record layouts against the header (a gcc probe)
# --------------------------------------------------------------------------------------------------
PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "lwse.h"
#define O(T, f) printf(#T " " #f " %zu\n", offsetof(T, f))
#define S(T) printf(#T " sizeof %zu\n", sizeof(T))
int main(void) {
  S(lwse_ds_drain); O(lwse_ds_drain, ds); O(lwse_ds_drain, flags); O(lwse_ds_drain, rows_touched);
  O(lwse_ds_drain, rows_zeroed); O(lwse_ds_drain, new_zeroed_roles); O(lwse_ds_drain, old_zeroed_roles);
  O(lwse_ds_drain, reserved); O(lwse_ds_drain, before); O(lwse_ds_drain, after);
  S(lwse_ds_drain_cost); O(lwse_ds_drain_cost, ds_touched); O(lwse_ds_drain_cost, ds_service_lost);
  O(lwse_ds_drain_cost, ds_old_service_lost); O(lwse_ds_drain_cost, ds_stalled); O(lwse_ds_drain_cost, rows_touched);
  O(lwse_ds_drain_cost, rows_zeroed); O(lwse_ds_drain_cost, reserved);
  S(lwse_ds_drain_query); O(lwse_ds_drain_query, ids); O(lwse_ds_drain_query, n_ids); O(lwse_ds_drain_query, scope);
  O(lwse_ds_drain_query, capacity); O(lwse_ds_drain_query, reserved); O(lwse_ds_drain_query, rows);
  O(lwse_ds_drain_query, role_out); O(lwse_ds_drain_query, revrole_out); O(lwse_ds_drain_query, n_touched);
  O(lwse_ds_drain_query, n_service_lost); O(lwse_ds_drain_query, n_old_service_lost); O(lwse_ds_drain_query, n_stalled);
  O(lwse_ds_drain_query, n_changed); O(lwse_ds_drain_query, rows_touched); O(lwse_ds_drain_query, rows_zeroed);
  O(lwse_ds_drain_query, rows_linked);
  printf("DSD %u %u %u %u %u\n", LWSE_DSD_TOUCHED, LWSE_DSD_SERVICE_LOST, LWSE_DSD_OLD_SERVICE_LOST, LWSE_DSD_STALLS,
         LWSE_DSD_CHANGED);
  return 0;
}
"""


def test_record_layouts_match_the_header():
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "probe.c"), os.path.join(tmp, "probe")
        with open(src, "w") as f:
            f.write(PROBE)
        subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        lines = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines()
    got = {}
    for ln in lines:
        parts = ln.split()
        if parts[0] == "DSD":
            assert [int(x) for x in parts[1:]] == [R.DSD_TOUCHED, R.DSD_SERVICE_LOST, R.DSD_OLD_SERVICE_LOST,
                                                  R.DSD_STALLS, R.DSD_CHANGED]
            continue
        got[(parts[0], parts[1])] = int(parts[2])
    for T, dt in (("lwse_ds_drain", R.DS_DRAIN), ("lwse_ds_drain_cost", R.DS_DRAIN_COST)):
        assert got[(T, "sizeof")] == dt.itemsize
        for name in dt.names:
            assert got[(T, name)] == dt.fields[name][1], (T, name)
    assert got[("lwse_ds_drain_query", "sizeof")] == C.sizeof(R.DsDrainQuery)
    for name, _ in R.DsDrainQuery._fields_:
        assert got[("lwse_ds_drain_query", name)] == getattr(R.DsDrainQuery, name).offset, name


# --------------------------------------------------------------------------------------------------
# the informer's report
# --------------------------------------------------------------------------------------------------
def test_report_names_revisions():
    from ds_world import DsWorld
    from lws_b200 import ds_informer

    enc = ds_informer.DsIncrementalEncoder(DsWorld(2).initial_items(), spare=1.0)
    key = sorted(enc.slots)[0]
    d = enc.ds_row(*key)
    old = enc.old_revisions(d)
    row = np.zeros(1, R.DS_DRAIN)
    row["ds"] = d
    row["flags"] = R.DSD_TOUCHED | R.DSD_SERVICE_LOST | R.DSD_OLD_SERVICE_LOST
    row["before"]["ready_revs"] = (1 << len(old)) - 1
    row["rows_zeroed"] = 2
    names = enc.role_names(d)
    row["new_zeroed_roles"] = 1 << (len(names) - 1)
    row["old_zeroed_roles"] = 1
    rep = enc.ds_drain_report({"rows": row})
    assert rep[0]["namespace"] == key[0] and rep[0]["name"] == key[1]
    assert rep[0]["service_lost"] == {"revision": enc.items[key][1], "roles": [names[-1]]}
    assert rep[0]["old_service_lost"] == [{"revision": rev, "roles": [names[0]]} for rev in old]
    assert rep[0]["conditions"] == ["touched", "service_lost", "old_service_lost"]
