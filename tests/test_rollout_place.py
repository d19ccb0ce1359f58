"""Rollout placement (lwse_resident_rollout_place) without a GPU: solving only ns_i against the literal definition
(every namespace solved) on seeded fuzz worlds and on the edge world, each edge on its side, the wrong statements
caught, the informer's query and report, the 24-bit guard against the sources and the record layout."""
import os
import re

import numpy as np
import pytest

from lws_b200 import records as R
from rollout_place_ref import EXCL, edge_queries, edge_world, fuzz_world, proposals, rollout_place_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fuzz_query(w, seed):
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, len(w.lws), 60).astype(np.uint32)
    ns = (rows.astype(np.int64) % w.n_ns).astype(np.uint32)  # synth deals objects to namespaces round-robin
    return rows, ns


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ns_only_equals_the_definition_on_fuzz_worlds(seed):
    w = fuzz_world(seed)
    rows, ns = _fuzz_query(w, seed)
    assert (w.lws["flags"][rows] & EXCL).any()
    for recs in (None, proposals(w.lws, rows, seed)[1]):
        a = rollout_place_ref(w, rows, ns, recs=recs)
        b = rollout_place_ref(w, rows, ns, recs=recs, mode="literal")
        assert a["rows"].tobytes() == b["rows"].tobytes()
        assert a["n_surge"] > 0


@pytest.fixture(scope="module")
def edge():
    w, rows = edge_world()
    return w, rows, edge_queries(w, rows)


def test_ns_only_equals_the_definition_on_the_edge_world(edge):
    w, _, ((rr, rn), (pr, pn, recs), _) = edge
    for q in ((rr, rn, None), (pr, pn, recs)):
        a = rollout_place_ref(w, *q)
        b = rollout_place_ref(w, *q, mode="literal")
        assert a["rows"].tobytes() == b["rows"].tobytes()


def test_each_edge_lands_on_its_side(edge):
    w, rows, ((rr, rn), (pr, pn, recs), labels) = edge
    res = dict(zip(rows, rollout_place_ref(w, rr, rn)["rows"]))
    got = dict(zip(labels, rollout_place_ref(w, pr, pn, recs=recs)["rows"]))
    # exactly k = 3 fitting domains: a surge of 3 places, 4 strands one; a second object alone also places 3
    assert (got["k_fits"]["surge"], got["k_fits"]["stranded"]) == (3, 0)
    assert (got["k_plus_1_strands"]["surge"], got["k_plus_1_strands"]["stranded"]) == (4, 1)
    assert got["k_plus_1_strands"]["flags"] & R.RPL_STRANDS
    assert (got["other_k_fits"]["surge"], got["other_k_fits"]["stranded"]) == (3, 0)
    # extra rows beat the unpinned holders of namespace 3
    assert got["bumps"]["bumped"] == 3 and got["bumps"]["flags"] & R.RPL_BUMPS and got["bumps"]["stranded"] == 0
    # the 1 024 / 1 025 and 256 / 257 namespace
    assert got["rows_1024"]["surge"] == 4 and got["rows_1025"]["surge"] == 5
    # two proposals on one row with different maxSurge
    assert got["surge_0"]["surge"] == 0 and got["surge_2"]["surge"] == 2 and got["surge_2"]["peak"] == 5
    # size and exclusive edits are not modelled
    assert got["size_edit"]["flags"] == R.RPL_NOT_MODELLED and got["exclusive_edit"]["flags"] == R.RPL_NOT_MODELLED
    # a group below group_count without its leader pod is extra; the unpinned present group 0 is not
    assert res["C"]["surge"] == 1 and res["C"]["namespaces_solved"] == 1
    assert got["identity_c"].tobytes() == res["C"].tobytes()
    # a scale-down in progress: the peak is the current sts_replicas (3), not replicas + surge (2)
    assert res["D"]["peak"] == 3 and res["D"]["surge"] == 1
    assert res["N"]["flags"] == R.RPL_NOT_EXCLUSIVE
    assert res["BT"]["flags"] == R.RPL_NOT_FORECAST and res["BT"]["fc_flags"] & R.LWSF_BAD_TABLE
    assert res["IR"]["flags"] == R.RPL_NOT_FORECAST and res["IR"]["fc_flags"] & R.LWSF_NOT_FORECAST
    assert res["A"]["flags"] == R.RPL_SOLVED and res["A"]["surge"] == 0 and res["A"]["namespaces_solved"] == 0
    # the extra rows: the encoder's mix of (uid_hash, g) for g in E_i, in L_i's group range
    x = rollout_place_ref(w, rr, rn)["extra"][list(rows).index("C")]
    c = rows["C"]
    assert x["group"].tolist() == [int(w.lws["group_base"][c]) + 1] and (x["leader_node"] == R.NONE).all()
    assert x["ns"].tolist() == [int(rn[list(rows).index("C")])] and x["size"].tolist() == [int(w.lws["size"][c])]


@pytest.mark.parametrize("variant", ["no_pod_present", "replicas_surge", "together"])
def test_wrong_statements_give_wrong_rows(edge, variant):
    w, _, ((rr, rn), (pr, pn, recs), _) = edge
    wrong = 0
    for q in ((rr, rn, None), (pr, pn, recs)):
        a = rollout_place_ref(w, *q)["rows"]
        b = rollout_place_ref(w, *q, variant=variant)["rows"]
        wrong += int((a.view(np.uint8).reshape(len(a), 64) != b.view(np.uint8).reshape(len(b), 64)).any(axis=1).sum())
    assert wrong > 0


def test_unfinished_forecasts_are_solved_with_their_peak(edge):
    """UF's replay stops at n' = 7 > C = 6 without a cycle: the entry is solved with the peak it replayed (the
    StatefulSet's 6 replicas), its forecast flags copied, in both query forms."""
    w, rows, ((rr, rn), (pr, pn, recs), labels) = edge
    res = dict(zip(rows, rollout_place_ref(w, rr, rn)["rows"]))["UF"]
    got = dict(zip(labels, rollout_place_ref(w, pr, pn, recs=recs)["rows"]))["identity_uf"]
    assert res["fc_flags"] & R.LWSF_UNFINISHED and not res["fc_flags"] & (R.LWSF_BAD_TABLE | R.LWSF_NOT_FORECAST)
    assert res["flags"] & R.RPL_SOLVED and res["peak"] == 6 and res["surge"] == 3  # groups 3, 4 and 5
    assert res["placed"] + res["stranded"] == 3 and res["namespaces_solved"] == 1
    assert got.tobytes() == res.tobytes()


def test_informer_query_and_report():
    from informer_world import make_world

    from lws_b200 import informer

    items, cluster = make_world(3, n_lws=14, n_nodes=28)
    enc = informer.IncrementalEncoder(items, cluster, "zone")
    rows, ns = enc.rollout_place_query()
    keys = sorted(k for k, sl in enc.slots.items() if int(enc.lws["flags"][sl.lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY)
    assert len(rows) == len(keys) > 0
    assert [enc.slots[k].lws_row for k in keys] == rows.tolist()
    assert [enc.ns_ids[k[0]] for k in keys] == ns.tolist()
    some = sorted(enc.slots)[:3]
    r2, n2 = enc.rollout_place_query(some)
    assert r2.tolist() == [enc.slots[k].lws_row for k in some]
    item = enc.items[keys[0]]
    row, rec, v = enc.rollout_place_proposal(item)
    assert row == enc.slots[keys[0]].lws_row and v == enc.ns_ids[keys[0][0]] and rec.dtype == R.LWS_REC
    out = np.zeros(len(rows), R.ROLLOUT_PLACE)
    out["flags"] = R.RPL_SOLVED
    out["flags"][0] |= R.RPL_STRANDS
    out["stranded"][0] = 2
    rep = enc.rollout_place_report({"rows": out, "lws_rows": rows, "ns": ns})
    assert len(rep) == 1 and (rep[0]["namespace"], rep[0]["name"]) == keys[0]
    assert rep[0]["stranded"] == 2 and rep[0]["flags"] == ["solved", "strands"]


def test_24_bit_guard_in_the_sources():
    src = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_engine.cu")).read()
    body = src[src.index("LWSE_API int lwse_resident_rollout_place("):]
    body = body[: body.index("\n}\n")]
    assert "e->xch_world > 0 || e->rn_reqs >= (1u << 24)" in body  # (the peer exchange is refused with it)
    assert re.search(r"\(uint64_t\)nr \+ max_extra >= \(1ull << 24\)\) return LWSE_ERR_UNSUPPORTED", body)
    # the refusal comes before anything is copied out
    assert body.index("max_extra >= (1ull << 24)") < body.index("cudaMemcpyAsync(q->out")


def test_record_matches_header():
    h = open(os.path.join(ROOT, "include", "lwse.h")).read()
    s = h[h.index("typedef struct lwse_rollout_place {"):]
    s = s[: s.index("} lwse_rollout_place;")]
    fields = re.findall(r"^\s+u?int32_t (\w+);", s, re.M)
    assert tuple(fields) == R.ROLLOUT_PLACE.names
    for name, bit in re.findall(r"#define LWSE_RPL_(\w+) \(1u << (\d+)\)", h):
        assert getattr(R, "RPL_" + name) == 1 << int(bit)
