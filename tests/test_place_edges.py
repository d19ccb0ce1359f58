"""The placement edge cases (tests/place_edges_world.py) without a GPU: the launchers' constants are the
ones the mirror restates, every case sits on its declared side of every threshold it names, and the spec
oracle gives each case the rows it was built for."""
import os
import re

import numpy as np
import pytest

import place_edges_world as W
from lws_b200 import records as R

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lws_b200", "csrc")
SMS = [W.H100_SXM_SMS, 114]  # H100 SXM and H100 PCIe


def _src(name: str) -> str:
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _body(src: str, head: str) -> str:
    body = src[src.index(head):]
    return body[: body.index("\n}\n")]


def _const(src: str, name: str) -> int:
    m = re.search(rf"constexpr uint32_t {name} = (\d+);", src)
    assert m, name
    return int(m.group(1))


def test_the_mirror_uses_the_launchers_constants():
    g, ns, eng = _src("lwse_place_kernels.cu"), _src("lwse_place_ns_kernels.cu"), _src("lwse_engine.cu")
    assert _const(g, "kPlaceThreads") == W.K_PLACE_THREADS
    assert _const(g, "kClusterCtas") == W.K_CLUSTER_CTAS
    assert _const(g, "kCacheQ") == W.K_CACHE_Q
    assert _const(ns, "kNsCache") == W.K_NS_CACHE
    assert _const(ns, "kNsKeep") == W.K_NS_KEEP
    assert _const(ns, "kNsThreads") == W.K_NS_THREADS
    assert _const(ns, "kNsScanThreads") == W.K_NS_SCAN_THREADS
    lp = _body(g, "int launch_place(")
    m = re.search(r"few_reqs = n_reqs <= kClusterCtas \* kPlaceWarps \* (\d+)u;", lp)
    assert m and int(m.group(1)) == W.FEW_PER_WARP
    m = re.search(r"expect_unpinned <= kClusterCtas \* kPlaceWarps \* (\d+)u && n_reqs <= \(1u << (\d+)\)\)", lp)
    assert m and (int(m.group(1)), 1 << int(m.group(2))) == (W.PREDICTED_PER_WARP, W.MAX_CLUSTER_REQS)
    m = re.search(r"n_nodes <= \(1u << (\d+)\) && \(uint64_t\)n_namespaces \* hold_stride_of\(n_domains\) <= \(1u << (\d+)\)", lp)
    assert m and (1 << int(m.group(1)), 1 << int(m.group(2))) == (W.MAX_CLUSTER_NODES, W.MAX_CLUSTER_HOLD)
    assert re.search(r"ctas = \(n_reqs \+ kPlaceWarps - 1u\) / kPlaceWarps;", lp)
    m = re.search(r"if \(ctas < (\d+)u\) ctas = (\d+)u;", lp)
    assert m and int(m.group(1)) == int(m.group(2)) == W.GRID_MIN_CTAS
    assert re.search(r"static uint32_t hold_stride_of\(uint32_t n_domains\) \{ return \(n_domains \+ 1u\) & ~1u; \}", g)
    m = re.search(r"if \(n_reqs > (\d+)u && e->place_unpinned && eager\)", eng)
    assert m and int(m.group(1)) == W.HISTORY_ABOVE
    # the namespace launcher: shared memory, the 200 KB and 100 KB limits, the grid
    sm = _body(ns, "static size_t ns_smem_bytes(")
    assert "(size_t)n_domains * 8 + 256 * 32 + 16 + 128;" in sm
    assert "return base + (stage ? (size_t)word_rows * 2048 : 0);" in sm
    assert "return base + (size_t)n_domains * 16 + free_bytes;" in sm
    m = re.search(r"ns_smem_bytes\(\(n_nodes \+ 255u\) / 256u, n_domains, false, false\) <= (\d+)u \* 1024u", ns)
    assert m and int(m.group(1)) * 1024 == W.NS_SMEM_LIMIT
    m = re.search(r"a\.stage_words = \(scan && with_words <= (\d+)u \* 1024u\)", ns)
    assert m and int(m.group(1)) * 1024 == W.STAGE_SMEM_LIMIT
    m = re.search(r"unsigned grid = n_namespaces < \(unsigned\)sm_count \* (\d+)u \? n_namespaces : \(unsigned\)sm_count \* (\d+)u;", ns)
    assert m and int(m.group(1)) == int(m.group(2)) == 2


def test_the_restated_rules_at_their_thresholds():
    assert W.place_ns_supported(6000, W.NS_DOMAIN_LIMIT) and not W.place_ns_supported(6000, W.NS_DOMAIN_LIMIT + 1)
    assert W.stage_words(11520, 48) and not W.stage_words(11521, 48)
    assert W.stage_words(9728, 1000) and not W.stage_words(9729, 1000)
    p = W.general_path
    assert p(1024, 100, 10, 1, 1024) == "cluster" and p(1025, 100, 10, 1, 1025) == "grid"
    assert p(16384, 100, 10, 1, 256) == "cluster" and p(16384, 100, 10, 1, 257) == "grid"
    assert p(16385, 100, 10, 1, 0) == "grid"
    assert p(1024, 65536, 10, 1, 0) == "cluster" and p(1024, 65537, 10, 1, 0) == "grid"
    assert p(100, 100, 8192, 8, 0) == "cluster" and p(100, 100, 8193, 8, 0) == "grid"
    assert [W.grid_ctas(n, 132) for n in (1, 256, 257, 2112, 2113, 10 ** 6)] == [16, 16, 17, 132, 132, 132]


def _cases(sm):
    return [(name, W.BUILDERS[name](sm)) for name in W.BUILDERS]


@pytest.fixture(scope="module", params=SMS, ids=lambda s: f"sm{s}")
def cases(request):
    return request.param, dict(_cases(request.param))


def test_every_case_sits_on_its_edges(cases):
    sm, all_cases = cases
    for name, c in all_cases.items():
        for e in c.edges:
            q, limit, side = e[:3]
            v = W.quantities(c, sm, e[3] if len(e) > 3 else 0)[q]
            assert (v <= limit) if side == "under" else (v > limit), (name, e, v)
        if c.entry == "general":
            assert [x["path"] for x in W.general_calls(c, sm)] == c.paths, name
            for reqs in c.calls:  # so that lwse_place_host runs the general form too
                assert W.host_form(reqs, len(c.nodes), c.n_domains) == "general", name
        else:
            assert W.grouped(c.calls[0]), name
            assert W.ns_view(c, sm)["supported"] == (name != "n3_domains_5457"), name


def test_the_general_cases_hit_their_counts(cases):
    sm, c = cases
    g1 = W.general_calls(c["g1_cluster_1024"], sm)[0]
    assert g1["live_unpinned"] == g1["n_reqs"] == 1024 and g1["per_warp"] == 8
    g1b = W.general_calls(c["g1_grid_1025"], sm)[0]
    assert g1b["live_unpinned"] == 1025 and g1b["ctas"] == min(65, sm) and g1b["per_warp"] == 1
    a, b, cc = W.general_calls(c["g2_misprediction"], sm)
    assert a["n_reqs"] == b["n_reqs"] == cc["n_reqs"] == W.MAX_CLUSTER_REQS
    assert 150 <= a["live_unpinned"] <= 256 and b["live_unpinned"] == cc["live_unpinned"] == 16384
    assert b["per_warp"] == 128 and cc["expect_unpinned"] == 16384 and cc["ctas"] == sm
    g3 = W.general_calls(c["g3_grid_overflow"], sm)[0]
    assert g3["ctas"] == sm and g3["live_unpinned"] > 4 * sm * W.K_PLACE_WARPS and g3["per_warp"] == 6
    assert W.general_calls(c["g4_nodes_65536"], sm)[0]["n_nodes"] == 65536
    g4 = W.general_calls(c["g4_nodes_65537"], sm)[0]
    assert g4["n_nodes"] == 65537 and g4["n_reqs"] <= 100 and g4["ctas"] == W.GRID_MIN_CTAS
    assert -(-g4["n_reqs"] // W.K_PLACE_WARPS) < W.GRID_MIN_CTAS
    assert W.general_calls(c["g4_hold_65536"], sm)[0]["hold"] == 65536
    assert W.general_calls(c["g4_hold_65552"], sm)[0]["hold"] == 65552 and c["g4_hold_65552"].n_domains % 2 == 1


def test_the_namespace_cases_hit_their_counts(cases):
    sm, c = cases
    v = W.ns_view(c["n1_cache"], sm)
    assert list(v["unpinned"]) == [256, 257, 640, 0] and v["pinned"][3] > 0
    assert (c["n1_cache"].calls[0]["ns"] >= 4).sum() == 5
    n2 = c["n2_unkept"]
    v = W.ns_view(n2, sm)
    assert tuple(v["rows"]) == W.N2_ROWS
    t = n2.calls[0]
    for ns, n in enumerate(W.N2_ROWS):
        rows = t[t["ns"] == ns]
        for keep in (W.KEEP_SCAN, W.KEEP_TWO_LEVEL):
            past = rows[keep:]
            if len(past):  # a pinned claim right past the kept positions, on a domain claimed before them
                assert past["leader_node"][0] != R.NONE
                d = n2.nodes["domain_id"][past["leader_node"][0]]
                assert d in n2.nodes["domain_id"][rows["leader_node"][:2]]
    for name, stage in (("n4_stage_11520", True), ("n4_stage_11521", False), ("n4_stage_9728", True),
                        ("n4_stage_9729", False)):
        assert W.ns_view(c[name], sm)["stage_words"] == stage, name
    n5 = c["n5_ctas"]
    v = W.ns_view(n5, sm)
    g = 2 * sm
    assert v["grid"] == g and n5.n_namespaces == g + W.N5_EXTRA
    for b in range(g):
        mine = list(range(b, n5.n_namespaces, g))
        work = [int(v["unpinned"][x]) for x in mine]
        if b < W.N5_EXTRA:  # work only in the later namespace
            assert work[0] == 0 and work[1] > 0, b
        assert work[0] == 0 or b % 3 == 0
    idle = [b for b in range(g) if all(v["unpinned"][x] == 0 for x in range(b, n5.n_namespaces, g))]
    assert any(v["pinned"][b] > 0 for b in idle) and any(v["rows"][b] == 0 for b in idle)


@pytest.mark.parametrize("name", list(W.BUILDERS))
def test_the_oracle_gives_the_counted_rows(name):
    import oracle

    c = W.BUILDERS[name](W.H100_SXM_SMS)
    displaced = 0
    for k, reqs in enumerate(c.calls[:2]):
        out = oracle.place(c.nodes, c.occ, c.n_domains, c.n_namespaces, reqs, threads=8)
        got = W.flag_counts(out)
        assert got == W.expected_counts(c.nodes, c.occ, c.n_domains, c.n_namespaces, reqs), (name, k)
        assert got["placed"] > 0 and got["unschedulable"] > 0, (name, k, got)
        pinned = reqs["leader_node"] != R.NONE
        assert got["conflict"] > 0 or not pinned.any(), (name, k, got)
        if c.contention:
            rounds, final = W.deferred_acceptance(c.nodes, c.occ, c.n_domains, c.n_namespaces, reqs)
            live = W.live_unpinned(reqs, c.n_namespaces)
            won = (out["flags"] & R.PLACE_PLACED) != 0
            want = np.where(won, out["domain_id"].astype(np.int64), -1)
            assert np.array_equal(final[live], want[live]), name
            displaced = max(displaced, *rounds.values())
    # a contention case: in some namespace claims meet holders in more than one round
    assert displaced >= 2 or not c.contention, name
