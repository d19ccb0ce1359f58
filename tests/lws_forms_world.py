"""Tables built to land on each form of the LWS sweep, at the form's boundaries.

``launch_lws_sweep`` (``lws_b200/csrc/lwse_lws_kernels.cu``) picks its kernels from the table shape
alone: the fused scan + group kernel when groups average 16-256 pods, else the pod scan and
``group_sweep_kernel<W>`` (W = 1/2/4/8 lanes per group); inside the fused kernel each CTA picks the
shared-memory window or ``DirectBits`` by the words its pod window spans, and the cooperative pair
list or the per-group visit by its (group, event pod) pairs; the LWS pass runs ``lws_sweep_kernel<W>``
with W from ``pick_tile``.  Every builder here sets the counts with numpy so that the table lands
exactly on its label, and the constants the labels depend on are restated below
(``tests/test_lws_forms.py`` reads them back from the kernel source).

Every table also holds groups whose pod ranges start at bit 0 and end at bit 31 of a bitmap word, a
single-pod group in mid-word and an empty group between full ones.  Each world carries a churn plan:
ticks of row patches on the pod state bytes, the identity rows (pods moving between nodes and becoming
unscheduled), the group rows and the LWS rows (replicas, partition, StatefulSet replicas, the UPDATED
bit), with the same set of tables in every tick of the plan.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from lws_b200 import records as R
from lws_b200 import synth

# the launcher's constants (lwse_lws_kernels.cu)
K_FUSED_THREADS = 256   # groups per CTA of group_fused_kernel
K_WIN_WORDS = 2048      # bitmap words of a CTA's shared-memory window
K_PAIR_CAP = 1280       # (group, event pod) pairs a CTA visits cooperatively
FUSED_MIN_AVG, FUSED_MAX_AVG = 16, 256   # average pods per group of the fused form
GROUP_W_ABOVE = (512, 1024, 2048)        # above these averages the group pass takes 2 / 4 / 8 lanes
LWS_TILE_DIV, LWS_TILE_CAP = 64, 32      # pick_tile: next power of two >= ceil(avg groups / 64), at most 32

N_NODES = 64
_OLD = np.uint64(0x9E3779B97F4A7C15)


# --------------------------------------------------------------------------- #
# the selection rule, restated
# --------------------------------------------------------------------------- #
def pick_tile(items: int, owners: int) -> int:
    if owners == 0:
        return 1
    avg = (-(-items // owners) + LWS_TILE_DIV - 1) // LWS_TILE_DIV
    w = 1
    while w < LWS_TILE_CAP and w < avg:
        w <<= 1
    return w


@dataclass(frozen=True)
class Form:
    fused: bool
    scan: bool
    group_w: int | None  # lanes per group of group_sweep_kernel, None = not launched
    lws_w: int | None    # lanes per object of lws_sweep_kernel, None = not launched

    @property
    def kernels(self) -> int:
        return int(self.fused) + int(self.scan) + int(self.group_w is not None) + int(self.lws_w is not None)


def sweep_form(n_lws: int, n_groups: int, n_pods: int) -> Form:
    """The kernels launch_lws_sweep launches for a table of this shape (no skip flags)."""
    avg = -(-n_pods // n_groups) if n_groups else 0
    fused = n_groups > 0 and FUSED_MIN_AVG <= avg <= FUSED_MAX_AVG
    scan = not fused and n_pods > 0 and n_groups > 0
    w = 1
    for k, above in enumerate(GROUP_W_ABOVE):
        if avg > above:
            w = 2 << k
    group_w = w if n_groups and not fused else None
    return Form(fused, scan, group_w, pick_tile(n_groups, n_lws) if n_lws else None)


def form_of(t) -> Form:
    return sweep_form(len(t.lws), len(t.groups), len(t.pod_state))


def pod_predicates(pod_state: np.ndarray):
    """(pending, event) per pod, as the scan derives them (pod_controller.go:356, pod_utils.go:29-50)."""
    phase = pod_state & R.POD_PHASE_MASK
    pending = phase == R.POD_PHASE_PENDING
    event = (((phase == R.POD_PHASE_PENDING) | (phase == R.POD_PHASE_RUNNING)) & ((pod_state & R.POD_ANY_RESTART) != 0)) | (
        (pod_state & R.POD_DELETING) != 0)
    return pending, event


def visited_pairs(lws, groups, pod_state) -> np.ndarray:
    """Per group: the event pods the group pass visits (policy on, not suppressed), 0 for bad rows."""
    n_pods, G = len(pod_state), len(groups)
    base = groups["pod_base"].astype(np.int64)
    cnt = groups["pod_count"].astype(np.int64)
    li = groups["lws_index"].astype(np.int64)
    bad = (li >= len(lws)) | (base + cnt > n_pods)
    pending, event = pod_predicates(pod_state)
    cp = np.concatenate([[0], np.cumsum(pending, dtype=np.int64)])
    ce = np.concatenate([[0], np.cumsum(event, dtype=np.int64)])
    lo, hi = np.where(bad, 0, base), np.where(bad, 0, base + cnt)
    n_pend, n_ev = cp[hi] - cp[lo], ce[hi] - ce[lo]
    if len(lws) == 0:
        return np.zeros(G, np.int64)
    own = lws[np.where(bad, 0, li)]
    lflags = own["flags"].astype(np.int64)
    size = own["size"].astype(np.int64) & 0xFFFFFFFF
    policy = (lflags & R.LWS_RESTART_MASK) >> R.LWS_RESTART_SHIFT
    on = (policy == R.RESTART_ON_POD_RESTART) | (policy == R.RESTART_AFTER_START)
    grp_pending = (size != cnt) | (n_pend > 0)
    suppressed = grp_pending & ((policy == R.RESTART_AFTER_START) | ((lflags & R.LWS_RECREATE_AFTER_START_ANNOT) != 0))
    return np.where(~bad & on & ~suppressed, n_ev, 0)


@dataclass
class Cta:
    words: int     # bitmap words of the CTA's pod window (128-byte aligned start)
    windowed: bool
    pairs: int     # (group, event pod) pairs it visits
    max_rel: int   # highest window position of a visited event pod, -1 = none


def fused_ctas(lws, groups, pod_state) -> list[Cta]:
    """What every CTA of group_fused_kernel sees."""
    n_pods, G = len(pod_state), len(groups)
    base = groups["pod_base"].astype(np.int64)
    cnt = groups["pod_count"].astype(np.int64)
    li = groups["lws_index"].astype(np.int64)
    bad = (li >= len(lws)) | (base + cnt > n_pods)
    has = ~bad & (cnt > 0)
    pairs = visited_pairs(lws, groups, pod_state)
    _, event = pod_predicates(pod_state)
    out = []
    for c0 in range(0, G, K_FUSED_THREADS):
        sl = slice(c0, min(c0 + K_FUSED_THREADS, G))
        h = has[sl]
        if h.any():
            lo = int((base[sl][h] >> 5).min()) & ~3
            hi = int(((base[sl][h] + cnt[sl][h] - 1) >> 5).max()) + 1
        else:
            lo = hi = 0
        words = hi - lo if hi > lo else 0
        max_rel = -1
        for g in np.flatnonzero(pairs[sl] > 0) + c0:
            ev = np.flatnonzero(event[base[g]: base[g] + cnt[g]])
            max_rel = max(max_rel, int(base[g] + ev[-1]) - 32 * lo)
        out.append(Cta(words, words <= K_WIN_WORDS, int(pairs[sl].sum()), max_rel))
    return out


# --------------------------------------------------------------------------- #
# the LWS pass, restated for Case 5 (rollingUpdatePartition, :643-673)
# --------------------------------------------------------------------------- #
def lws_case(l) -> int:
    """Which case of rollingUpdateParameters an object row takes: 1-5, 0 = an error return."""
    f = int(l["flags"])
    if not f & R.LWS_STS_EXISTS:
        return 1
    if f & R.LWS_INTSTR_INVALID:
        return 0
    if f & R.LWS_UPDATED:
        return 2
    r, n = int(l["replicas"]), int(l["sts_replicas"])
    if (int(l["sts_partition"]) == 0 and n == r) or n < r:
        return 3
    if not f & R.LWS_ANNOT_VALID:
        return 0
    return 4 if int(l["sts_replicas_annotation"]) != r else 5


def _scaled(val: int, percent: bool, total: int, up: bool) -> int:
    if not percent:
        return val
    q, rem = divmod(val * total, 100)
    return q + (1 if up and rem else 0)


def case5_walk(l, group_out) -> dict:
    """Case 5's walk over the replica states the group pass left in ``group_out``: the highest slot that
    is not ready ∧ updated (``max_bad``), the rolling-step partition ``rsp``, the walk's start ``hi`` and
    the blocker it stops at (-1 = none)."""
    f = int(l["flags"])
    r, n = int(l["replicas"]), int(l["sts_replicas"])
    mu = _scaled(int(l["max_unavailable"]), bool(f & R.LWS_UNAVAIL_IS_PERCENT), r, False)
    surge = min(_scaled(int(l["max_surge"]), bool(f & R.LWS_SURGE_IS_PERCENT), r, True), r)
    gb, gc = int(l["group_base"]), int(l["group_count"])
    st = np.zeros(max(n, 0), np.int64)
    live = min(n, gc)
    st[:live] = group_out["flags"][gb: gb + live] & 3  # bit 0 ready, bit 1 updated
    ready, updated = (st & 1) != 0, (st & 2) != 0
    bad = np.flatnonzero(~(ready & updated))
    max_bad = int(bad[-1]) if len(bad) else -1
    step = mu + surge - (r + surge - n)
    rsp = max(0, max_bad + 1 - step)
    part = rsp + int((~ready[:rsp]).sum())
    hi = min(part, n - 1)
    cand = np.flatnonzero(ready[rsp: hi + 1] & ~updated[rsp: hi + 1]) if hi >= rsp else np.zeros(0, np.int64)
    blocker = int(cand[-1]) + rsp if len(cand) else -1
    if hi >= rsp:
        part = rsp if blocker < 0 else blocker + 1 if blocker < hi else part
    return {"max_bad": max_bad, "rsp": rsp, "hi": hi, "blocker": blocker, "walk": hi >= rsp, "part": part}


# --------------------------------------------------------------------------- #
# builders
# --------------------------------------------------------------------------- #
@dataclass
class FormWorld:
    label: str
    tables: synth.Tables
    plan: list   # one dict per tick: table -> (rows uint32, values)
    bad_groups: bool = False  # every group row is BAD_TABLE by construction


def boundary_pattern(avg: int) -> np.ndarray:
    """Pod counts of m groups (m * avg pods) from a 32-aligned pod: bits 0-31 of a word | bits 0-14 |
    a single pod at bit 15 | an empty group | bits 16-31 | the rest spread over the remaining groups."""
    head = [32, 15, 1, 0, 16]
    m = 6
    while m * avg < sum(head) + (m - len(head)):
        m += 1
    rest, k = m * avg - sum(head), m - len(head)
    tail = np.full(k, rest // k, np.int64)
    tail[: rest % k] += 1
    return np.concatenate([head, tail]).astype(np.int64)


def _counts(G: int, avg: int, rng, at: int = 0, jitter: bool = True) -> np.ndarray:
    """G pod counts summing to exactly avg * G, the boundary pattern at group ``at`` (32-aligned there)."""
    c = np.full(G, avg, np.int64)
    p = boundary_pattern(avg)
    c[at: at + len(p)] = p
    if jitter:  # move pods between random pairs of groups outside the pattern: the sum stays
        free = np.setdiff1d(np.arange(G), np.arange(at, at + len(p)))
        for _ in range(len(free) // 4):
            i, j = rng.choice(free, 2, replace=False)
            d = int(rng.integers(0, max(1, min(c[j] - 1, avg // 2) + 1)))
            c[i] += d
            c[j] -= d
    assert c.sum() == avg * G and (c >= 0).all()
    return c


def _split(G: int, rng, mean: int) -> np.ndarray:
    """Group counts per object summing to G (0 .. 2 mean each; empty objects included)."""
    out, left = [], G
    while left > 0:
        k = min(left, int(rng.integers(0, 2 * mean + 1)))
        out.append(k)
        left -= k
    return np.asarray(out, np.int64)


def _lws_rows(rng, gcs: np.ndarray, sizes: np.ndarray, group_base: np.ndarray | None = None):
    """Object rows over consecutive group ranges, every case of rollingUpdateParameters represented.
    → (lws, kind per object: 1 no sts, 2 updated, 3 steady, 4 replicas changed, 5 rolling, 6 done)."""
    L = len(gcs)
    lws = R.aligned_empty(L, R.LWS_REC)
    if group_base is None:
        group_base = np.concatenate([[0], np.cumsum(gcs)[:-1]]) if L else np.zeros(0, np.int64)
    kind = rng.choice(np.arange(1, 7), size=L, p=[0.08, 0.12, 0.1, 0.12, 0.46, 0.12])
    lws["rev_hash"] = rng.integers(0, 1 << 63, size=L, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    lws["size"] = sizes
    policy = rng.choice(3, size=L, p=[0.2, 0.6, 0.2]).astype(np.uint32)
    flags = (policy << np.uint32(R.LWS_RESTART_SHIFT)) | np.uint32(R.LWS_ANNOT_VALID)
    flags |= np.where(kind != 1, R.LWS_STS_EXISTS, 0).astype(np.uint32)
    flags |= np.where(kind == 2, R.LWS_UPDATED, 0).astype(np.uint32)
    flags |= np.where(rng.random(L) < 0.05, R.LWS_RECREATE_AFTER_START_ANNOT, 0).astype(np.uint32)
    flags |= np.where(rng.random(L) < 0.1, R.LWS_STARTUP_LEADER_READY, 0).astype(np.uint32)
    flags |= np.where(rng.random(L) < 0.3, R.LWS_EXCLUSIVE_TOPOLOGY, 0).astype(np.uint32)
    pct = rng.random(L) < 0.3
    flags |= np.where(pct, R.LWS_SURGE_IS_PERCENT, 0).astype(np.uint32)
    n = gcs + rng.choice([-1, 0, 0, 0, 1], size=L)
    n = np.maximum(n, 0)
    surge = np.where(pct, rng.choice([10, 50, 100], size=L), rng.integers(0, 3, size=L))
    surge_abs = np.where(pct, -(-surge * n // 100), surge)
    r = np.where(kind == 5, np.maximum(n - np.minimum(surge_abs, n // 2), 0), n)
    r = np.where(kind == 2, np.maximum(n - rng.integers(0, 2, size=L), 0), r)
    mu = rng.integers(0, 4, size=L)
    cur = np.where(kind == 3, 0, np.where(kind == 6, 0, rng.integers(1, np.maximum(n, 1) + 1)))
    annot = np.where(kind == 4, r + rng.choice([-2, 1, 3], size=L), r)
    lws["flags"] = flags
    lws["replicas"] = r
    lws["partition"] = np.where(rng.random(L) < 0.1, rng.integers(0, np.maximum(r, 1) + 1), 0)
    lws["max_surge"] = surge
    lws["max_unavailable"] = mu
    lws["sts_replicas"] = n
    lws["sts_partition"] = cur
    lws["sts_replicas_annotation"] = annot
    lws["subgroup_size"] = 0
    lws["uid_hash"] = rng.integers(0, 1 << 63, size=L, dtype=np.uint64)
    lws["group_base"] = group_base
    lws["group_count"] = gcs
    return lws, kind


def _group_rows(rng, lws, kind, owner, pod_base, pod_count, ready=None, updated=None):
    G = len(owner)
    g = R.aligned_empty(G, R.GROUP_REC)
    has_owner = owner < len(lws)
    o = np.where(has_owner, owner, 0)
    rev = lws["rev_hash"][o] if len(lws) else np.zeros(G, np.uint64)
    size = lws["size"][o].astype(np.int64) if len(lws) else np.full(G, 2, np.int64)
    k = kind[o] if len(lws) else np.full(G, 5)
    if ready is None:
        ready = np.where(k == 6, True, rng.random(G) < 0.85)
    if updated is None:
        # a rolling update moves from the highest slot down: slots at or above a frontier are updated
        slot = np.arange(G) - (lws["group_base"][o].astype(np.int64) if len(lws) else 0)
        frontier = (rng.random(len(lws)) * (lws["group_count"].astype(np.int64) + 1)).astype(np.int64) if len(lws) else 0
        updated = np.where(k == 6, True, np.where(k == 2, rng.random(G) < 0.1, slot >= (frontier[o] if len(lws) else 0)))
        updated ^= rng.random(G) < 0.05
    g["leader_rev_hash"] = np.where(updated, rev, rev ^ _OLD)
    g["wsts_rev_hash"] = np.where(updated & (rng.random(G) > 0.03), rev, rev ^ _OLD)
    g["wsts_spec_replicas"] = np.maximum(size - 1, 0)
    g["wsts_avail_replicas"] = np.maximum(size - 1, 0)
    g["leader_uid_hash"] = rng.integers(0, 1 << 32, size=G, dtype=np.uint64).astype(np.uint32)
    g["wsts_uid_hash"] = rng.integers(0, 1 << 32, size=G, dtype=np.uint64).astype(np.uint32)
    g["wsts_owner_uid_hash"] = np.where(rng.random(G) < 0.97, g["leader_uid_hash"], g["wsts_uid_hash"])
    g["leader_node"] = np.where(rng.random(G) < 0.1, R.NONE, rng.integers(0, N_NODES, size=G)).astype(np.uint32)
    g["pod_base"] = pod_base
    g["pod_count"] = pod_count
    g["lws_index"] = owner
    gf = np.full(G, R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH | R.GRP_POD_RUNNING | R.GRP_WSTS_LABEL_NAME_MATCH
                 | R.GRP_WSTS_FOUND | R.GRP_WSTS_REV_SETTLED | R.GRP_WSTS_OWNER_IS_POD | R.GRP_WSTS_OWNER_NAME_MATCH
                 | R.GRP_REVISION_EXISTS, dtype=np.uint32)
    gf |= np.where(ready, R.GRP_POD_READY, 0).astype(np.uint32)
    gf |= np.where(rng.random(G) < 0.02, R.GRP_POD_DELETING, 0).astype(np.uint32)
    gf &= ~np.where(rng.random(G) < 0.03, R.GRP_WSTS_FOUND | R.GRP_WSTS_LABEL_NAME_MATCH, 0).astype(np.uint32)
    g["flags"] = gf
    g["reserved"] = 0
    return g


def _pods(rng, groups, n_pods, p_event=0.01):
    """State bytes and identity rows: the first pod of a group is its leader; pods outside every
    group's range get states too."""
    pst = R.aligned_empty(n_pods, R.POD_STATE)
    base = groups["pod_base"].astype(np.int64)
    cnt = groups["pod_count"].astype(np.int64)
    pg = np.full(n_pods, -1, np.int64)
    for_g = np.repeat(np.arange(len(groups)), cnt)
    idx = np.concatenate([np.arange(b, b + c) for b, c in zip(base, cnt)]) if len(groups) else np.zeros(0, np.int64)
    idx = idx.astype(np.int64)
    pg[idx] = for_g
    leader = np.zeros(n_pods, bool)
    leader[base[cnt > 0]] = True
    phase = np.where(rng.random(n_pods) < 0.03, R.POD_PHASE_PENDING, R.POD_PHASE_RUNNING).astype(np.uint32)
    phase[rng.random(n_pods) < 0.01] = 0
    bits = phase
    bits |= np.where(rng.random(n_pods) < p_event, R.POD_ANY_RESTART, 0).astype(np.uint32)
    bits |= np.where(rng.random(n_pods) < p_event / 4, R.POD_DELETING, 0).astype(np.uint32)
    bits |= np.uint32(R.POD_OWNER_STS << R.POD_OWNER_SHIFT)
    bits |= np.where(rng.random(n_pods) < 0.98, R.POD_OWNER_NAME_MATCH, 0).astype(np.uint32)
    bits |= np.where(leader, R.POD_IS_LEADER, 0).astype(np.uint32)
    pst[:] = bits.astype(np.uint8)
    gi = np.where(pg >= 0, pg, 0)
    rev = groups["leader_rev_hash"][gi] if len(groups) else np.zeros(n_pods, np.uint64)
    rev = np.where(rng.random(n_pods) < 0.98, rev, rev ^ np.uint64(1))
    uid = groups["wsts_uid_hash"][gi] if len(groups) else np.zeros(n_pods, np.uint32)
    uid = np.where(rng.random(n_pods) < 0.98, uid, uid ^ np.uint32(1))
    node = rng.integers(0, N_NODES, size=n_pods).astype(np.uint32)
    place = np.where(rng.random(n_pods) < 0.99, R.PODID_NAME_OK, 0).astype(np.uint32)
    place |= np.where(rng.random(n_pods) < 0.85, np.uint32(R.PODID_SCHEDULED) | (node << np.uint32(R.PODID_NODE_SHIFT)),
                      0).astype(np.uint32)
    return pst, R.pod_ident_table(rev, uid, place)


def _assemble(label, rng, gcs, pod_count, pod_base=None, n_pods=None, p_event=0.01, sizes=None, lws=None, kind=None,
              ready=None, updated=None, tables=None, all_rows=None):
    """Object rows over ``gcs`` groups each, group rows over pod ranges (consecutive unless ``pod_base``)."""
    pod_count = np.asarray(pod_count, np.int64)
    if pod_base is None:
        pod_base = np.concatenate([[0], np.cumsum(pod_count)[:-1]]) if len(pod_count) else np.zeros(0, np.int64)
    if n_pods is None:
        n_pods = int((pod_base + pod_count).max()) if len(pod_count) else 0
    G = len(pod_count)
    owner = np.repeat(np.arange(len(gcs)), gcs) if gcs is not None else np.zeros(G, np.int64)
    assert len(owner) == G
    if lws is None:
        if sizes is None:  # an object's size = the pod count of its first group (its groups are not pending)
            first = np.concatenate([[0], np.cumsum(gcs)[:-1]]).astype(np.int64)
            sizes = np.where(gcs > 0, pod_count[np.minimum(first, max(G - 1, 0))] if G else 1, 2)
            sizes = np.maximum(sizes, 1)
        lws, kind = _lws_rows(rng, gcs, sizes)
    grp = _group_rows(rng, lws, kind, owner, pod_base, pod_count, ready, updated)
    pst, pid = _pods(rng, grp, n_pods, p_event)
    nodes, n_domains = synth.make_nodes(synth.Profile(label, len(lws), n_nodes=N_NODES, nodes_per_domain=4), rng)
    t = synth.Tables(synth.Profile(label, len(lws), n_nodes=N_NODES, nodes_per_domain=4), lws, grp, pst, pid, nodes,
                     n_domains, R.SWEEP_GANG)
    if tables is None:
        tables = [x for x, n in ((R.TABLE_POD_STATE, n_pods), (R.TABLE_POD_IDENT, n_pods), (R.TABLE_GROUPS, G),
                                 (R.TABLE_LWS, len(lws))) if n]
    return FormWorld(label, t, make_plan(t, rng, tables, all_rows=all_rows))


# --------------------------------------------------------------------------- #
# churn
# --------------------------------------------------------------------------- #
def _sample(rng, n, k):
    return np.sort(rng.choice(n, size=min(max(k, 1), n), replace=False)).astype(np.uint32)


def make_plan(t, rng, tables, n_ticks: int = 4, all_rows=None) -> list:
    """``n_ticks`` ticks of row patches on ``tables``, every tick touching each of them.  ``all_rows``:
    the table whose every row changes in every tick."""
    m = {R.TABLE_LWS: t.lws.copy(), R.TABLE_GROUPS: t.groups.copy(), R.TABLE_POD_STATE: t.pod_state.copy(),
         R.TABLE_POD_IDENT: t.pod_ident.copy()}
    plan = []
    for _ in range(n_ticks):
        tick = {}
        for tb in tables:
            cur = m[tb]
            n = len(cur)
            rows = np.arange(n, dtype=np.uint32) if tb == all_rows else _sample(rng, n, n // 40)
            vals = R.aligned_empty(len(rows), cur.dtype)
            vals[:] = cur[rows]
            k = len(rows)
            if tb == R.TABLE_POD_STATE:
                v = vals.copy()
                r = rng.random(k)
                ph = v & R.POD_PHASE_MASK
                flip = (r < 0.5) & ((ph == R.POD_PHASE_PENDING) | (ph == R.POD_PHASE_RUNNING))
                v[flip] ^= np.uint8(3)
                v[(r >= 0.5) & (r < 0.85)] ^= np.uint8(R.POD_ANY_RESTART)
                v[r >= 0.85] ^= np.uint8(R.POD_DELETING)
                vals[:] = v
            elif tb == R.TABLE_POD_IDENT:
                node = rng.integers(0, N_NODES, size=k).astype(np.uint32)
                moved = (vals["place"] & ~np.uint32(R.PODID_SCHEDULED | (R.POD_NODE_MAX << R.PODID_NODE_SHIFT))) | (
                    np.uint32(R.PODID_SCHEDULED) | (node << np.uint32(R.PODID_NODE_SHIFT)))
                vals["place"] = np.where(rng.random(k) < 0.6, moved, vals["place"] & ~np.uint32(R.PODID_SCHEDULED))
            elif tb == R.TABLE_GROUPS:
                vals["flags"] ^= np.where(rng.random(k) < 0.5, R.GRP_POD_READY, 0).astype(np.uint32)
                li = np.minimum(vals["lws_index"], max(len(t.lws) - 1, 0))
                rev = m[R.TABLE_LWS]["rev_hash"][li] if len(t.lws) else np.zeros(k, np.uint64)
                to_new = rng.random(k) < 0.5
                upd = rng.random(k) < 0.4
                vals["leader_rev_hash"] = np.where(upd, np.where(to_new, rev, rev ^ _OLD), vals["leader_rev_hash"])
                vals["wsts_rev_hash"] = np.where(upd, np.where(to_new, rev, rev ^ _OLD), vals["wsts_rev_hash"])
                vals["wsts_avail_replicas"] = np.where(rng.random(k) < 0.2, np.maximum(vals["wsts_spec_replicas"] - 1, 0),
                                                       vals["wsts_spec_replicas"])
            elif tb == R.TABLE_LWS:
                r = vals["replicas"].astype(np.int64)
                n_ = vals["sts_replicas"].astype(np.int64)
                new_r = np.maximum(r + rng.choice([-1, 0, 0, 1], size=k), 0)
                vals["replicas"] = new_r
                vals["sts_replicas"] = np.where(rng.random(k) < 0.3, np.maximum(n_ + rng.choice([-1, 1], size=k), 0), n_)
                vals["sts_partition"] = (rng.random(k) * (vals["sts_replicas"].astype(np.int64) + 1)).astype(np.int32)
                vals["sts_replicas_annotation"] = np.where(rng.random(k) < 0.75, new_r, vals["sts_replicas_annotation"])
                vals["flags"] ^= np.where(rng.random(k) < 0.2, R.LWS_UPDATED, 0).astype(np.uint32)
            cur[rows] = vals
            tick[tb] = (rows, vals)
        plan.append(tick)
    return plan


def apply_tick(tick: dict, lws, groups, pod_state, pod_ident) -> None:
    """The host mirror of one tick's patches."""
    dst = {R.TABLE_LWS: lws, R.TABLE_GROUPS: groups, R.TABLE_POD_STATE: pod_state, R.TABLE_POD_IDENT: pod_ident}
    for tb, (rows, vals) in tick.items():
        dst[tb][rows] = vals


# --------------------------------------------------------------------------- #
# the worlds
# --------------------------------------------------------------------------- #
def _group_world(label, seed, G, avg, at=0, jitter=True, mean_groups=8, p_event=0.01):
    rng = np.random.Generator(np.random.PCG64(seed))
    counts = _counts(G, avg, rng, at, jitter)
    return _assemble(label, rng, _split(G, rng, mean_groups), counts, p_event=p_event), rng


def fused_lo():
    return _group_world("fused_lo", 1, 1024, FUSED_MIN_AVG)[0]


def three_w1_below():
    return _group_world("three_w1_below", 2, 1024, FUSED_MIN_AVG - 1)[0]


def fused_hi():
    """avg exactly 256 pods with every CTA's 65 536 pods starting on a 128-pod boundary: every window
    is exactly 2048 words.  The last pod of CTA 1 — window position 65 535 — is a visited event pod."""
    rng = np.random.Generator(np.random.PCG64(3))
    G = 3 * K_FUSED_THREADS
    counts = np.full(G, FUSED_MAX_AVG, np.int64)
    p = boundary_pattern(FUSED_MAX_AVG)
    counts[K_FUSED_THREADS: K_FUSED_THREADS + len(p)] = p
    w = _assemble("fused_hi", rng, _split(G, rng, 8), counts, p_event=0.004)
    t = w.tables
    g = 2 * K_FUSED_THREADS - 1
    o = int(t.groups["lws_index"][g])
    f = int(t.lws["flags"][o]) & ~(R.LWS_RESTART_MASK | R.LWS_RECREATE_AFTER_START_ANNOT)
    t.lws["flags"][o] = f | (R.RESTART_ON_POD_RESTART << R.LWS_RESTART_SHIFT)
    t.lws["size"][o] = FUSED_MAX_AVG
    lo, hi =int(t.groups["pod_base"][g]), int(t.groups["pod_base"][g] + t.groups["pod_count"][g])
    t.pod_state[lo:hi] = (t.pod_state[lo:hi] & ~np.uint8(R.POD_PHASE_MASK)) | np.uint8(R.POD_PHASE_RUNNING)
    t.pod_state[hi - 1] |= np.uint8(R.POD_ANY_RESTART)
    w.plan = make_plan(t, rng, [R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_GROUPS, R.TABLE_LWS])
    return w


def three_w1_above():
    return _group_world("three_w1_above", 4, 300, FUSED_MAX_AVG + 1)[0]


def fused_direct():
    """A 32-pod first group, then 256-pod groups: avg stays 256, and every CTA after the first starts
    32 pods past a 128-pod boundary, so its window is 2049 words and it takes DirectBits."""
    rng = np.random.Generator(np.random.PCG64(5))
    G = 3 * K_FUSED_THREADS
    counts = np.full(G, FUSED_MAX_AVG, np.int64)
    counts[0] = 32
    p = boundary_pattern(FUSED_MAX_AVG)
    counts[K_FUSED_THREADS: K_FUSED_THREADS + len(p)] = p
    return _assemble("fused_direct", rng, _split(G, rng, 8), counts, p_event=0.004)


def fused_one_giant():
    """64-pod groups and one 70 000-pod group: its CTA's window cannot fit, the others do."""
    rng = np.random.Generator(np.random.PCG64(6))
    G = 4 * K_FUSED_THREADS
    counts = _counts(G, 64, rng, 0, jitter=False)
    giant = K_FUSED_THREADS + 44
    counts[giant] = 70_000
    gcs = _split(G, rng, 8)
    w = _assemble("fused_one_giant", rng, gcs, counts, p_event=0.003)
    t = w.tables
    o = int(t.groups["lws_index"][giant])
    f = int(t.lws["flags"][o]) & ~(R.LWS_RESTART_MASK | R.LWS_RECREATE_AFTER_START_ANNOT)
    t.lws["flags"][o] = f | (R.RESTART_ON_POD_RESTART << R.LWS_RESTART_SHIFT)
    w.plan = make_plan(t, rng, [R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_GROUPS, R.TABLE_LWS])
    return w


def _fused_pairs(label, seed, target):
    """CTA 0 visits exactly ``target`` (group, event pod) pairs; events in groups whose policy is off or
    whose visit is suppressed are there too and do not count."""
    rng = np.random.Generator(np.random.PCG64(seed))
    G = 2 * K_FUSED_THREADS
    counts = _counts(G, 64, rng, 0)
    w = _assemble(label, rng, _split(G, rng, 8), counts, p_event=0.0)
    t = w.tables
    pst = t.pod_state
    pst &= ~np.uint8(R.POD_ANY_RESTART | R.POD_DELETING)
    # a random spread of events everywhere, then visited ones in CTA 0 trimmed / topped up to `target`
    ev = rng.random(len(pst)) < 0.2
    ph = pst & R.POD_PHASE_MASK
    running_or_pending = (ph == R.POD_PHASE_PENDING) | (ph == R.POD_PHASE_RUNNING)
    pst[ev & running_or_pending] |= np.uint8(R.POD_ANY_RESTART)
    pst[ev & ~running_or_pending] |= np.uint8(R.POD_DELETING)
    _, event = pod_predicates(pst)
    pairs = visited_pairs(t.lws, t.groups, pst)
    visit_g = np.flatnonzero(pairs[:K_FUSED_THREADS] > 0)
    base, cnt = t.groups["pod_base"].astype(np.int64), t.groups["pod_count"].astype(np.int64)
    pods = np.concatenate([np.arange(base[g], base[g] + cnt[g]) for g in visit_g])
    have = pods[event[pods]]
    assert len(have) >= target, (label, len(have))
    drop = rng.choice(have, size=len(have) - target, replace=False)
    pst[drop] &= ~np.uint8(R.POD_ANY_RESTART | R.POD_DELETING)
    # (a group's visit does not depend on its own events beyond having one, so the others keep theirs)
    assert sum(visited_pairs(t.lws, t.groups, pst)[:K_FUSED_THREADS]) == target
    w.plan = make_plan(t, rng, [R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_GROUPS, R.TABLE_LWS])
    return w


def fused_pairs_1280():
    return _fused_pairs("fused_pairs_1280", 7, K_PAIR_CAP)


def fused_pairs_1281():
    return _fused_pairs("fused_pairs_1281", 8, K_PAIR_CAP + 1)


def three(label, seed, avg, G=48):
    return _group_world(label, seed, G, avg, mean_groups=4, p_event=0.002)[0]


THREE = {"three_w1_512": 512, "three_w2_513": 513, "three_w2_1024": 1024, "three_w4_1025": 1025,
         "three_w4_2048": 2048, "three_w8_2049": 2049, "three_w8_5000": 5000}


def three_w1_skew():
    """8-pod groups and one 60 000-pod group; avg stays below 16, so one lane walks ~1 900 words."""
    rng = np.random.Generator(np.random.PCG64(20))
    G = 10_000
    counts = _counts(G, 8, rng, 0, jitter=False)
    counts[5000] = 60_000
    return _assemble("three_w1_skew", rng, _split(G, rng, 8), counts, p_event=0.005)


def lws_width(label, seed, per_obj, L=8):
    """Objects with ``per_obj`` groups on average — exactly — of about two pods each."""
    rng = np.random.Generator(np.random.PCG64(seed))
    gcs = np.full(L, per_obj, np.int64)
    d = rng.integers(-7, 8, size=L // 2)
    gcs[: L // 2] += d
    gcs[L // 2: 2 * (L // 2)] -= d
    G = int(gcs.sum())
    counts = _counts(G, 2, rng, 0)
    return _assemble(label, rng, gcs, counts, p_event=0.01)


LWS_WIDTHS = {"lws_w1_64": (64, 8), "lws_w2_65": (65, 8), "lws_w2_128": (128, 8), "lws_w4_129": (129, 8),
              "lws_w4_256": (256, 8), "lws_w8_257": (257, 8), "lws_w8_512": (512, 8), "lws_w16_513": (513, 8),
              "lws_w16_1024": (1024, 8), "lws_w32_1025": (1025, 8), "lws_w32_5000": (5000, 4)}


def lws_skew():
    """Objects of about two groups and one of 20 000: W stays 1, one lane walks 2 500 words."""
    rng = np.random.Generator(np.random.PCG64(30))
    gcs = rng.integers(0, 5, size=400)
    gcs[123] = 20_000
    G = int(gcs.sum())
    return _assemble("lws_skew", rng, gcs, _counts(G, 2, rng, 0))


def lws_align(label="lws_align", seed=40, extra=0):
    """Case-5 objects for every group_base % 8 x group_count % 8.  The states put the highest bad slot,
    the rolling-step partition rsp and the walk's start hi on flag bytes 8k-1, 8k and 8k+1 of the column
    (all nine combinations over the objects), with the walk stopping below hi, at hi, or running
    through; objects with more StatefulSet replicas than group rows, and with more rows than replicas,
    are among them.  ``extra`` adds that many groups to every object (wider tiles)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    objs = []  # (gbase % 8, gc, n, states, R, surge, mu)
    combos = [(b, c) for b in range(8) for c in range(8)]
    res = [7, 0, 1]
    for i, (b, c) in enumerate(combos):
        for v in range(3):
            gc = 48 + c + extra
            r1, r2, r3 = res[(i + v) % 3], res[(i // 3 + v) % 3], res[(i // 9 + 2 * v) % 3]
            if v == 2 and i % 2:  # more replicas than rows: slots past the rows are neither ready nor updated
                n = gc + 1 + (i % 5)
            else:
                n = gc - 3 - (i % 4)
            rsp = 16 + ((r1 - b - 16) % 8)
            hi = rsp + ((r2 - b - rsp) % 8)
            mb = hi + ((r3 - b - hi) % 8)
            if n > gc:
                mb = n - 1
            st = np.full(gc, 3, np.int64)  # ready | updated
            below = rng.permutation(rsp)
            st[below[: hi - rsp]] = 2              # not ready: hi - rsp of them below rsp
            st[below[hi - rsp:]] = rng.choice([1, 3], size=rsp - (hi - rsp))
            walk = (i + v) % 3  # 0 stops below hi, 1 at hi, 2 runs through
            for s in range(rsp, min(hi + 1, gc)):
                st[s] = rng.choice([0, 3])
            if walk == 0 and hi > rsp:
                st[int(rng.integers(rsp, hi))] = 1
            elif walk == 1:
                st[hi] = 1
            if mb < gc:
                if st[mb] == 3:
                    st[mb] = 0
                st[mb + 1: min(n, gc)] = 3
            surge = 2 if (i + v) % 2 and mb + 1 - rsp >= 2 else 0
            mu = mb + 1 - rsp - surge
            objs.append((b, gc, n, st, n - surge, surge, mu))
    # lay the objects out: filler rows (owned by object 0, a Case 1 object) bring each base to its residue
    L = len(objs) + 1
    gbase, owner, states, gcs = [], [0] * 3, [3] * 3, []
    pos = 3
    for k, (b, gc, n, st, r, surge, mu) in enumerate(objs):
        pad = (b - pos) % 8
        owner += [0] * pad
        states += [3] * pad
        pos += pad
        gbase.append(pos)
        gcs.append(gc)
        owner += [k + 1] * gc
        states += list(st)
        pos += gc
    G = pos
    lws = R.aligned_empty(L, R.LWS_REC)
    lws["rev_hash"] = rng.integers(0, 1 << 63, size=L, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    lws["size"] = 2
    lws["flags"] = R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID | (R.RESTART_ON_POD_RESTART << R.LWS_RESTART_SHIFT)
    lws["flags"][0] = R.LWS_ANNOT_VALID
    lws["subgroup_size"] = 0
    lws["uid_hash"] = rng.integers(0, 1 << 63, size=L, dtype=np.uint64)
    lws["group_base"][0], lws["group_count"][0] = 0, 0
    lws["replicas"][0] = lws["sts_replicas"][0] = lws["sts_replicas_annotation"][0] = 0
    lws["partition"] = 0
    lws["sts_partition"][0] = lws["max_surge"][0] = lws["max_unavailable"][0] = 0
    for k, (b, gc, n, st, r, surge, mu) in enumerate(objs):
        i = k + 1
        lws["group_base"][i], lws["group_count"][i] = gbase[k], gc
        lws["sts_replicas"][i], lws["replicas"][i], lws["sts_replicas_annotation"][i] = n, r, r
        lws["max_surge"][i], lws["max_unavailable"][i] = surge, mu
        lws["sts_partition"][i] = n  # the walk's result is not clamped away
    owner = np.asarray(owner, np.int64)
    states = np.asarray(states, np.int64)
    counts = _counts(G, 2, rng, 0)
    kind = np.full(L, 5)
    kind[0] = 1
    pod_base = np.concatenate([[0], np.cumsum(counts)[:-1]])
    grp = _group_rows(rng, lws, kind, owner, pod_base, counts, (states & 1) != 0, (states & 2) != 0)
    # ready / updated exactly as chosen: no group without its worker StatefulSet, no stale revision
    grp["flags"] |= np.uint32(R.GRP_WSTS_FOUND | R.GRP_WSTS_LABEL_NAME_MATCH)
    grp["wsts_rev_hash"] = grp["leader_rev_hash"]
    pst, pid = _pods(rng, grp, int(counts.sum()))
    nodes, n_domains = synth.make_nodes(synth.Profile(label, L, n_nodes=N_NODES, nodes_per_domain=4), rng)
    t = synth.Tables(synth.Profile(label, L, n_nodes=N_NODES, nodes_per_domain=4), lws, grp, pst, pid, nodes, n_domains,
                     R.SWEEP_GANG)
    return FormWorld(label, t, make_plan(t, rng, [R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_GROUPS, R.TABLE_LWS]))


def no_pods():
    """Group rows with no pods at all (an empty pod table): no scan, the group pass is the sweep's
    first kernel.  Every group row changes in every tick."""
    rng = np.random.Generator(np.random.PCG64(50))
    gcs = _split(3000, rng, 6)
    return _assemble("no_pods", rng, gcs, np.zeros(int(gcs.sum()), np.int64), n_pods=0,
                     tables=[R.TABLE_GROUPS, R.TABLE_LWS], all_rows=R.TABLE_GROUPS)


def no_groups():
    """Object rows only: the LWS pass is the sweep's only kernel.  Every LWS row changes in every tick."""
    rng = np.random.Generator(np.random.PCG64(51))
    L = 5000
    lws, kind = _lws_rows(rng, np.zeros(L, np.int64), np.full(L, 4))
    lws["group_base"] = 0
    lws["sts_replicas"] = rng.integers(0, 6, size=L)  # slots without any group row
    lws["replicas"] = np.minimum(lws["replicas"], lws["sts_replicas"])
    return _assemble("no_groups", rng, np.zeros(L, np.int64), np.zeros(0, np.int64), n_pods=0, lws=lws, kind=kind,
                     tables=[R.TABLE_LWS], all_rows=R.TABLE_LWS)


def no_lws():
    """Group rows (32 pods on average: the fused form) and no LWS table: every group is BAD_TABLE."""
    rng = np.random.Generator(np.random.PCG64(52))
    G = 600
    counts = _counts(G, 32, rng, 0)
    lws = R.aligned_empty(0, R.LWS_REC)
    w = _assemble("no_lws", rng, None, counts, lws=lws, kind=np.zeros(0, np.int64),
                  tables=[R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_GROUPS])
    w.bad_groups = True
    return w


BUILDERS = {
    "fused_lo": fused_lo,
    "three_w1_below": three_w1_below,
    "fused_hi": fused_hi,
    "three_w1_above": three_w1_above,
    "fused_direct": fused_direct,
    "fused_one_giant": fused_one_giant,
    "fused_pairs_1280": fused_pairs_1280,
    "fused_pairs_1281": fused_pairs_1281,
    **{k: (lambda k=k, a=a, s=i: three(k, 10 + s, a)) for i, (k, a) in enumerate(THREE.items())},
    "three_w1_skew": three_w1_skew,
    **{k: (lambda k=k, v=v, s=i: lws_width(k, 60 + s, *v)) for i, (k, v) in enumerate(LWS_WIDTHS.items())},
    "lws_skew": lws_skew,
    "lws_align": lws_align,
    "lws_align_w8": lambda: lws_align("lws_align_w8", 41, extra=300),
    "no_pods": no_pods,
    "no_groups": no_groups,
    "no_lws": no_lws,
}

_CACHE: dict = {}


def world(label: str) -> FormWorld:
    """The world of this label (built once per process; callers copy before they mutate)."""
    if label not in _CACHE:
        _CACHE[label] = BUILDERS[label]()
    return _CACHE[label]


def expected_form(label: str) -> dict:
    """What each label promises about its table, checked by tests/test_lws_forms.py."""
    if label.startswith("fused"):
        return {"fused": True}
    if label.startswith("three_w"):
        return {"fused": False, "group_w": int(label.split("_")[1][1:])}
    if label.startswith("lws_w"):
        return {"lws_w": int(label.split("_")[1][1:])}
    return {}
