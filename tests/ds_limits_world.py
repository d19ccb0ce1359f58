"""DisaggregatedSet tables at the limits of the DS table format (include/lwse.h): 32 old revisions,
10 roles with removed ones, creation stamps in orders unlike row order (30-bit extremes, ties, partly
present revisions), bit 31 of ``drained_revs`` / ``ready_revs``, and role targets near 10^5 with
percent surges, chosen so that the planner's divisions land on or next to an integer.

Each family is a seeded function that returns ``(ds, roles, revroles)`` with contiguous ranges (role
rows and revision-role rows in DS order), as ``synth.make_ds`` does.  ``past_limits`` appends DS rows
just outside the format, which every path must report ``BAD_TABLE``."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from lws_b200 import records as R
from lws_b200 import synth

TS_MAX = (1 << 30) - 1  # the 30-bit creation-rank field of lwse_ds_revrole_rec.flags
PERCENTS = (0, 1, 33, 50, 99, 100)
STAMP_MODES = ("perm", "reversed", "equal", "tie_newest", "extremes", "partial")


@dataclass
class DsRows:
    """One DS before layout: its role rows and its (n_old_revs + 1) x n_roles revision-role rows."""
    n_spec: int
    n_old: int
    flags: int
    roles: np.ndarray  # [n] DS_ROLE_REC
    rr: np.ndarray     # [(n_old + 1) * n] DS_REVROLE_REC, revision-major
    uid: int = 0


def assemble(items) -> tuple:
    """Contiguous layout of a list of DsRows → (ds, roles, revroles)."""
    ds = R.aligned_empty(len(items), R.DS_REC)
    roles = R.aligned_empty(sum(len(x.roles) for x in items), R.DS_ROLE_REC)
    rr = R.aligned_empty(sum(len(x.rr) for x in items), R.DS_REVROLE_REC)
    rb = vb = 0
    for d, x in enumerate(items):
        n = len(x.roles)
        assert len(x.rr) == (x.n_old + 1) * n
        ds[d] = (x.uid or d + 1, rb, n, x.n_spec, vb, x.n_old, x.flags)
        roles[rb: rb + n] = x.roles
        rr[vb: vb + len(x.rr)] = x.rr
        rb, vb = rb + n, vb + len(x.rr)
    return ds, roles, rr


def split(ds, roles, rr) -> list:
    """The DsRows of every DS of a contiguous table (the inverse of ``assemble``)."""
    out = []
    for d in range(len(ds)):
        h = ds[d]
        rb, n, vb, V = int(h["role_base"]), int(h["n_roles"]), int(h["rev_base"]), int(h["n_old_revs"])
        out.append(DsRows(int(h["n_spec_roles"]), V, int(h["flags"]), roles[rb: rb + n].copy(),
                          rr[vb: vb + (V + 1) * n].copy(), int(h["uid_hash"])))
    return out


def _empty(n_spec, n_removed, V, has_new=True) -> DsRows:
    n = n_spec + n_removed
    roles = np.zeros(n, R.DS_ROLE_REC)
    roles["flags"][:n_spec] = R.ROLE_IN_SPEC
    rr = np.zeros((V + 1) * n, R.DS_REVROLE_REC)
    rr["initial_replicas"] = -1
    return DsRows(n_spec, V, R.DS_HAS_NEW_REVISION if has_new else 0, roles, rr)


def _put(x: DsRows, r, i, replicas, initial=-1, ready=None, stamp=0, nil=False):
    k = r * len(x.roles) + i
    x.rr[k] = (replicas, initial, replicas if ready is None else ready,
               R.RR_EXISTS | (R.RR_REPLICAS_NIL if nil else 0) | (int(stamp) << R.RR_TS_SHIFT))


def revision_stamps(rng, V, mode) -> np.ndarray:
    """Creation stamps of V old revisions, in row order."""
    if V == 0:
        return np.zeros(0, np.int64)
    if mode == "perm":
        return rng.permutation(V) + 1
    if mode == "reversed":
        return np.arange(V, 0, -1)
    if mode == "equal":
        return np.full(V, 5)
    if mode == "tie_newest":  # two or more revisions share the newest stamp
        s = rng.permutation(V) + 1
        if V > 1:
            s[rng.choice(V, size=min(V, int(rng.integers(2, 4))), replace=False)] = V
        return s
    if mode == "extremes":  # distinct, spanning the whole 30-bit field
        s = np.sort(rng.choice(TS_MAX - 1, size=V, replace=False) + 1)
        s[0], s[-1] = 0, TS_MAX
        return s[rng.permutation(V)]
    if mode == "partial":
        return (rng.permutation(V) + 1) * 3
    raise ValueError(mode)


def _stamp(x: DsRows, rng, st, mode):
    """Write the creation stamps into the existing rows; the new revision is newer than every old one.
    ``partial``: one revision loses some of its roles, its remaining rows get stamps below the
    revision's, and a missing row keeps a stamp above every other (rows that do not exist carry no
    stamp the kernel may read: the revision's stamp is the max over the rows that exist)."""
    n, V = len(x.roles), x.n_old
    f = x.rr["flags"].reshape(V + 1, n)
    ex = (f & R.RR_EXISTS) != 0
    ts = np.zeros((V + 1, n), np.int64)
    ts[:V] = st[:, None]
    ts[V] = min(int(st.max()) + 1, TS_MAX) if V else 1
    gone = np.zeros((V + 1, n), bool)
    live = np.flatnonzero(ex[:V].sum(axis=1) >= 2)
    if mode == "partial" and len(live):
        r = int(rng.choice(live))
        keep = int(rng.choice(np.flatnonzero(ex[r])))
        gone[r] = ex[r] & (rng.random(n) < 0.4)
        gone[r, int(rng.choice(np.flatnonzero(ex[r] & (np.arange(n) != keep))))] = True
        gone[r, keep] = False
        ts[r] = np.maximum(ts[r] - rng.integers(0, 3, size=n), 0)
        ts[r, keep] = st[r]
        ts[r, gone[r]] = TS_MAX  # rows that do not exist: their stamp is never read
        ex &= ~gone
    words = (f & np.uint32(R.RR_REPLICAS_NIL)) | np.uint32(R.RR_EXISTS) | (ts.astype(np.uint32) << np.uint32(R.RR_TS_SHIFT))
    words = np.where(ex, words, np.where(gone, ts.astype(np.uint32) << np.uint32(R.RR_TS_SHIFT), 0))
    x.rr["flags"] = words.reshape(-1).astype(np.uint32)


def _config(rng, x: DsRows, i):
    kind = int(rng.integers(0, 7))
    surge, unav, fl = [(0, 0, 0), (1, 0, 1), (2, 0, 1), (25, 0, 1 | 2), (0, 1, 1), (1, 2, 1), (50, 33, 1 | 2 | 4)][kind]
    flags = R.ROLE_IN_SPEC
    if fl & 1:
        flags |= R.ROLE_HAS_ROLLING_CONFIG
    if fl & 2:
        flags |= R.ROLE_SURGE_IS_PERCENT
    if fl & 4:
        flags |= R.ROLE_UNAVAIL_IS_PERCENT
    x.roles[i]["max_surge"], x.roles[i]["max_unavailable"], x.roles[i]["flags"] = surge, unav, flags


def random_ds(rng, n_spec, n_removed, V, stamp_mode="perm", max_rep=4) -> DsRows:
    """A mid-rollout DS with small counts: old revisions hold a share of their initial counts, removed
    roles live only in old revisions, the new revision (when it exists) is mostly stable."""
    x = _empty(n_spec, n_removed, V, has_new=rng.random() < 0.9)
    n = n_spec + n_removed
    for i in range(n_spec):
        x.roles[i]["target_replicas"] = int(rng.integers(0, 9)) if rng.random() < 0.95 else 0
        _config(rng, x, i)
    for r in range(V):
        for i in range(n):
            if rng.random() < (0.9 if i < n_spec else 0.6):
                rep = 0 if rng.random() < 0.15 else int(rng.integers(1, max_rep + 1))
                init = rep + int(rng.integers(0, 3)) if rng.random() < 0.8 else -1
                ready = max(rep - 1, 0) if rng.random() < 0.1 else rep
                nil = rng.random() < 0.02
                _put(x, r, i, 1 if nil else rep, init, ready, nil=nil)
    for i in range(n_spec, n):  # a removed role is in some old revision
        if V and not (x.rr["flags"][i::n][:V] & R.RR_EXISTS).any():
            _put(x, int(rng.integers(0, V)), i, int(rng.integers(1, max_rep + 1)))
    if x.flags & R.DS_HAS_NEW_REVISION:
        for i in range(n_spec):
            t = int(x.roles[i]["target_replicas"])
            rep = int(rng.integers(0, t + 1))
            _put(x, V, i, rep, -1, rep if rng.random() < 0.8 else max(rep - 1, 0))
    _stamp(x, rng, revision_stamps(rng, V, stamp_mode), stamp_mode)
    return x


def drain_ds(rng, n_spec, V, stamp_mode="perm") -> DsRows:
    """A DS whose next step drains exactly one replica per role: every old revision holds one replica
    per role (initial 1), target V, one new replica each, no rolling config.  The planner gives
    past = V - 1, so scaleDownOld zeroes the newest old revision (executor.go:283-302, 366-373) and
    leaves the others: which one shows the newest-first order."""
    x = _empty(n_spec, 0, V)
    x.roles["target_replicas"] = V
    for r in range(V):
        for i in range(n_spec):
            _put(x, r, i, 1, 1, 1)
    for i in range(n_spec):
        _put(x, V, i, 1, -1, 1)
    _stamp(x, rng, revision_stamps(rng, V, stamp_mode), stamp_mode)
    return x


# --------------------------------------------------------------------------------------------------
# families
# --------------------------------------------------------------------------------------------------
def v_sweep_items(seed=1) -> list:
    """V in {0, 1, 2, 31, 32} x n in {2, 3, 10}: for n = 3 and n = 10 some DS have one removed role
    (2 + 1, 9 + 1), others none (3, 10 spec roles).  The first DS is a drain DS with V = 32, n = 10."""
    rng = np.random.default_rng(seed)
    items = [drain_ds(rng, 10, 32, "perm")]
    for V in (0, 1, 2, 31, 32):
        for n in (2, 3, 10):
            for k in range(6):
                removed = 1 if (n > 2 and V > 0 and k % 2) else 0
                items.append(random_ds(rng, n - removed, removed, V, STAMP_MODES[k % len(STAMP_MODES)]))
            if V >= 2:
                items.append(drain_ds(rng, n, V, "perm"))
    return items


def stamp_items(seed=2) -> list:
    """Every stamp order on drain DS (V from 2 to 32, n in {2, 3, 10}) and on random DS."""
    rng = np.random.default_rng(seed)
    items = []
    for mode in STAMP_MODES:
        for V in (2, 5, 17, 31, 32):
            for n in (2, 3, 10):
                items.append(drain_ds(rng, n, V, mode))
            items.append(random_ds(rng, 3, 1, V, mode))
    return items


def bit31_items(seed=3) -> list:
    """V = 32 DS whose revision 31 is drained (every existing row at 0), ready (every spec role
    present and ready), or both (nil replicas: 1 for the count, 0 for cleanup)."""
    rng = np.random.default_rng(seed)
    items = []
    for n in (2, 3, 10):
        for what in ("drained", "ready", "both"):
            for make in (lambda: random_ds(rng, n, 0, 32, "perm"), lambda: drain_ds(rng, n, 32, "perm")):
                x = make()
                k = 31 * n
                f = x.rr["flags"][k: k + n]
                st = f & ~np.uint32(3)
                if what == "drained":
                    x.rr["replicas"][k: k + n] = 0
                    x.rr["ready_replicas"][k: k + n] = 0
                    x.rr["flags"][k: k + n] = st | R.RR_EXISTS
                    x.rr["flags"][k] = st[0]  # one role absent: cleanup needs one existing row only
                elif what == "ready":
                    x.rr["replicas"][k: k + n] = np.maximum(x.rr["replicas"][k: k + n], 1)
                    x.rr["ready_replicas"][k: k + n] = x.rr["replicas"][k: k + n]
                    x.rr["flags"][k: k + n] = st | R.RR_EXISTS
                else:
                    x.rr["replicas"][k: k + n] = 1
                    x.rr["ready_replicas"][k: k + n] = 1
                    x.rr["flags"][k: k + n] = st | R.RR_EXISTS | R.RR_REPLICAS_NIL
                items.append(x)
    return items


def _scaled(v, total, up):
    q, r = divmod(v * total, 100)
    return q + (1 if up and r else 0)


def planner_config(target, surge_pct, unav_pct):
    """(maxSurge, maxUnavailable) of a role with percent values (executor.go:235-260)."""
    s, u = _scaled(surge_pct, target, True), _scaled(unav_pct, target, False)
    if u > 0:
        return s, u
    return (s, 0) if s > 0 else (1, 0)


def _near(rng, c, a, k):
    """Some x in [0, c] with a·x ≡ k (mod c) when one exists, else a random x."""
    g = np.gcd(a, c)
    if k % g:
        return int(rng.integers(0, c + 1))
    a2, c2 = a // g, c // g
    x0 = ((k // g) * pow(int(a2), -1, int(c2))) % c2 if c2 > 1 else 0
    m = int(rng.integers(0, g + 1)) if g > 1 else 0
    return int(min(x0 + m * c2, c))


def rounding_items(seed=4, n_ds=240) -> list:
    """Role targets up to about 10^5 with percent maxSurge / maxUnavailable from {0, 1, 33, 50, 99,
    100}: new replica counts chosen so that cur_new·total_steps / target is an integer or one away
    from one, and old counts so that removed·total_steps / initial_old is; the step that follows
    divides next_idx·target and next_idx·initial_old by total_steps."""
    rng = np.random.default_rng(seed)
    bases = (100_000, 99_999, 100_001, 65_536, 33_333, 3 * 33_333 + 1, 50_000, 99, 100, 101, 7, 1)
    items = []
    for d in range(n_ds):
        n, V = int(rng.integers(2, 4)), int(rng.integers(1, 4))
        x = _empty(n, 0, V)
        tgt, cfg, init = [], [], []
        for i in range(n):
            t = int(bases[int(rng.integers(0, len(bases)))]) if rng.random() < 0.6 else int(rng.integers(1, 100_001))
            ps, pu = int(rng.choice(PERCENTS)), int(rng.choice(PERCENTS))
            x.roles[i] = (t, ps, pu, R.ROLE_IN_SPEC | R.ROLE_HAS_ROLLING_CONFIG | R.ROLE_SURGE_IS_PERCENT
                          | R.ROLE_UNAVAIL_IS_PERCENT)
            tgt.append(t)
            cfg.append(planner_config(t, ps, pu))
            init.append(max(t + int(rng.choice([0, 0, 1, -1, int(rng.integers(-t // 2 - 1, t // 2 + 2))])), 1))
        T = max(-(-max(init[i], tgt[i]) // (cfg[i][0] if cfg[i][0] > 0 else max(1, cfg[i][1]))) for i in range(n))
        phase = d % 3  # 0: nothing drained yet; 1: partly drained; 2: new at a boundary, old full
        for i in range(n):
            k = int(rng.choice([0, 1, -1]))
            cur_new = _near(rng, tgt[i], T, k % tgt[i])
            if phase == 0:
                cur_old = init[i]
            else:
                cur_old = init[i] - _near(rng, init[i], T, int(rng.choice([0, 1, -1])) % init[i])
            if phase == 2:
                cur_old = init[i]
            # split initial and current over the old revisions
            cuts_i = np.sort(rng.integers(0, init[i] + 1, size=V - 1))
            parts_i = np.diff(np.concatenate([[0], cuts_i, [init[i]]]))
            left = cur_old
            for r in range(V):
                rep = int(min(parts_i[r], left)) if r < V - 1 else int(left)
                left -= rep
                _put(x, r, i, rep, int(parts_i[r]) if r < V - 1 else int(init[i] - parts_i[:V - 1].sum()), rep)
            _put(x, V, i, cur_new, -1, cur_new)
        _stamp(x, rng, revision_stamps(rng, V, "perm"), "perm")
        items.append(x)
    return items


def _table(items):
    return assemble(items)


def v_sweep(seed=1):
    return _table(v_sweep_items(seed))


def stamp_orders(seed=2):
    return _table(stamp_items(seed))


def bit31(seed=3):
    return _table(bit31_items(seed))


def rounding(seed=4, n_ds=240):
    return _table(rounding_items(seed, n_ds))


FAMILIES = {"v_sweep": v_sweep, "stamps": stamp_orders, "bit31": bit31, "rounding": rounding}


def limit_items(seed=0, with_rounding=True) -> list:
    return (v_sweep_items(seed + 1) + stamp_items(seed + 2) + bit31_items(seed + 3)
            + (rounding_items(seed + 4, 60) if with_rounding else []))


def mixed(seed=5, copies=3, with_rounding=True):
    """As many ``synth.make_ds(..., fuzz=0.05)`` DS as limit DS, alternating in one table, so that the
    threads of a warp mix narrow and wide DS.  ``with_rounding=False`` leaves out the DS with
    replica counts near 10^5 (a table of one size-1 child LeaderWorkerSet per replica stays small)."""
    lim = [x for c in range(copies) for x in limit_items(seed * 10 + c, with_rounding)]
    t = synth.make_ds(len(lim), (2, 3, 10), fuzz=0.05, seed=seed)
    narrow = split(t.ds, t.roles, t.revroles)
    items = [x for pair in zip(narrow, lim) for x in pair]
    return assemble(items)


def past_limits(ds, roles, rr):
    """The table with DS rows just past the format appended: V = 33, 11 roles (10 spec + 1 removed),
    n_spec_roles > n_roles, and a revision range that ends one row past the table beside one that
    ends exactly at it.  The rows they name are appended too, and a valid DS whose range ends at the
    last row comes last.  → (ds, roles, revroles, bad): ``bad`` marks the rows past the format;
    ``ds[~bad]`` is a table the same other DS see."""
    rng = np.random.default_rng(7)
    items = split(ds, roles, rr)
    bad = [False] * len(items)
    v33 = random_ds(rng, 2, 0, 33, "perm")
    r11 = random_ds(rng, 10, 1, 3, "perm")
    sp = random_ds(rng, 3, 0, 2, "perm")
    sp.n_spec = 4
    last = random_ds(rng, 2, 0, 1, "perm")
    items += [v33, r11, sp, last]
    bad += [True, True, True, False]
    d2, ro2, rr2 = assemble(items)
    over = d2[-1:].copy()  # the last DS's range moved one row on: it ends one past the table
    over["rev_base"] += 1
    d3 = R.aligned_empty(len(d2) + 1, R.DS_REC)
    d3[:-1], d3[-1] = d2, over[0]
    return d3, ro2, rr2, np.array(bad + [True])
