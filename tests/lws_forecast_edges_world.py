"""Tables built to land on the edges of the LeaderWorkerSet rolling-update forecast
(``lws_b200/csrc/lwse_lws_forecast_kernels.cu``, ``lwse_lws_forecast_host`` / ``lwse_resident_forecast``).

An object gets ``C = max(group_count, sts_replicas, replicas + surge)`` private flag slots (surge scaled,
rounded up, clamped to [0, replicas]); objects with C above ``LWS_FORECAST_MAX_SLOTS`` are not forecast.
The slot pass rounds C up to 8, a scan turns the counts into offsets, and the engine refuses a slot sum of
2^31 or more.  One W-lane tile replays each object, W from ``pick_tile(n_groups, n_lws)``: the group
table's average, not C.  The apply walks the object's words with byte-lane masks at n' and p'; the replay
stops when nothing changes, when n' > C, or at ``min(2C + 8, LWS_FORECAST_MAX_CYCLES)`` cycles.  Grids
are capped at ``sm_count * 8`` CTAs of ``256 / W`` tiles and stride beyond.

Every world is a list of objects over a group result table; each case names the edge it tests and the
side of that edge it sits on (``below``, ``at``, ``above``), and ``tests/test_lws_forecast_edges.py``
checks that it does, with the constants below read back from the sources.  Group rows past every
object's range ("filler") set the table's average, and so the tile width, without adding slots.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from lws_b200 import records as R

# the forecast's constants (lwse_lws_forecast_kernels.cu, lwse_lws_kernels.cu, lwse_engine.cu, lwse.h)
FLAG_MASK = 0x1F               # kForecastFlagMask: the low five bits of group_out.flags
MAX_SLOTS = R.LWS_FORECAST_MAX_SLOTS
MAX_CYCLES = R.LWS_FORECAST_MAX_CYCLES
SLOT_ROUND = 8                 # (C + 7) & ~7
CAP_MUL, CAP_ADD = 2, 8        # min(2 * C + 8, MAX_CYCLES)
GRID_CTAS_PER_SM = 8           # sm_count * 8u, slot pass and replay
BLOCK = 256                    # threads per CTA, slot pass and replay
TILE_DIV = 64                  # pick_tile: groups per lane
TILE_MAX = 32
SLOT_SUM_LIMIT = 0x80000000    # the engine refuses n_slots >= 2^31
H100_SMS = 132
WIDTHS = (1, 2, 4, 8, 16, 32)

READY_OLD = 1 | 4 | 8          # STATE_READY | COUNTED | COND_READY: ready at the old revision
READY_NEW = 31                 # ready and updated
UPD = R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID | R.LWS_UPDATED  # a template change is pending
REST = R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID
# flag bytes a group pass can give (as tests/test_gpu_lws_forecast.py's _BYTES)
BYTES = np.array([0, 1, 2, 3, 4, 4 | 8, 4 | 16, 4 | 8 | 16, 1 | 4 | 8, 2 | 4 | 16, 31], np.uint32)


def pick_tile(n_groups: int, n_lws: int) -> int:
    if n_lws == 0:
        return 1
    avg = (-(-n_groups // n_lws) + TILE_DIV - 1) // TILE_DIV
    w = 1
    while w < TILE_MAX and w < avg:
        w <<= 1
    return w


def scaled_surge(v: int, pct: bool, reps: int) -> int:
    """intstr's scaled value, rounded up (small values only: no int32 extremes here)."""
    return -(-v * reps // 100) if pct else v


def slots_of(lws, n_groups: int) -> np.ndarray:
    """C per object (int64), -1 where the group range is outside the table."""
    out = np.zeros(len(lws), np.int64)
    for i, r in enumerate(lws):
        gb, gc, reps = int(r["group_base"]), int(r["group_count"]), int(r["replicas"])
        if gb + gc > n_groups:
            out[i] = -1
            continue
        s = scaled_surge(int(r["max_surge"]), bool(r["flags"] & R.LWS_SURGE_IS_PERCENT), reps)
        s = max(min(s, reps), 0)
        out[i] = max(gc, int(r["sts_replicas"]), reps + s, 0)
    return out


def round8(c):
    return (np.asarray(c, np.int64) + SLOT_ROUND - 1) // SLOT_ROUND * SLOT_ROUND


def cycle_cap(c):
    return np.minimum(CAP_MUL * np.asarray(c, np.int64) + CAP_ADD, MAX_CYCLES)


def cap_rows(reps: int, u: int, n: int | None = None) -> np.ndarray:
    """The closed-form trajectory of a rollout from rest (every group ready at the old revision, a pending
    template change, integer maxUnavailable u, maxSurge 0, partition 0): row k is
    (max(R - u(k+1), 0), R, R, min(uk, R)) for k = 0 .. ceil(R / u), ending DONE; the first n rows."""
    k = np.arange(-(-reps // u) + 1 if n is None else n, dtype=np.int64)
    rows = np.zeros(len(k), R.LWS_FORECAST_STEP)
    rows["partition"] = np.maximum(reps - u * (k + 1), 0)
    rows["sts_replicas"] = reps
    rows["ready_replicas"] = reps
    rows["updated_replicas"] = np.minimum(u * k, reps)
    return rows


@dataclass
class Case:
    name: str
    edge: str
    side: str          # below | at | above
    row: int           # the object's row
    value: int = 0     # the quantity on the edge (C, word count, n', ...), as declared


@dataclass
class World:
    label: str
    lws: np.ndarray
    group_out: np.ndarray
    owner: np.ndarray  # per group row: the object it is built for (filler: object 0)
    cases: list = field(default_factory=list)
    notes: dict = field(default_factory=dict)

    def of(self, name):
        return [c for c in self.cases if c.name == name]

    def groups(self):
        """Group rows whose group pass gives these flag bytes (for the resident tables)."""
        from lws_forecast_ref import _rows_from_bytes

        return _rows_from_bytes(self.group_out["flags"] & FLAG_MASK, self.owner, self.lws)


class Builder:
    def __init__(self, label: str, seed: int = 0, noise: bool = True):
        self.label, self.rows, self.bytes, self.owner, self.cases = label, [], [], [], []
        self.rng = np.random.default_rng(seed)
        self.noise = noise
        self.n_groups = 0

    def add(self, reps, gc, sts, surge=0, mu=1, flags=UPD, byte=READY_OLD, s_pct=False, u_pct=False, part=0,
            sts_part=None, annot=None, base=None, size=1):
        i = len(self.rows)
        r = np.zeros(1, R.LWS_REC)[0]
        r["replicas"], r["group_count"], r["sts_replicas"] = reps, gc, sts
        r["max_surge"], r["max_unavailable"], r["partition"] = surge, mu, part
        r["sts_partition"] = (reps if flags & R.LWS_UPDATED else 0) if sts_part is None else sts_part
        r["sts_replicas_annotation"] = reps if annot is None else annot
        r["size"], r["rev_hash"], r["uid_hash"] = size, 0x5EED_0000_0000_0001 + 7919 * i, 1 + i
        f = flags | (R.LWS_SURGE_IS_PERCENT if s_pct else 0) | (R.LWS_UNAVAIL_IS_PERCENT if u_pct else 0)
        r["flags"] = f
        if base is None:
            r["group_base"] = self.n_groups
            b = np.full(gc, byte, np.uint32) if np.isscalar(byte) else np.asarray(byte, np.uint32)
            assert len(b) == gc
            self.bytes.append(b)
            self.owner.append(np.full(gc, i, np.int64))
            self.n_groups += gc
        else:
            r["group_base"] = base
        self.rows.append(r)
        return i

    def case(self, name, edge, side, row, value=0):
        self.cases.append(Case(name, edge, side, row, value))
        return row

    def filler(self, n, byte=None):
        """n group rows no object owns (random group-pass bytes unless ``byte``)."""
        b = self.rng.choice(BYTES, n) if byte is None else np.full(n, byte, np.uint32)
        self.bytes.append(b.astype(np.uint32))
        self.owner.append(np.zeros(n, np.int64))
        self.n_groups += n

    def fill_to_width(self, w, n_lws=None, extra=0):
        """Filler up to 64 w groups per object plus ``extra`` rows: pick_tile gives w, or 2 w when
        0 < extra <= n_lws (the average is then 64 w + 1).  n_lws defaults to the objects so far."""
        n = len(self.rows) if n_lws is None else n_lws
        want = TILE_DIV * w * n + extra
        assert want >= self.n_groups, (self.label, want, self.n_groups)
        self.filler(want - self.n_groups)

    def world(self, **notes) -> World:
        lws = R.aligned_empty(len(self.rows), R.LWS_REC)
        lws[:] = np.array(self.rows, R.LWS_REC) if self.rows else lws
        b = np.concatenate(self.bytes) if self.bytes else np.zeros(0, np.uint32)
        go = R.aligned_empty(len(b), R.GROUP_OUT)
        go[:] = np.zeros(1, R.GROUP_OUT)
        hi = self.rng.integers(0, 1 << 9, len(b), dtype=np.uint32) << 5 if self.noise else 0
        go["flags"] = b | hi  # bits above the flag mask are not the forecast's
        own = np.concatenate(self.owner) if self.owner else np.zeros(0, np.int64)
        return World(self.label, lws, go, own, self.cases, notes)


# --------------------------------------------------------------------------- #
# 1. C at the slot cap, through each term of C
# --------------------------------------------------------------------------- #
SIDES = {-1: "below", 0: "at", 1: "above"}


def _pct_reps(target: int, pct: int) -> int:
    """replicas R with R + ceil(R * pct / 100) == target while R + floor(R * pct / 100) == target - 1."""
    r = target * 100 // (100 + pct)
    for reps in range(r - 4, r + 5):
        if reps + scaled_surge(pct, True, reps) == target and (reps * pct) % 100:
            return reps
    raise ValueError((target, pct))


def slot_cap(terms=("groups", "sts", "surge", "percent", "clamp")) -> World:
    """Every object replays one cycle (or none) and stops: the objects at or below the cap are cheap for
    the reference apart from their C slots."""
    b = Builder("slot_cap")
    for term in terms:
        for d in (-1, 0, 1):
            if term == "groups":  # real group rows, ready at the new revision; replicas a little lower
                c = MAX_SLOTS + d
                i = b.add(c - 5, c, c - 5, flags=REST, byte=READY_NEW)
            elif term == "sts":
                c = MAX_SLOTS + d
                i = b.add(4, 4, c, flags=REST, byte=READY_NEW)
            elif term == "surge":
                c = MAX_SLOTS + d
                i = b.add(c - 3, 4, c - 3, surge=3, flags=REST, byte=READY_NEW)
            elif term == "percent":  # 1 % of R, rounded up across the edge
                c = MAX_SLOTS + d
                i = b.add(_pct_reps(c, 1), 4, _pct_reps(c, 1), surge=1, s_pct=True, flags=REST, byte=READY_NEW)
            else:  # maxSurge R + 7 clamped to R: C = 2R is even, so the sides are 2^20 -/+ 2
                c = MAX_SLOTS + 2 * d
                i = b.add(c // 2, 4, c // 2, surge=c // 2 + 7, flags=REST, byte=READY_NEW)
            b.case(f"{term}_{SIDES[d]}", "C <= MAX_SLOTS", SIDES[d], i, c)
    return b.world()


# --------------------------------------------------------------------------- #
# 2. words and lanes, for every tile width
# --------------------------------------------------------------------------- #
def words(w: int) -> World:
    """Rollouts from rest with C = 8 (nw - 1) + m for nw in {w - 1, w, w + 1} and m in 1..8 (C mod 8 takes
    every value), C carried by replicas + surge over group_count = replicas (surge slots past the
    groups).  maxUnavailable 1 walks p' through every slot, and n' sits at C while the surge is up and at
    replicas after it.  Filler sets the table's average to 64 w."""
    b = Builder(f"words_{w}", seed=w)
    for nw in (w - 1, w, w + 1):
        if nw < 1:
            continue
        for m in range(1, 9):
            c = 8 * (nw - 1) + m
            s = (m + nw) % 3 if c > 2 else 0
            reps = c - s
            i = b.add(reps, reps, reps, surge=s, mu=1 + (m == 5 and reps > 4))
            b.case(f"nw{nw}_m{m % 8}", "words = W -/+ 1, C mod 8", SIDES[(nw > w) - (nw < w)], i, c)
    b.fill_to_width(w)
    return b.world(width=w)


# --------------------------------------------------------------------------- #
# 3. tile thresholds, and the mixed tables
# --------------------------------------------------------------------------- #
TILE_AVGS = tuple(a for k in (1, 2, 4, 8, 16) for a in (64 * k, 64 * k + 1)) + (64 * 32 * 4,)


def _rollouts(b: Builder, n: int, seed: int):
    rng = np.random.default_rng(seed)
    for j in range(n):
        reps = int(rng.integers(1, 20))
        kind = j % 4
        if kind == 0:
            b.add(reps, reps, reps, mu=1)
        elif kind == 1:
            b.add(reps, reps, reps, surge=int(rng.integers(1, 4)), mu=int(rng.integers(0, 3)))
        elif kind == 2:
            b.add(reps, reps + 2, reps, surge=25, s_pct=True, mu=30, u_pct=True)
        else:
            b.add(reps, reps, reps + 3, flags=REST, byte=rng.choice(BYTES, reps))


def tile(avg: int) -> World:
    """16 objects over a table whose ceil(n_groups / n_lws) is ``avg``."""
    b = Builder(f"tile_{avg}", seed=avg)
    _rollouts(b, 16, avg)
    n = len(b.rows)
    b.filler(avg * n - b.n_groups)
    return b.world(avg=avg)


def w1_sts() -> World:
    """A W = 1 table where some objects' C is far above their group count, carried by sts_replicas: one
    lane walks 2^17 words for the largest."""
    b = Builder("w1_sts", seed=11)
    _rollouts(b, 40, 11)
    for c in (5000, 65536 + 3, MAX_SLOTS):
        i = b.add(4, 4, c, flags=REST, byte=READY_NEW)
        b.case(f"sts_{c}", "C >> group_count at W = 1", "above", i, c)
    i = b.add(6, 3, 900, surge=2, flags=UPD, byte=READY_OLD)
    b.case("sts_rollout", "C >> group_count at W = 1", "above", i, 900)
    return b.world()


def w32_small() -> World:
    """A W = 32 table where most objects have C <= 8: 31 lanes of their tile hold no word."""
    b = Builder("w32_small", seed=12)
    for c in range(1, 9):
        for s in (0, 1):
            if c - s < 1:
                continue
            i = b.add(c - s, c - s, c - s, surge=s, mu=1)
            b.case(f"c{c}_s{s}", "C <= 8 at W = 32", "below", i, c)
    i = b.add(4, 4, 4, mu=1, byte=rng_bytes(4, 12))
    b.case("c4_mixed", "C <= 8 at W = 32", "below", i, 4)
    b.fill_to_width(32)
    return b.world()


def rng_bytes(n, seed):
    return np.random.default_rng(seed).choice(BYTES, n)


# --------------------------------------------------------------------------- #
# 4. n' > C, 5. the cycle cap, 6. group ranges, 7. degenerate objects
# --------------------------------------------------------------------------- #
def n_over_c() -> World:
    """fuzzed()'s construction: a pending template change, maxSurge = replicas and a negative integer
    maxUnavailable -k, so the first pass asks for n' = 2R + k.  sts_replicas 2R + k - d makes C = n' - d:
    d = 0 lands n' on C (the replay goes on), d = 1 one past it (UNFINISHED, no cycle)."""
    b = Builder("n_over_c")
    for reps, k in ((5, 1), (8, 3), (13, 2), (64, 5)):
        for d in (0, 1):
            n2 = 2 * reps + k
            i = b.add(reps, reps, n2 - d, surge=reps, mu=-k)
            b.case(f"r{reps}_k{k}_{'at' if d == 0 else 'above'}", "n' <= C", "at" if d == 0 else "above", i, n2)
    return b.world()


CAP_REPLICAS = MAX_CYCLES + 4  # its rollout needs R + 1 cycles


def cycle_cap_world() -> World:
    """One rollout from rest that is still changing after MAX_CYCLES cycles (cap_rows with u = 1), beside
    the same rollout at 2^16 - 2 replicas, which ends DONE one cycle below the cap."""
    b = Builder("cycle_cap")
    i = b.add(CAP_REPLICAS, CAP_REPLICAS, CAP_REPLICAS, mu=1)
    b.case("cap", "cycles <= MAX_CYCLES", "above", i, CAP_REPLICAS + 1)
    i = b.add(MAX_CYCLES - 2, MAX_CYCLES - 2, MAX_CYCLES - 2, mu=1)
    b.case("below_cap", "cycles <= MAX_CYCLES", "below", i, MAX_CYCLES - 1)
    return b.world()


def ranges() -> World:
    """group_base + group_count at n_groups (runs) and one past it (BAD_TABLE), an empty range at
    n_groups (runs), and group_base 0xFFFFFFFF with one group, whose 32-bit sum wraps to 0 (BAD_TABLE)."""
    b = Builder("ranges", seed=6)
    _rollouts(b, 6, 6)
    b.filler(23)
    a = b.add(7, 5, 7, mu=1)  # its five group rows end the table
    G = b.n_groups
    z = b.add(3, 0, 3, mu=1, base=G)
    p = b.add(7, 6, 7, mu=1, base=G - 5)
    wrap = b.add(4, 1, 4, mu=1, base=0xFFFFFFFF)
    b.case("end_at", "group_base + group_count <= n_groups", "at", a, G)
    b.case("empty_at_end", "group_base + group_count <= n_groups", "at", z, G)
    b.case("end_past", "group_base + group_count <= n_groups", "above", p, G + 1)
    b.case("u32_wrap", "group_base + group_count <= n_groups", "above", wrap, 1 << 32)
    return b.world()


def degenerate() -> World:
    b = Builder("degenerate", seed=7)
    i = b.add(0, 0, 0, flags=0)
    b.case("c0", "C = 0", "at", i, 0)
    i = b.add(0, 0, 0, flags=REST)
    b.case("c0_sts", "C = 0", "at", i, 0)
    i = b.add(0, 0, 0, flags=UPD, surge=3)
    b.case("c0_updated", "C = 0", "at", i, 0)
    for reps, gc, fl in ((5, 5, UPD), (5, 5, REST), (3, 9, UPD), (9, 3, REST), (0, 4, UPD)):
        i = b.add(reps, gc, reps, flags=fl, byte=0)
        b.case(f"zeros_r{reps}_g{gc}", "zero bytes", "at", i, max(reps, gc))
    return b.world()


# --------------------------------------------------------------------------- #
# 8. the slot sum
# --------------------------------------------------------------------------- #
SUM_OBJECTS = SLOT_SUM_LIMIT // MAX_SLOTS  # 2048


def slot_sum(refused: bool) -> World:
    """2048 objects whose C = 2^20 is carried by sts_replicas over 4 groups (one cycle each); the last one
    has C = 2^20 - 8 unless ``refused``.  Filler makes the tiles 32 lanes wide."""
    b = Builder("slot_sum_" + ("refused" if refused else "runs"), noise=False)
    for j in range(SUM_OBJECTS):
        c = MAX_SLOTS - (0 if refused or j < SUM_OBJECTS - 1 else SLOT_ROUND)
        b.add(4, 4, c, flags=REST, byte=READY_NEW)
    b.case("sum", "slot sum < 2^31", "at" if refused else "below", SUM_OBJECTS - 1,
           SLOT_SUM_LIMIT - (0 if refused else SLOT_ROUND))
    b.fill_to_width(16, extra=1)
    return b.world()


def slot_sum_objects() -> World:
    """The two kinds of object of the slot-sum worlds, alone: the reference runs these."""
    b = Builder("slot_sum_objects", noise=False)
    b.add(4, 4, MAX_SLOTS, flags=REST, byte=READY_NEW)
    b.add(4, 4, MAX_SLOTS - SLOT_ROUND, flags=REST, byte=READY_NEW)
    return b.world()


# --------------------------------------------------------------------------- #
# 9. grid strides, 10. trajectory capacity
# --------------------------------------------------------------------------- #
def grid_objects(sms: int, w: int) -> int:
    return sms * GRID_CTAS_PER_SM * (BLOCK // w) + 3


def grid(sms: int, w: int) -> World:
    """Just more objects than the replay grid has tiles at width w (and, for w = 1, than the slot pass's
    grid has threads): objects of one to three groups, at rest or (every 50th, and the last four) a
    rollout.  For w > 1 filler gives the least average that picks w: 32 w + 1 groups."""
    n = grid_objects(sms, w)
    j = np.arange(n, dtype=np.int64)
    roll = (j % 50 == 0) | (j >= n - 4)
    reps = np.where(roll, 1 + j % 3, 1 + j % 2)
    lws = R.aligned_empty(n, R.LWS_REC)
    lws[:] = np.zeros(1, R.LWS_REC)
    for k in ("replicas", "group_count", "sts_replicas", "sts_replicas_annotation"):
        lws[k] = reps
    lws["sts_partition"] = np.where(roll, reps, 0)
    lws["group_base"] = np.cumsum(reps) - reps
    lws["max_surge"] = np.where(roll, j % 2, 0)
    lws["max_unavailable"] = 1
    lws["size"] = 1
    lws["rev_hash"] = 0x5EED_0000_0000_0001 + 7919 * j
    lws["uid_hash"] = 1 + j
    lws["flags"] = np.where(roll, UPD, REST)
    owner = np.repeat(j, reps)
    rng = np.random.default_rng(w)
    b = np.where(roll[owner], READY_OLD, np.where(owner % 3 != 0, READY_NEW, rng.choice(BYTES, len(owner))))
    G = int(reps.sum()) if w == 1 else (TILE_DIV * (w // 2) + 1) * n
    go = R.aligned_empty(G, R.GROUP_OUT)
    go[:] = np.zeros(1, R.GROUP_OUT)
    go["flags"][: len(b)] = b
    own = np.zeros(G, np.int64)
    own[: len(owner)] = owner
    return World(f"grid_{w}", lws, go, own, [Case("grid", "objects > SMs * 8 * 256 / W", "above", n - 1, n)],
                 {"width": w, "sms": sms})


def capacity() -> World:
    """Rollouts (rows) with objects of no rows between them."""
    b = Builder("capacity", seed=10)
    for j in range(12):
        reps = 2 + j % 5
        b.add(reps, reps, reps, mu=1 + j % 2)
        for _ in range(j % 3):
            b.add(reps, reps, reps, flags=REST, byte=READY_NEW)  # at rest: no row
    return b.world()


SMALL = ("degenerate", "n_over_c", "ranges", "capacity", "w32_small") + tuple(f"words_{w}" for w in WIDTHS) \
    + tuple(f"tile_{a}" for a in TILE_AVGS)
BUILDERS = {
    "degenerate": degenerate, "n_over_c": n_over_c, "ranges": ranges, "capacity": capacity,
    "w32_small": w32_small, "w1_sts": w1_sts, "slot_cap": slot_cap, "cycle_cap": cycle_cap_world,
    "slot_sum_objects": slot_sum_objects,
    **{f"words_{w}": (lambda w=w: words(w)) for w in WIDTHS},
    **{f"tile_{a}": (lambda a=a: tile(a)) for a in TILE_AVGS},
}
_CACHE = {}


def world(label: str) -> World:
    if label not in _CACHE:
        _CACHE[label] = BUILDERS[label]()
    return _CACHE[label]
