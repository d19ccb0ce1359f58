"""Fixed-width record tables of the engine — numpy mirrors of ``include/lwse.h``.

Every dtype below has exactly the layout of the C struct of the same name; the
``tests/test_abi.py`` suite checks the sizes and field offsets against the
header through the compiled library.  Field meaning and the reference lines
each field comes from are documented once, in the header.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

ABI_VERSION = 2
NONE = 0xFFFFFFFF
NODE_NOT_FOUND = 0xFFFFFFFE

# --------------------------------------------------------------------------- #
# input records
# --------------------------------------------------------------------------- #
LWS_REC = np.dtype(
    [
        ("rev_hash", "<u8"),
        ("size", "<i4"),
        ("flags", "<u4"),
        ("replicas", "<i4"),
        ("partition", "<i4"),
        ("max_surge", "<i4"),
        ("max_unavailable", "<i4"),
        ("sts_replicas", "<i4"),
        ("sts_partition", "<i4"),
        ("sts_replicas_annotation", "<i4"),
        ("subgroup_size", "<i4"),
        ("uid_hash", "<u8"),
        ("group_base", "<u4"),
        ("group_count", "<u4"),
    ],
    align=False,
)
assert LWS_REC.itemsize == 64

LWS_SURGE_IS_PERCENT = 1 << 0
LWS_UNAVAIL_IS_PERCENT = 1 << 1
LWS_STS_EXISTS = 1 << 2
LWS_UPDATED = 1 << 3
LWS_ANNOT_VALID = 1 << 4
LWS_RESTART_SHIFT = 5
LWS_RESTART_MASK = 3 << 5
LWS_RECREATE_AFTER_START_ANNOT = 1 << 7
LWS_STARTUP_LEADER_READY = 1 << 8
LWS_EXCLUSIVE_TOPOLOGY = 1 << 9
LWS_SUBGROUP_LEADER_EXCLUDED = 1 << 10
LWS_GROUP_LABEL_INVALID = 1 << 11
LWS_INTSTR_INVALID = 1 << 12
LWS_IRREGULAR = 1 << 13

RESTART_NONE = 0
RESTART_ON_POD_RESTART = 1
RESTART_AFTER_START = 2

GROUP_REC = np.dtype(
    [
        ("leader_rev_hash", "<u8"),
        ("wsts_rev_hash", "<u8"),
        ("wsts_spec_replicas", "<i4"),
        ("wsts_avail_replicas", "<i4"),
        ("leader_uid_hash", "<u4"),
        ("wsts_uid_hash", "<u4"),
        ("wsts_owner_uid_hash", "<u4"),
        ("leader_node", "<u4"),
        ("pod_base", "<u4"),
        ("pod_count", "<u4"),
        ("lws_index", "<u4"),
        ("flags", "<u4"),
        ("reserved", "<u4", (2,)),
    ],
    align=False,
)
assert GROUP_REC.itemsize == 64

GRP_POD_PRESENT = 1 << 0
GRP_POD_NAME_MATCH = 1 << 1
GRP_POD_RUNNING = 1 << 2
GRP_POD_READY = 1 << 3
GRP_POD_DELETING = 1 << 4
GRP_WSTS_LABEL_NAME_MATCH = 1 << 5
GRP_WSTS_FOUND = 1 << 6
GRP_WSTS_REV_SETTLED = 1 << 7
GRP_WSTS_OWNER_IS_POD = 1 << 8
GRP_WSTS_OWNER_NAME_MATCH = 1 << 9
GRP_MISTAKEN_ANNOTATION = 1 << 10
GRP_REVISION_EXISTS = 1 << 11

POD_STATE = np.dtype("u1")  # lwse_pod_state: the hot byte column
POD_IDENT = np.dtype([("rev_hash", "<u8"), ("owner_uid_hash", "<u4"), ("place", "<u4")], align=False)
assert POD_IDENT.itemsize == 16


def pod_ident_table(rev_hash: np.ndarray, owner_uid_hash: np.ndarray, place: np.ndarray | int = 0) -> np.ndarray:
    """Build the identity column from 64-bit revision hashes, 32-bit owner uid hashes and the
    ``place`` words (PODID_NAME_OK | PODID_SCHEDULED | node << PODID_NODE_SHIFT)."""
    t = aligned_empty(len(rev_hash), POD_IDENT)
    t["rev_hash"] = np.asarray(rev_hash, dtype=np.uint64)
    t["owner_uid_hash"] = owner_uid_hash
    t["place"] = place
    return t


POD_PHASE_MASK = 3
POD_PHASE_PENDING = 1
POD_PHASE_RUNNING = 2
POD_ANY_RESTART = 1 << 2
POD_DELETING = 1 << 3
POD_OWNER_SHIFT = 4
POD_OWNER_MASK = 3 << 4
POD_OWNER_NONE, POD_OWNER_POD, POD_OWNER_STS, POD_OWNER_OTHER = 0, 1, 2, 3
POD_OWNER_NAME_MATCH = 1 << 6
POD_IS_LEADER = 1 << 7
PODID_NAME_OK = 1 << 0
PODID_SCHEDULED = 1 << 1
PODID_NODE_SHIFT = 10
POD_NODE_MAX = (1 << 22) - 1


def occupancy_of(pod_ident: np.ndarray, n_nodes: int) -> np.ndarray:
    """Scheduled pods per node of an identity column (what the engine counts at load)."""
    place = pod_ident["place"]
    sched = (place & PODID_SCHEDULED) != 0
    node = (place[sched] >> PODID_NODE_SHIFT).astype(np.int64)
    return np.bincount(node[node < n_nodes], minlength=n_nodes).astype(np.uint32)


NODE_REC = np.dtype(
    [("topo_value_hash", "<u8"), ("domain_id", "<u4"), ("capacity", "<u2"), ("flags", "<u2")],
    align=False,
)
assert NODE_REC.itemsize == 16
NODE_HAS_TOPOLOGY = 1 << 0
NODE_SCHEDULABLE = 1 << 1

# --------------------------------------------------------------------------- #
# output records
# --------------------------------------------------------------------------- #
LWS_OUT = np.dtype(
    [
        ("sts_partition", "<i4"),
        ("sts_replicas", "<i4"),
        ("sts_max_unavailable", "<i4"),
        ("ready_replicas", "<i4"),
        ("updated_replicas", "<i4"),
        ("min_member", "<i4"),
        ("flags", "<u4"),
        ("unready_replicas", "<i4"),
    ],
    align=False,
)
assert LWS_OUT.itemsize == 32

LOUT_RUP_ERROR = 1 << 0
LOUT_STATUS_ERROR = 1 << 1
LOUT_COND_SHIFT = 2
LOUT_COND_MASK = 3 << 2
LOUT_UPDATE_DONE = 1 << 4
LOUT_EVENT_SHIFT = 5
LOUT_EVENT_MASK = 3 << 5
LOUT_IRREGULAR = 1 << 7
LOUT_BAD_TABLE = 1 << 8
COND_PROGRESSING, COND_AVAILABLE, COND_UPDATE_IN_PROGRESS = 0, 1, 2
EVENT_NONE, EVENT_DELETE_ONE, EVENT_DELETE_RANGE = 0, 1, 2

GROUP_OUT = np.dtype(
    [("flags", "<u4"), ("first_trigger", "<u4"), ("worker_replicas", "<i4"), ("domain_id", "<u4")],
    align=False,
)
assert GROUP_OUT.itemsize == 16

GOUT_STATE_READY = 1 << 0
GOUT_STATE_UPDATED = 1 << 1
GOUT_COUNTED = 1 << 2
GOUT_COND_READY = 1 << 3
GOUT_COND_UPDATED = 1 << 4
GOUT_PENDING = 1 << 5
GOUT_DELETE_LEADER = 1 << 6
GOUT_LEADER_DELETING = 1 << 7
GOUT_RESTART_ERROR = 1 << 8
GOUT_CREATE_WSTS = 1 << 9
GOUT_WAIT_SCHEDULE = 1 << 10
GOUT_TOPOLOGY_ERROR = 1 << 11
GOUT_REQUEUE_REVISION = 1 << 12
GOUT_CREATE_PODGROUP = 1 << 13
GOUT_BAD_TABLE = 1 << 14

SWEEP_GANG = 1 << 0
SWEEP_SKIP_GROUP_PASS = 1 << 1
SWEEP_SKIP_LWS_PASS = 1 << 2
SWEEP_SKIP_POD_SCAN = 1 << 3
SWEEP_REUSE_POD_IDENT = 1 << 4
SWEEP_PLACE_GROUPED = 1 << 5
SWEEP_PLACE_SCAN = 1 << 6
EXCHANGE_LAGGED = 1 << 16

# --------------------------------------------------------------------------- #
# placement
# --------------------------------------------------------------------------- #
PLACE_REQ = np.dtype(
    [
        ("priority", "<u8"),
        ("group_key", "<u8"),
        ("group", "<u4"),
        ("ns", "<u4"),
        ("size", "<i4"),
        ("leader_node", "<u4"),
    ],
    align=False,
)
assert PLACE_REQ.itemsize == 32
PLACE_OUT = np.dtype(
    [("domain_id", "<u4"), ("leader_node", "<u4"), ("flags", "<u4"), ("score", "<u4")], align=False
)
assert PLACE_OUT.itemsize == 16
PLACE_PLACED = 1 << 0
PLACE_PINNED = 1 << 1
PLACE_CONFLICT = 1 << 2
PLACE_UNSCHEDULABLE = 1 << 3

# --------------------------------------------------------------------------- #
# DisaggregatedSet
# --------------------------------------------------------------------------- #
DS_MAX_ROLES = 10
DS_REC = np.dtype(
    [
        ("uid_hash", "<u8"),
        ("role_base", "<u4"),
        ("n_roles", "<u4"),
        ("n_spec_roles", "<u4"),
        ("rev_base", "<u4"),
        ("n_old_revs", "<u4"),
        ("flags", "<u4"),
    ],
    align=False,
)
assert DS_REC.itemsize == 32
DS_HAS_NEW_REVISION = 1 << 0

DS_ROLE_REC = np.dtype(
    [("target_replicas", "<i4"), ("max_surge", "<i4"), ("max_unavailable", "<i4"), ("flags", "<u4")],
    align=False,
)
assert DS_ROLE_REC.itemsize == 16
ROLE_SURGE_IS_PERCENT = 1 << 0
ROLE_UNAVAIL_IS_PERCENT = 1 << 1
ROLE_HAS_ROLLING_CONFIG = 1 << 2
ROLE_IN_SPEC = 1 << 3
ROLE_SURGE_INVALID = 1 << 4
ROLE_UNAVAIL_INVALID = 1 << 5

DS_REVROLE_REC = np.dtype(
    [("replicas", "<i4"), ("initial_replicas", "<i4"), ("ready_replicas", "<i4"), ("flags", "<u4")],
    align=False,
)
assert DS_REVROLE_REC.itemsize == 16
RR_EXISTS = 1 << 0
RR_REPLICAS_NIL = 1 << 1
RR_TS_SHIFT = 2

DS_OUT = np.dtype(
    [("flags", "<u4"), ("drained_revs", "<u4"), ("ready_revs", "<u4"), ("reserved", "<u4")], align=False
)
assert DS_OUT.itemsize == 16
DOUT_ROLLING = 1 << 0
DOUT_INIT = 1 << 1
DOUT_STABLE = 1 << 2
DOUT_STEP = 1 << 3
DOUT_COMPLETE = 1 << 4
DOUT_NEW_READY = 1 << 5
DOUT_BAD_TABLE = 1 << 6
DS_MAX_OLD_REVS = 32

DS_ROLE_OUT = np.dtype([("next_old", "<i4"), ("next_new", "<i4")], align=False)
assert DS_ROLE_OUT.itemsize == 8
DS_REVROLE_OUT = np.dtype("<i4")

# lwse_ds_link: revision-role row → its child's row in the resident LWS table (TABLE_DS_LINKS)
DS_LINK = np.dtype([("lws_uid_hash", "<u8"), ("lws_row", "<u4"), ("reserved", "<u4")], align=False)
assert DS_LINK.itemsize == 16

# rollout forecast (lwse_ds_forecast_*): per DS, per role row; trajectory rows are DS_ROLE_OUT {old, new}
DS_FORECAST = np.dtype(
    [("flags", "<u4"), ("cycles", "<u4"), ("step_base", "<u4"), ("n_steps", "<u4")], align=False
)
assert DS_FORECAST.itemsize == 16
DS_FORECAST_ROLE = np.dtype(
    [("peak_replicas", "<i4"), ("floor_available", "<i4"), ("final_old", "<i4"), ("final_new", "<i4")], align=False
)
assert DS_FORECAST_ROLE.itemsize == 16
DSF_ROLLING = 1 << 0
DSF_WAITING = 1 << 1
DSF_DONE = 1 << 2
DSF_UNFINISHED = 1 << 3
DSF_TRUNCATED = 1 << 4
DSF_BAD_TABLE = 1 << 6
DS_FORECAST_MAX_CYCLES = 65536

# DS rollout what-if (lwse_resident_ds_rollout_whatif): one proposal per DS edit; with DSP_ROLES its role rows
# are rows [i * DS_MAX_ROLES, i * DS_MAX_ROLES + n_roles) of the query's role table
DS_PROPOSAL = np.dtype([("ds", "<u4"), ("flags", "<u4")], align=False)
assert DS_PROPOSAL.itemsize == 8
DSP_NEW_REVISION = 1 << 0
DSP_ROLES = 1 << 1
DS_WHATIF_MAX_PROPOSALS = (2**32 - 1) // ((DS_MAX_OLD_REVS + 1) * DS_MAX_ROLES)

# rolling-update forecast of the LeaderWorkerSets (lwse_lws_forecast_*): per LWS, and the trajectory rows
LWS_FORECAST = np.dtype(
    [("flags", "<u4"), ("cycles", "<u4"), ("step_base", "<u4"), ("n_steps", "<u4"), ("peak_sts_replicas", "<i4"),
     ("floor_ready", "<i4"), ("final_partition", "<i4"), ("final_replicas", "<i4")], align=False
)
assert LWS_FORECAST.itemsize == 32
LWS_FORECAST_STEP = np.dtype(
    [("partition", "<i4"), ("sts_replicas", "<i4"), ("ready_replicas", "<i4"), ("updated_replicas", "<i4")],
    align=False
)
assert LWS_FORECAST_STEP.itemsize == 16
LWSF_ROLLING = 1 << 0
LWSF_WAITING = 1 << 1
LWSF_DONE = 1 << 2
LWSF_UNFINISHED = 1 << 3
LWSF_TRUNCATED = 1 << 4
LWSF_HELD = 1 << 5
LWSF_BAD_TABLE = 1 << 6
LWSF_NOT_FORECAST = 1 << 7
LWS_FORECAST_MAX_CYCLES = 65536
LWS_FORECAST_MAX_SLOTS = 1 << 20


# --------------------------------------------------------------------------- #
# ctypes bundles (lwse_lws_tables / lwse_ds_tables / lwse_config)
# --------------------------------------------------------------------------- #
class LwsTables(C.Structure):
    _fields_ = [
        ("lws", C.c_void_p),
        ("n_lws", C.c_uint32),
        ("groups", C.c_void_p),
        ("n_groups", C.c_uint32),
        ("pod_state", C.c_void_p),
        ("pod_ident", C.c_void_p),
        ("n_pods", C.c_uint64),
        ("lws_out", C.c_void_p),
        ("group_out", C.c_void_p),
        ("node_occupancy", C.c_void_p),
        ("flags", C.c_uint32),
    ]


class Changes(C.Structure):
    _fields_ = [
        ("lws_rows", C.c_void_p),
        ("lws_out", C.c_void_p),
        ("lws_capacity", C.c_uint32),
        ("n_lws", C.c_uint32),
        ("group_rows", C.c_void_p),
        ("group_out", C.c_void_p),
        ("group_capacity", C.c_uint32),
        ("n_groups", C.c_uint32),
    ]


TABLE_LWS, TABLE_GROUPS, TABLE_POD_STATE, TABLE_POD_IDENT, TABLE_PLACE_REQS, TABLE_NODES = 0, 1, 2, 3, 4, 5
TABLE_DS, TABLE_DS_ROLES, TABLE_DS_REVROLES = 6, 7, 8  # lwse_ds_resident_tick only
TABLE_DS_LINKS = 9  # lwse_ds_resident_tick only: DS_LINK rows, one per revision-role row
PATCH_RANGE = 1 << 0
TICK_MAX_SEGS = 8
TICK_PLACE = 1 << 8
TICK_NO_SWEEP = 1 << 9
TICK_SHARED_OCCUPANCY = 1 << 10


class PatchSeg(C.Structure):
    _fields_ = [
        ("table", C.c_uint32),
        ("flags", C.c_uint32),
        ("n", C.c_uint32),
        ("first_row", C.c_uint32),
        ("rows", C.c_void_p),
        ("values", C.c_void_p),
    ]


class Tick(C.Structure):
    _fields_ = [
        ("segs", C.POINTER(PatchSeg)),
        ("n_segs", C.c_uint32),
        ("flags", C.c_uint32),
        ("lws_rows", C.c_void_p),
        ("lws_out", C.c_void_p),
        ("n_lws", C.c_uint32),
        ("n_groups", C.c_uint32),
        ("group_rows", C.c_void_p),
        ("group_out", C.c_void_p),
        ("place_rows", C.c_void_p),
        ("place_out", C.c_void_p),
        ("n_place", C.c_uint32),
        ("place_rounds", C.c_uint32),
    ]


class NodeInfo(C.Structure):
    """lwse_node_info: what the node-row patches of the last submitted tick did."""

    _fields_ = [
        ("rows_patched", C.c_uint32),
        ("index_built", C.c_uint32),
        ("n_usable", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class DsTables(C.Structure):
    _fields_ = [
        ("ds", C.c_void_p),
        ("n_ds", C.c_uint32),
        ("roles", C.c_void_p),
        ("n_roles", C.c_uint32),
        ("revroles", C.c_void_p),
        ("n_revroles", C.c_uint32),
        ("ds_out", C.c_void_p),
        ("role_out", C.c_void_p),
        ("revrole_out", C.c_void_p),
    ]


class DsChanges(C.Structure):
    """lwse_ds_changes: the changed DS rows and the full output mirrors of a DS tick (engine-owned pinned memory)."""

    _fields_ = [
        ("ds_rows", C.c_void_p),
        ("n_changed", C.c_uint32),
        ("reserved", C.c_uint32),
        ("ds_out", C.c_void_p),
        ("role_out", C.c_void_p),
        ("revrole_out", C.c_void_p),
    ]


class DsTickInfo(C.Structure):
    """lwse_ds_tick_info: how the last DS tick read ready counts."""

    _fields_ = [
        ("linked", C.c_uint32),
        ("rows_from_lws", C.c_uint32),
        ("rows_fallback", C.c_uint32),
        ("reserved", C.c_uint32),
        ("lws_ticks", C.c_uint64),
    ]


class DsForecastOut(C.Structure):
    """lwse_ds_forecast_out: where a forecast goes, and the trajectory rows it wrote / needed."""

    _fields_ = [
        ("ds", C.c_void_p),
        ("roles", C.c_void_p),
        ("steps", C.c_void_p),
        ("step_capacity", C.c_uint32),
        ("n_steps_written", C.c_uint32),
        ("n_steps_needed", C.c_uint64),
    ]


class LwsForecastOut(C.Structure):
    """lwse_lws_forecast_out: where an LWS forecast goes, and the trajectory rows it wrote / needed."""

    _fields_ = [
        ("lws", C.c_void_p),
        ("steps", C.c_void_p),
        ("step_capacity", C.c_uint32),
        ("n_steps_written", C.c_uint32),
        ("n_steps_needed", C.c_uint64),
    ]


class RolloutWhatIf(C.Structure):
    """lwse_rollout_whatif: proposed LWS rows for resident rows in; the controller's first write and the
    forecast of the rollout each proposal would start out."""

    _fields_ = [
        ("rows", C.c_void_p),
        ("recs", C.c_void_p),
        ("n", C.c_uint32),
        ("reserved", C.c_uint32),
        ("now", C.c_void_p),
        ("fc", LwsForecastOut),
    ]


class DsRolloutWhatIf(C.Structure):
    """lwse_ds_rollout_whatif: proposed DS edits in; the DS controller's first decision and the forecast of
    the rollout each proposal would start out."""

    _fields_ = [
        ("proposals", C.c_void_p),
        ("roles", C.c_void_p),
        ("n", C.c_uint32),
        ("reserved", C.c_uint32),
        ("now", C.c_void_p),
        ("now_roles", C.c_void_p),
        ("fc", DsForecastOut),
    ]


class PlaceWhatIf(C.Structure):
    """lwse_place_whatif: a hypothetical placement round over the resident tables (segments and extra
    rows in, changed rows and the PLACE_WHATIF counters out)."""

    _fields_ = [
        ("segs", C.c_void_p),
        ("n_segs", C.c_uint32),
        ("extra", C.c_void_p),
        ("n_extra", C.c_uint32),
        ("n_namespaces", C.c_uint32),
        ("capacity", C.c_uint32),
        ("rows", C.c_void_p),
        ("before", C.c_void_p),
        ("after", C.c_void_p),
        ("extra_out", C.c_void_p),
        ("n_changed", C.c_uint32),
        ("n_lost", C.c_uint32),
        ("n_moved", C.c_uint32),
        ("n_gained", C.c_uint32),
        ("n_placed", C.c_uint32),
        ("n_unschedulable", C.c_uint32),
        ("n_conflict", C.c_uint32),
        ("namespaces_solved", C.c_uint32),
        ("form", C.c_uint32),
    ]


# the counters of a what-if, as Engine.resident_place_whatif returns them
PLACE_WHATIF = ("n_changed", "n_lost", "n_moved", "n_gained", "n_placed", "n_unschedulable", "n_conflict",
                "namespaces_solved")


class DrainWhatIf(C.Structure):
    """lwse_drain_whatif: the group rows of a sweep with the pods of a set of nodes deleting (node rows in,
    changed group rows and the DRAIN_WHATIF counters out)."""

    _fields_ = [
        ("nodes", C.c_void_p),
        ("n_nodes", C.c_uint32),
        ("capacity", C.c_uint32),
        ("rows", C.c_void_p),
        ("before", C.c_void_p),
        ("after", C.c_void_p),
        ("n_changed", C.c_uint32),
        ("n_pods_evicted", C.c_uint32),
        ("n_leaders_evicted", C.c_uint32),
        ("n_groups_restarted", C.c_uint32),
        ("n_ready_restarted", C.c_uint32),
        ("reserved", C.c_uint32),
        ("n_pods_recreated", C.c_uint64),
    ]


# the counters of a drain what-if, as Engine.resident_drain_whatif returns them
DRAIN_WHATIF = ("n_changed", "n_pods_evicted", "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted",
                "n_pods_recreated")

# lwse_drain_cost: per node, the totals of a drain what-if of that node alone
DRAIN_COST = np.dtype(
    [("pods", "<u4"), ("leaders", "<u4"), ("groups_restarted", "<u4"), ("ready_restarted", "<u4"),
     ("pods_recreated", "<u8"), ("reserved", "<u8")],
    align=False,
)
assert DRAIN_COST.itemsize == 32

# drain budget (lwse_resident_drain_budget*): the drain set's scope and the flags of a touched LWS row
DRAIN_NODES, DRAIN_DOMAINS = 0, 1
DRAINB_NOT_EVALUATED = 1 << 0
DRAINB_BREACHED = 1 << 1
DRAINB_ALREADY_BELOW = 1 << 2
DRAINB_LOSES_AVAILABLE = 1 << 3

# lwse_drain_budget: one touched LWS row of a drain
DRAIN_BUDGET = np.dtype(
    [("lws", "<u4"), ("flags", "<u4"), ("replicas", "<i4"), ("floor", "<i4"), ("ready_before", "<i4"),
     ("ready_after", "<i4"), ("groups_restarted", "<u4"), ("reserved", "<u4")],
    align=False,
)
assert DRAIN_BUDGET.itemsize == 32

# lwse_drain_budget_cost: per node or per domain, the DRAIN_COST totals and the budget columns
DRAIN_BUDGET_COST = np.dtype(DRAIN_COST.descr + [("lws_touched", "<u4"), ("lws_breached", "<u4"),
                                                 ("lws_loses_available", "<u4"), ("min_margin", "<i4")])
assert DRAIN_BUDGET_COST.itemsize == 48

# lwse_drain_place_cost: per node or per domain, whether the groups its drain restarts find a new domain
DRAIN_PLACE_COST = np.dtype(
    [("groups_restarted", "<u4"), ("unpinned", "<u4"), ("stranded", "<u4"), ("bumped", "<u4"), ("n_changed", "<u4"),
     ("n_lost", "<u4"), ("n_moved", "<u4"), ("n_gained", "<u4"), ("n_placed", "<u4"), ("n_unschedulable", "<u4"),
     ("n_conflict", "<u4"), ("namespaces_solved", "<u4"), ("reserved", "<u4", (4,))],
    align=False,
)
assert DRAIN_PLACE_COST.itemsize == 64


class DrainBudgetQuery(C.Structure):
    """lwse_drain_budget_query: the touched LWS rows of one drain set (node rows or domain ids in, the
    DRAIN_BUDGET rows and the DRAIN_BUDGET_TOTALS out)."""

    _fields_ = [
        ("ids", C.c_void_p),
        ("n_ids", C.c_uint32),
        ("scope", C.c_uint32),
        ("capacity", C.c_uint32),
        ("reserved", C.c_uint32),
        ("rows", C.c_void_p),
        ("n_touched", C.c_uint32),
        ("n_breached", C.c_uint32),
        ("n_loses_available", C.c_uint32),
        ("n_already_below", C.c_uint32),
        ("n_pods_evicted", C.c_uint32),
        ("n_leaders_evicted", C.c_uint32),
        ("n_groups_restarted", C.c_uint32),
        ("n_ready_restarted", C.c_uint32),
        ("n_pods_recreated", C.c_uint64),
    ]


# the totals of a drain budget query, as Engine.resident_drain_budget returns them
DRAIN_BUDGET_TOTALS = ("n_touched", "n_breached", "n_loses_available", "n_already_below", "n_pods_evicted",
                       "n_leaders_evicted", "n_groups_restarted", "n_ready_restarted", "n_pods_recreated")

# drain waves (lwse_resident_drain_waves): the wave cap and the status of a key
DRAIN_WAVES_MAX = 64
DRAINW_PLANNED = 0
DRAINW_BREACHES_ALONE = 1
DRAINW_NO_WAVE = 2

# lwse_drain_wave_key: one key of the plan, in query order
DRAIN_WAVE_KEY = np.dtype(
    [("id", "<u4"), ("wave", "<u4"), ("status", "<u4"), ("groups_restarted", "<u4"), ("ready_restarted", "<u4"),
     ("lws_touched", "<u4"), ("lws_breached", "<u4"), ("reserved", "<u4")],
    align=False,
)
assert DRAIN_WAVE_KEY.itemsize == 32

# lwse_drain_wave: one opened wave, the set-form totals over its ids
DRAIN_WAVE = np.dtype(
    [("n_keys", "<u4"), ("lws_touched", "<u4"), ("lws_loses_available", "<u4"), ("n_pods_evicted", "<u4"),
     ("n_leaders_evicted", "<u4"), ("n_groups_restarted", "<u4"), ("n_ready_restarted", "<u4"), ("min_margin", "<i4"),
     ("n_pods_recreated", "<u8"), ("reserved", "<u8")],
    align=False,
)
assert DRAIN_WAVE.itemsize == 48


class DrainWavesQuery(C.Structure):
    """lwse_drain_waves_query: a first-fit plan of distinct node rows or domain ids into waves (the ids and the wave
    cap in, the DRAIN_WAVE_KEY and DRAIN_WAVE rows and the DRAIN_WAVES_TOTALS out)."""

    _fields_ = [
        ("ids", C.c_void_p),
        ("n_ids", C.c_uint32),
        ("scope", C.c_uint32),
        ("max_waves", C.c_uint32),
        ("reserved", C.c_uint32),
        ("keys", C.c_void_p),
        ("waves", C.c_void_p),
        ("n_waves", C.c_uint32),
        ("n_planned", C.c_uint32),
        ("n_breaches_alone", C.c_uint32),
        ("n_no_wave", C.c_uint32),
    ]


# the totals of a drain waves query, as Engine.resident_drain_waves returns them
DRAIN_WAVES_TOTALS = ("n_waves", "n_planned", "n_breaches_alone", "n_no_wave")


# DS drain (lwse_resident_ds_drain*): the flags of a touched DS
DSD_TOUCHED = 1 << 0
DSD_SERVICE_LOST = 1 << 1
DSD_OLD_SERVICE_LOST = 1 << 2
DSD_STALLS = 1 << 3
DSD_CHANGED = 1 << 4

# lwse_ds_drain: one touched DS of a drain, with its ds_out row in the before and the after sweep
DS_DRAIN = np.dtype(
    [("ds", "<u4"), ("flags", "<u4"), ("rows_touched", "<u4"), ("rows_zeroed", "<u4"), ("new_zeroed_roles", "<u4"),
     ("old_zeroed_roles", "<u4"), ("reserved", "<u4", (2,)), ("before", DS_OUT), ("after", DS_OUT)],
    align=False,
)
assert DS_DRAIN.itemsize == 64

# lwse_ds_drain_cost: per node or per domain, the set form's DS counts for that key alone
DS_DRAIN_COST = np.dtype(
    [("ds_touched", "<u4"), ("ds_service_lost", "<u4"), ("ds_old_service_lost", "<u4"), ("ds_stalled", "<u4"),
     ("rows_touched", "<u4"), ("rows_zeroed", "<u4"), ("reserved", "<u4", (2,))],
    align=False,
)
assert DS_DRAIN_COST.itemsize == 32


class DsDrainQuery(C.Structure):
    """lwse_ds_drain_query: the touched DisaggregatedSets of one drain set (node rows or domain ids in, the
    DS_DRAIN rows, optionally the after sweep's full role_out / revrole_out, and the DS_DRAIN_TOTALS out)."""

    _fields_ = [
        ("ids", C.c_void_p),
        ("n_ids", C.c_uint32),
        ("scope", C.c_uint32),
        ("capacity", C.c_uint32),
        ("reserved", C.c_uint32),
        ("rows", C.c_void_p),
        ("role_out", C.c_void_p),
        ("revrole_out", C.c_void_p),
        ("n_touched", C.c_uint32),
        ("n_service_lost", C.c_uint32),
        ("n_old_service_lost", C.c_uint32),
        ("n_stalled", C.c_uint32),
        ("n_changed", C.c_uint32),
        ("rows_touched", C.c_uint32),
        ("rows_zeroed", C.c_uint32),
        ("rows_linked", C.c_uint32),
    ]


# the totals of a DS drain query, as Engine.resident_ds_drain returns them
DS_DRAIN_TOTALS = ("n_touched", "n_service_lost", "n_old_service_lost", "n_stalled", "n_changed", "rows_touched",
                   "rows_zeroed", "rows_linked")

# DS drain waves (lwse_resident_ds_drain_waves): the verdicts a plan keeps (`constraints`) and a key triggers alone
DSW_LWS_FLOOR = 1 << 0
DSW_DS_SERVICE = 1 << 1
DSW_DS_OLD_SERVICE = 1 << 2
DSW_DS_STALL = 1 << 3
DSW_ALL = DSW_LWS_FLOOR | DSW_DS_SERVICE | DSW_DS_OLD_SERVICE | DSW_DS_STALL
DSW_NAMES = {DSW_LWS_FLOOR: "lws_floor", DSW_DS_SERVICE: "ds_service", DSW_DS_OLD_SERVICE: "ds_old_service",
             DSW_DS_STALL: "ds_stall"}

# lwse_ds_drain_wave_key: one key of the plan, in query order
DS_DRAIN_WAVE_KEY = np.dtype(
    [("id", "<u4"), ("wave", "<u4"), ("status", "<u4"), ("alone", "<u4"), ("groups_restarted", "<u4"),
     ("ready_restarted", "<u4"), ("lws_touched", "<u4"), ("lws_breached", "<u4"), ("ds_touched", "<u4"),
     ("ds_service_lost", "<u4"), ("ds_old_service_lost", "<u4"), ("ds_stalled", "<u4")],
    align=False,
)
assert DS_DRAIN_WAVE_KEY.itemsize == 48

# lwse_ds_drain_wave: one opened wave, the set-form totals of the drain budget and the DS drain over its ids
DS_DRAIN_WAVE = np.dtype(
    [("n_keys", "<u4"), ("lws_touched", "<u4"), ("lws_breached", "<u4"), ("lws_loses_available", "<u4"),
     ("n_pods_evicted", "<u4"), ("n_leaders_evicted", "<u4"), ("n_groups_restarted", "<u4"),
     ("n_ready_restarted", "<u4"), ("min_margin", "<i4"), ("ds_touched", "<u4"), ("ds_service_lost", "<u4"),
     ("ds_old_service_lost", "<u4"), ("ds_stalled", "<u4"), ("rows_touched", "<u4"), ("rows_zeroed", "<u4"),
     ("reserved", "<u4"), ("n_pods_recreated", "<u8"), ("reserved2", "<u8")],
    align=False,
)
assert DS_DRAIN_WAVE.itemsize == 80


class DsDrainWavesQuery(C.Structure):
    """lwse_ds_drain_waves_query: a first-fit plan of distinct node rows or domain ids into waves that keep the
    verdicts named in ``constraints`` (the ids, the cap and the DSW_* mask in, the DS_DRAIN_WAVE_KEY and
    DS_DRAIN_WAVE rows and the DS_DRAIN_WAVES_TOTALS out)."""

    _fields_ = [
        ("ids", C.c_void_p),
        ("n_ids", C.c_uint32),
        ("scope", C.c_uint32),
        ("max_waves", C.c_uint32),
        ("constraints", C.c_uint32),
        ("reserved", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("keys", C.c_void_p),
        ("waves", C.c_void_p),
        ("n_waves", C.c_uint32),
        ("n_planned", C.c_uint32),
        ("n_breaches_alone", C.c_uint32),
        ("n_no_wave", C.c_uint32),
    ]


assert C.sizeof(DsDrainWavesQuery) == 64

# the totals of a DS drain waves query, as Engine.resident_ds_drain_waves returns them
DS_DRAIN_WAVES_TOTALS = ("n_waves", "n_planned", "n_breaches_alone", "n_no_wave")

# drain placement waves (lwse_resident_drain_place_waves): the verdicts a plan keeps and a key triggers alone
DPW_LWS_FLOOR = 1 << 0
DPW_STRANDED = 1 << 1
DPW_BUMPED = 1 << 2
DPW_ALL = DPW_LWS_FLOOR | DPW_STRANDED | DPW_BUMPED
DPW_NAMES = {DPW_LWS_FLOOR: "lws_floor", DPW_STRANDED: "stranded", DPW_BUMPED: "bumped"}

# lwse_drain_place_wave_key: one key of the plan, in query order
DRAIN_PLACE_WAVE_KEY = np.dtype(
    [("id", "<u4"), ("wave", "<u4"), ("status", "<u4"), ("alone", "<u4"), ("groups_restarted", "<u4"),
     ("ready_restarted", "<u4"), ("lws_touched", "<u4"), ("lws_breached", "<u4"), ("unpinned", "<u4"),
     ("stranded", "<u4"), ("bumped", "<u4"), ("reserved", "<u4")],
    align=False,
)
assert DRAIN_PLACE_WAVE_KEY.itemsize == 48

# lwse_drain_place_wave: one opened wave, the set-form totals of the drain budget and the drain placement
DRAIN_PLACE_WAVE = np.dtype(
    [("n_keys", "<u4"), ("lws_touched", "<u4"), ("lws_loses_available", "<u4"), ("n_pods_evicted", "<u4"),
     ("n_leaders_evicted", "<u4"), ("n_groups_restarted", "<u4"), ("n_ready_restarted", "<u4"), ("min_margin", "<i4"),
     ("n_pods_recreated", "<u8"), ("lws_breached", "<u4"), ("unpinned", "<u4"), ("stranded", "<u4"), ("bumped", "<u4"),
     ("n_changed", "<u4"), ("n_lost", "<u4"), ("n_moved", "<u4"), ("n_gained", "<u4"), ("n_placed", "<u4"),
     ("n_unschedulable", "<u4"), ("n_conflict", "<u4"), ("namespaces_solved", "<u4"), ("reserved", "<u4", (2,))],
    align=False,
)
assert DRAIN_PLACE_WAVE.itemsize == 96


class DrainPlaceWavesQuery(C.Structure):
    """lwse_drain_place_waves_query: a first-fit plan of distinct node rows or domain ids into waves whose
    restarted groups find a new exclusive domain (the ids, the cap and the DPW_* mask in, the DRAIN_PLACE_WAVE_KEY
    and DRAIN_PLACE_WAVE rows and the DRAIN_WAVES_TOTALS out)."""

    _fields_ = DsDrainWavesQuery._fields_


assert C.sizeof(DrainPlaceWavesQuery) == 64


# lwse_rollout_place: per entry, whether the groups its rollout adds find an exclusive domain
ROLLOUT_PLACE = np.dtype(
    [("flags", "<u4"), ("fc_flags", "<u4"), ("peak", "<i4"), ("surge", "<u4"), ("placed", "<u4"), ("stranded", "<u4"),
     ("own_lost", "<u4"), ("bumped", "<u4"), ("n_changed", "<u4"), ("n_lost", "<u4"), ("n_moved", "<u4"),
     ("n_gained", "<u4"), ("n_placed", "<u4"), ("n_unschedulable", "<u4"), ("n_conflict", "<u4"),
     ("namespaces_solved", "<u4")],
    align=False,
)
assert ROLLOUT_PLACE.itemsize == 64

RPL_SOLVED = 1 << 0
RPL_NOT_EXCLUSIVE = 1 << 1
RPL_NOT_FORECAST = 1 << 2
RPL_NOT_MODELLED = 1 << 3
RPL_STRANDS = 1 << 4
RPL_BUMPS = 1 << 5
RPL_NAMES = {RPL_SOLVED: "solved", RPL_NOT_EXCLUSIVE: "not_exclusive", RPL_NOT_FORECAST: "not_forecast",
             RPL_NOT_MODELLED: "not_modelled", RPL_STRANDS: "strands", RPL_BUMPS: "bumps"}
ROLLOUT_PLACE_TOTALS = ("n_solved", "n_strands", "n_surge", "n_stranded")


class RolloutPlaceQuery(C.Structure):
    """lwse_rollout_place_query: entries (LWS row, namespace id, optional proposed LWS_REC) in, one ROLLOUT_PLACE
    row per entry, optionally every entry's extra PLACE_REQ rows, and the ROLLOUT_PLACE_TOTALS out."""

    _fields_ = [
        ("rows", C.c_void_p),
        ("ns", C.c_void_p),
        ("recs", C.c_void_p),
        ("n", C.c_uint32),
        ("reserved", C.c_uint32),
        ("out", C.c_void_p),
        ("extra", C.c_void_p),
        ("extra_capacity", C.c_uint64),
        ("n_solved", C.c_uint32),
        ("n_strands", C.c_uint32),
        ("n_surge", C.c_uint64),
        ("n_stranded", C.c_uint64),
    ]


assert C.sizeof(RolloutPlaceQuery) == 80


# rollout placement waves (lwse_resident_rollout_place_waves): the verdicts a wave keeps and the status of a key
RPW_STRANDED = 1 << 0
RPW_BUMPED = 1 << 1
RPW_ALL = RPW_STRANDED | RPW_BUMPED
RPW_NAMES = {RPW_STRANDED: "stranded", RPW_BUMPED: "bumped"}
ROLLW_PLANNED = DRAINW_PLANNED
ROLLW_TRIGGERS_ALONE = DRAINW_BREACHES_ALONE
ROLLW_NO_WAVE = DRAINW_NO_WAVE
ROLLW_NOT_SOLVED = 3
ROLLW_NAMES = {ROLLW_PLANNED: "planned", ROLLW_TRIGGERS_ALONE: "triggers_alone", ROLLW_NO_WAVE: "no_wave",
               ROLLW_NOT_SOLVED: "not_solved"}

# lwse_rollout_wave_key: one key of the plan, in query order
ROLLOUT_WAVE_KEY = np.dtype([("wave", "<u4"), ("status", "<u4"), ("alone", "<u4"), ("reserved", "<u4")], align=False)
assert ROLLOUT_WAVE_KEY.itemsize == 16

# lwse_rollout_wave: one opened wave, the set-form totals over its keys
ROLLOUT_WAVE = np.dtype(
    [("n_keys", "<u4"), ("surge", "<u4"), ("placed", "<u4"), ("stranded", "<u4"), ("own_lost", "<u4"), ("bumped", "<u4"),
     ("n_changed", "<u4"), ("n_lost", "<u4"), ("n_moved", "<u4"), ("n_gained", "<u4"), ("n_placed", "<u4"),
     ("n_unschedulable", "<u4"), ("n_conflict", "<u4"), ("namespaces", "<u4"), ("reserved", "<u4", (2,))],
    align=False,
)
assert ROLLOUT_WAVE.itemsize == 64
ROLLOUT_WAVES_TOTALS = ("n_waves", "n_planned", "n_triggers_alone", "n_no_wave", "n_not_solved")


class RolloutPlaceWavesQuery(C.Structure):
    """lwse_rollout_place_waves_query: the entries of RolloutPlaceQuery (distinct rows), the cap and the RPW_* mask
    in; the ROLLOUT_WAVE_KEY and ROLLOUT_WAVE rows, optionally the ROLLOUT_PLACE alone rows, and the
    ROLLOUT_WAVES_TOTALS out."""

    _fields_ = [
        ("rows", C.c_void_p),
        ("ns", C.c_void_p),
        ("recs", C.c_void_p),
        ("n", C.c_uint32),
        ("max_waves", C.c_uint32),
        ("constraints", C.c_uint32),
        ("reserved", C.c_uint32),
        ("keys", C.c_void_p),
        ("waves", C.c_void_p),
        ("alone_rows", C.c_void_p),
        ("n_waves", C.c_uint32),
        ("n_planned", C.c_uint32),
        ("n_triggers_alone", C.c_uint32),
        ("n_no_wave", C.c_uint32),
        ("n_not_solved", C.c_uint32),
        ("reserved1", C.c_uint32),
    ]


assert C.sizeof(RolloutPlaceWavesQuery) == 88


# lwse_scale_headroom: per entry, how far the object can scale up before a group it adds finds no exclusive domain
SCALE_HEADROOM = np.dtype(
    [("flags", "<u4"), ("replicas", "<i4"), ("max_replicas", "<i4"), ("probe", "<i4"), ("surge", "<u4"),
     ("placed", "<u4"), ("stranded", "<u4"), ("own_lost", "<u4"), ("bumped", "<u4"), ("n_changed", "<u4"),
     ("n_lost", "<u4"), ("n_moved", "<u4"), ("n_gained", "<u4"), ("n_placed", "<u4"), ("n_unschedulable", "<u4"),
     ("n_conflict", "<u4")],
    align=False,
)
assert SCALE_HEADROOM.itemsize == 64

SHR_SOLVED = 1 << 0
SHR_NOT_EXCLUSIVE = 1 << 1
SHR_NOT_FORECAST = 1 << 2
SHR_NOT_SETTLED = 1 << 3
SHR_BLOCKED = 1 << 4
SHR_AT_CEILING = 1 << 5
SHR_STRANDS = 1 << 6
SHR_BUMPS = 1 << 7
SHR_NAMES = {SHR_SOLVED: "solved", SHR_NOT_EXCLUSIVE: "not_exclusive", SHR_NOT_FORECAST: "not_forecast",
             SHR_NOT_SETTLED: "not_settled", SHR_BLOCKED: "blocked", SHR_AT_CEILING: "at_ceiling",
             SHR_STRANDS: "strands", SHR_BUMPS: "bumps"}
SCALE_HEADROOM_TOTALS = ("n_solved", "n_blocked", "n_at_ceiling", "rounds", "headroom")


class ScaleHeadroomQuery(C.Structure):
    """lwse_scale_headroom_query: entries (LWS row, namespace id, optional ceiling) and the RPW_* mask in; one
    SCALE_HEADROOM row per entry, optionally the ROLLOUT_PLACE rows of the resident rows, and the
    SCALE_HEADROOM_TOTALS out."""

    _fields_ = [
        ("rows", C.c_void_p),
        ("ns", C.c_void_p),
        ("ceilings", C.c_void_p),
        ("n", C.c_uint32),
        ("constraints", C.c_uint32),
        ("reserved", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("out", C.c_void_p),
        ("current", C.c_void_p),
        ("n_solved", C.c_uint32),
        ("n_blocked", C.c_uint32),
        ("n_at_ceiling", C.c_uint32),
        ("rounds", C.c_uint32),
        ("headroom", C.c_uint64),
    ]


assert C.sizeof(ScaleHeadroomQuery) == 80


# lwse_place_explain_row: why a row of a placement round has its verdict (per-domain classes and named domains)
PLACE_EXPLAIN = np.dtype(
    [("row", "<u4"), ("flags", "<u4"), ("place_flags", "<u4"), ("n_own", "<u4"), ("n_no_usable", "<u4"),
     ("n_too_small", "<u4"), ("n_held_pinned", "<u4"), ("n_held_earlier", "<u4"), ("n_held_later", "<u4"),
     ("n_open", "<u4"), ("n_fit_uncordoned", "<u4"), ("best_domain", "<u4"), ("blocker_domain", "<u4"),
     ("blocker_row", "<u4"), ("shortfall", "<u4"), ("shortfall_domain", "<u4")],
    align=False,
)
assert PLACE_EXPLAIN.itemsize == 64
# the class counts of a row, in the order of the query's n_class totals
PLACE_EXPLAIN_CLASSES = ("n_own", "n_no_usable", "n_too_small", "n_held_pinned", "n_held_earlier", "n_held_later",
                         "n_open", "n_fit_uncordoned")

PEX_CAPACITY = 1 << 0
PEX_EXCLUSIVE = 1 << 1
PEX_CORDONED = 1 << 2
PEX_CONFLICT = 1 << 3
PEX_NO_CLAIM = 1 << 4
PEX_NO_NAMESPACE = 1 << 5
PEX_BAD_SIZE = 1 << 6
PEX_NAMES = {PEX_CAPACITY: "capacity", PEX_EXCLUSIVE: "exclusive", PEX_CORDONED: "cordoned", PEX_CONFLICT: "conflict",
             PEX_NO_CLAIM: "no_claim", PEX_NO_NAMESPACE: "no_namespace", PEX_BAD_SIZE: "bad_size"}


class PlaceExplainQuery(C.Structure):
    """lwse_place_explain_query: the round (segments, extra rows, namespaces as PlaceWhatIf) and the rows (a list,
    or a PLACE_* mask) in; PLACE_EXPLAIN rows, the class sums and the PEX_* flag counts out."""

    _fields_ = [
        ("segs", C.c_void_p),
        ("n_segs", C.c_uint32),
        ("n_extra", C.c_uint32),
        ("extra", C.c_void_p),
        ("n_namespaces", C.c_uint32),
        ("mask", C.c_uint32),
        ("rows", C.c_void_p),
        ("n_rows", C.c_uint32),
        ("capacity", C.c_uint32),
        ("out", C.c_void_p),
        ("n_explained", C.c_uint32),
        ("round_rows", C.c_uint32),
        ("n_domains", C.c_uint32),
        ("whatif", C.c_uint32),
        ("form", C.c_uint32),
        ("n_flag", C.c_uint32 * 7),
        ("n_class", C.c_uint64 * 8),
    ]


assert C.sizeof(PlaceExplainQuery) == 168


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("device", C.c_int32),
        ("flags", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


def aligned_empty(n: int, dtype: np.dtype, align: int = 64) -> np.ndarray:
    """An ``n``-row table whose base address is ``align``-byte aligned."""
    dtype = np.dtype(dtype)
    raw = np.zeros(n * dtype.itemsize + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off : off + n * dtype.itemsize].view(dtype)


def ptr(a) -> int | None:
    """Base address of a numpy array / torch tensor, or None."""
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return a.ctypes.data


FNV_OFFSET = 0xCBF29CE484222325
FNV_PRIME = 0x100000001B3


def hash64(s: str | bytes) -> int:
    """FNV-1a 64 — the string hash of the encoders (same as ``lwse_hash64``)."""
    if isinstance(s, str):
        s = s.encode()
    h = FNV_OFFSET
    for b in s:
        h = ((h ^ b) * FNV_PRIME) & 0xFFFFFFFFFFFFFFFF
    return h


def hash32(s: str | bytes) -> int:
    h = hash64(s)
    return (h ^ (h >> 32)) & 0xFFFFFFFF
