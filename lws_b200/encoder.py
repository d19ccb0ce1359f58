"""Objects → fixed-width records (the host side of the boundary).

The encoder performs the string / label / lookup work that the reference does
with informer-cache ``List``/``Get`` calls and leaves every comparison and
count that decides an output to the device:

* label-selector lists + ``SortByIndex`` (pkg/utils/utils.go:53-71) become the
  row order of the group table (row r of an object = group index r);
* names are reduced to the *NAME_MATCH* flags the reference checks at
  pkg/controllers/leaderworkerset_controller.go:609-612;
* revision keys, UIDs and topology label values become hashes (compared for
  equality on the device);
* ``GetParentNameAndOrdinal`` (pkg/utils/statefulset/statefulset_utils.go:27-45)
  is evaluated here (it is a regex over a string) and reduced to ``NAME_OK``.

Objects the fixed-width form cannot express exactly (two leader pods with the
same group index, a worker whose name does not derive from its group's leader,
a leader pod whose name is not ``<lws>-<index>`` …) get ``LWS_IRREGULAR`` so
that the caller reconciles them through the stock path; see DESIGN.md.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Iterable, Optional

import numpy as np

from . import api
from . import records as R

_STATEFUL_POD_RE = re.compile(r"(.*)-([0-9]+)$", re.S)


def get_parent_name_and_ordinal(name: str) -> tuple[str, int]:
    """pkg/utils/statefulset/statefulset_utils.go:33-45."""
    m = _STATEFUL_POD_RE.match(name)
    if not m:
        return "", -1
    parent, digits = m.group(1), m.group(2)
    try:
        v = int(digits)
    except ValueError:  # pragma: no cover
        return parent, -1
    if v > 0x7FFFFFFF:  # strconv.ParseInt(..., 10, 32) overflows → err → ordinal stays -1
        return parent, -1
    return parent, v


def atoi(s: Optional[str]) -> Optional[int]:
    """strconv.Atoi: optional sign, decimal digits only; None on error."""
    if s is None or not re.fullmatch(r"[+-]?[0-9]+", s):
        return None
    v = int(s)
    if not -(1 << 63) <= v < (1 << 63):
        return None
    return v


def parse_int_or_percent(v: api.IntOrString) -> tuple[int, bool, bool]:
    """→ (value, is_percent, valid), as intstr.GetScaledValueFromIntOrPercent parses."""
    if isinstance(v, int):
        return v, False, True
    if isinstance(v, str) and v.endswith("%"):
        n = atoi(v[:-1])
        if n is not None:
            return n, True, True
    return 0, False, False


@dataclass
class LwsItem:
    """Everything ``Reconcile`` looks at for one LeaderWorkerSet."""

    lws: api.LeaderWorkerSet
    revision_key: str  # revisionutils.GetRevisionKey(updatedRevision)
    lws_updated: bool = False  # leaderWorkerSetUpdated
    leader_sts: Optional[api.StatefulSet] = None
    existing_revisions: Optional[set] = None  # ControllerRevision keys; None = all exist


@dataclass
class Cluster:
    """The slice of the informer cache the path reads."""

    pods: list = field(default_factory=list)
    statefulsets: list = field(default_factory=list)
    nodes: list = field(default_factory=list)


@dataclass
class LwsTables:
    lws: np.ndarray
    groups: np.ndarray
    pod_state: np.ndarray
    pod_ident: np.ndarray
    nodes: np.ndarray
    n_domains: int
    domain_values: list  # domain id → topology label value
    node_names: list
    # bookkeeping for reading results back by name
    lws_names: list
    group_pod_names: list  # per group row: names of its pod rows


def _state_column(pod_rows) -> np.ndarray:
    col = R.aligned_empty(len(pod_rows), R.POD_STATE)
    col[:] = np.array([r[2] for r in pod_rows], dtype=np.uint8)
    return col


def encode_node(n: api.Node, topology_key: Optional[str], domains: dict) -> tuple:
    """One node row.  ``domains``: label value → dense domain id; a new value takes the next id."""
    flags = R.NODE_SCHEDULABLE if n.schedulable else 0
    dom = R.NONE
    h = 0
    if topology_key is not None and topology_key in n.labels:
        val = n.labels[topology_key]
        flags |= R.NODE_HAS_TOPOLOGY
        dom = domains.setdefault(val, len(domains))
        h = R.hash64(val)
    return (h, dom, min(n.capacity, 0xFFFF), flags)


def encode_nodes(nodes: Iterable[api.Node], topology_key: Optional[str]):
    nodes = list(nodes)
    rec = R.aligned_empty(len(nodes), R.NODE_REC)
    domains: dict[str, int] = {}
    for i, n in enumerate(nodes):
        rec[i] = encode_node(n, topology_key, domains)
    values = [None] * len(domains)
    for v, d in domains.items():
        values[d] = v
    return rec, values, {n.name: i for i, n in enumerate(nodes)}


def encode_lws(items: Iterable[LwsItem], cluster: Cluster, topology_key: Optional[str] = None,
               encoded_nodes=None) -> LwsTables:
    """``encoded_nodes``: the result of ``encode_nodes`` when the caller encodes many object batches
    against one node table (the incremental encoder re-encodes one object per watch event)."""
    items = list(items)
    node_rec, domain_values, node_index = encoded_nodes if encoded_nodes is not None else encode_nodes(cluster.nodes, topology_key)

    pods_by_ns_set: dict[tuple, list] = {}
    for p in cluster.pods:
        key = (p.namespace, p.labels.get(api.SetNameLabelKey))
        pods_by_ns_set.setdefault(key, []).append(p)
    sts_by_ns_set: dict[tuple, list] = {}
    sts_by_name: dict[tuple, api.StatefulSet] = {}
    for s in cluster.statefulsets:
        sts_by_ns_set.setdefault((s.namespace, s.labels.get(api.SetNameLabelKey)), []).append(s)
        sts_by_name[(s.namespace, s.name)] = s

    lws_rows, group_rows, pod_rows = [], [], []
    group_pod_names: list = []

    for li, it in enumerate(items):
        lws = it.lws
        irregular = False
        flags = 0
        surge, surge_pct, surge_ok = parse_int_or_percent(lws.rollingUpdate.maxSurge)
        unav, unav_pct, unav_ok = parse_int_or_percent(lws.rollingUpdate.maxUnavailable)
        if surge_pct:
            flags |= R.LWS_SURGE_IS_PERCENT
        if unav_pct:
            flags |= R.LWS_UNAVAIL_IS_PERCENT
        if not (surge_ok and unav_ok):
            flags |= R.LWS_INTSTR_INVALID
        sts = it.leader_sts
        sts_replicas = sts_partition = annot = 0
        if sts is not None:
            flags |= R.LWS_STS_EXISTS
            sts_replicas, sts_partition = sts.replicas, sts.partition
            a = atoi(sts.annotations.get(api.ReplicasAnnotationKey, ""))
            if a is not None:
                flags |= R.LWS_ANNOT_VALID
                annot = a
        if it.lws_updated:
            flags |= R.LWS_UPDATED
        policy = {
            api.RecreateGroupOnPodRestart: R.RESTART_ON_POD_RESTART,
            api.RecreateGroupAfterStart: R.RESTART_AFTER_START,
        }.get(lws.restartPolicy, R.RESTART_NONE)
        flags |= policy << R.LWS_RESTART_SHIFT
        if api.RecreateGroupAfterStartAnnotationKey in lws.annotations:
            flags |= R.LWS_RECREATE_AFTER_START_ANNOT
        if lws.startupPolicy == api.LeaderReadyStartupPolicy:
            flags |= R.LWS_STARTUP_LEADER_READY
        if api.ExclusiveKeyAnnotationKey in lws.annotations:
            flags |= R.LWS_EXCLUSIVE_TOPOLOGY
            if lws.annotations[api.ExclusiveKeyAnnotationKey] != topology_key:
                irregular = True  # one topology key per node table
        if lws.subGroupPolicyType == api.SubGroupPolicyTypeLeaderExcluded:
            flags |= R.LWS_SUBGROUP_LEADER_EXCLUDED

        all_pods = pods_by_ns_set.get((lws.namespace, lws.name), [])
        all_sts = sts_by_ns_set.get((lws.namespace, lws.name), [])

        # List(leader pods) + SortByIndex (leaderworkerset_controller.go:584-593)
        leader_by_idx: dict[int, api.Pod] = {}
        for p in all_pods:
            if p.labels.get(api.WorkerIndexLabelKey) != "0":
                continue
            idx = atoi(p.labels.get(api.GroupIndexLabelKey, ""))
            if idx is None:
                flags |= R.LWS_GROUP_LABEL_INVALID  # :434-437 (SortByIndex merely drops it)
                continue
            if idx < 0:
                irregular = True
                continue
            if idx in leader_by_idx:
                irregular = True  # two leader pods, one slot
            leader_by_idx[idx] = p  # last writer wins (utils.go:68)
        # List(sts) + SortByIndex (:595-603); the leader sts has no group-index label
        sts_by_idx: dict[int, api.StatefulSet] = {}
        for s in all_sts:
            idx = atoi(s.labels.get(api.GroupIndexLabelKey, ""))
            if idx is None or idx < 0:
                continue
            sts_by_idx[idx] = s
        # pods per group (pod_controller.go:338-349 selects by the label *string*)
        pods_by_idx: dict[int, list] = {}
        for p in all_pods:
            gi = p.labels.get(api.GroupIndexLabelKey)
            idx = atoi(gi if gi is not None else "")
            if idx is None or idx < 0 or str(idx) != gi:
                if gi is not None:
                    irregular = True
                continue
            pods_by_idx.setdefault(idx, []).append(p)

        n_groups = 1 + max([-1, *leader_by_idx, *sts_by_idx, *pods_by_idx])
        group_base = len(group_rows)
        for idx in range(n_groups):
            nominated = f"{lws.name}-{idx}"
            gflags = 0
            pod = leader_by_idx.get(idx)
            leader_rev = wsts_rev = 0
            leader_uid = wsts_uid = wsts_owner_uid = 0
            wsts_spec = wsts_avail = 0
            leader_node = R.NONE
            wsts = None
            if pod is not None:
                gflags |= R.GRP_POD_PRESENT
                if pod.name == nominated:
                    gflags |= R.GRP_POD_NAME_MATCH
                else:
                    irregular = True
                if pod.phase == "Running":
                    gflags |= R.GRP_POD_RUNNING
                if pod.readyCondition:
                    gflags |= R.GRP_POD_READY
                if pod.deletionTimestamp:
                    gflags |= R.GRP_POD_DELETING
                if pod.annotations.get(api.LeaderPodNameAnnotationKey, "") != "":
                    gflags |= R.GRP_MISTAKEN_ANNOTATION
                leader_rev = R.hash64(pod.labels.get(api.RevisionKey, ""))
                leader_uid = R.hash32(pod.uid)
                if it.existing_revisions is None or pod.labels.get(api.RevisionKey, "") in it.existing_revisions:
                    gflags |= R.GRP_REVISION_EXISTS
                if pod.nodeName != "":
                    leader_node = node_index.get(pod.nodeName, R.NODE_NOT_FOUND)
                wsts = sts_by_name.get((lws.namespace, pod.name))
            label_sts = sts_by_idx.get(idx)
            if label_sts is not None and label_sts.name == nominated:
                gflags |= R.GRP_WSTS_LABEL_NAME_MATCH
            if wsts is not None:
                gflags |= R.GRP_WSTS_FOUND
                wsts_rev = R.hash64(wsts.labels.get(api.RevisionKey, ""))
                wsts_uid = R.hash32(wsts.uid)
                wsts_spec, wsts_avail = wsts.replicas, wsts.availableReplicas
                if wsts.currentRevision == wsts.updateRevision:
                    gflags |= R.GRP_WSTS_REV_SETTLED
                owner = api.controller_of(wsts)
                if owner is not None and owner.kind == "Pod":
                    gflags |= R.GRP_WSTS_OWNER_IS_POD
                    wsts_owner_uid = R.hash32(owner.uid)
                    if pod is not None and owner.name == pod.name:
                        gflags |= R.GRP_WSTS_OWNER_NAME_MATCH

            gpods = pods_by_idx.get(idx, [])
            pod_base = len(pod_rows)
            names = []
            for p in gpods:
                bits = {"Pending": R.POD_PHASE_PENDING, "Running": R.POD_PHASE_RUNNING}.get(p.phase, 0)
                if any(c > 0 for c in p.initContainerRestartCounts) or any(
                    c > 0 for c in p.containerRestartCounts
                ):
                    bits |= R.POD_ANY_RESTART
                if p.deletionTimestamp:
                    bits |= R.POD_DELETING
                owner = api.controller_of(p)
                owner_uid = 0
                if owner is not None:
                    kind = {"Pod": R.POD_OWNER_POD, "StatefulSet": R.POD_OWNER_STS}.get(
                        owner.kind, R.POD_OWNER_OTHER
                    )
                    bits |= kind << R.POD_OWNER_SHIFT
                    owner_uid = R.hash32(owner.uid)
                    if owner.name == nominated:
                        bits |= R.POD_OWNER_NAME_MATCH
                    elif kind == R.POD_OWNER_STS:
                        irregular = True  # would Get() a foreign StatefulSet
                place = 0  # the cold word: name check + node binding
                if p.labels.get(api.WorkerIndexLabelKey) == "0":
                    bits |= R.POD_IS_LEADER
                    place |= R.PODID_NAME_OK
                else:
                    parent, ordinal = get_parent_name_and_ordinal(p.name)
                    if ordinal != -1:
                        place |= R.PODID_NAME_OK
                        if parent != nominated:
                            irregular = True  # leader lookup would hit another group
                if p.nodeName != "" and p.nodeName in node_index:
                    ni = node_index[p.nodeName]
                    if ni <= R.POD_NODE_MAX:
                        place |= R.PODID_SCHEDULED | (ni << R.PODID_NODE_SHIFT)
                pod_rows.append((R.hash64(p.labels.get(api.RevisionKey, "")), owner_uid, bits, place))
                names.append(p.name)
            group_pod_names.append(names)
            group_rows.append(
                (leader_rev, wsts_rev, wsts_spec, wsts_avail, leader_uid, wsts_uid, wsts_owner_uid,
                 leader_node, pod_base, len(gpods), li, gflags, (0, 0))
            )

        if irregular:
            flags |= R.LWS_IRREGULAR
        lws_rows.append(
            dict(
                rev_hash=R.hash64(it.revision_key), size=lws.size, flags=flags, replicas=lws.replicas,
                partition=lws.rollingUpdate.partition, max_surge=surge, max_unavailable=unav,
                sts_replicas=sts_replicas, sts_partition=sts_partition, sts_replicas_annotation=annot,
                subgroup_size=lws.subGroupSize or 0, uid_hash=R.hash64(lws.uid),
                group_base=group_base, group_count=n_groups,
            )
        )

    def table(rows, dtype):
        t = R.aligned_empty(len(rows), dtype)
        for i, r in enumerate(rows):
            if isinstance(r, dict):
                for k, v in r.items():
                    t[i][k] = v
            else:
                t[i] = r
        return t

    return LwsTables(
        lws=table(lws_rows, R.LWS_REC),
        groups=table(group_rows, R.GROUP_REC),
        pod_state=_state_column(pod_rows),
        pod_ident=R.pod_ident_table(
            np.array([r[0] for r in pod_rows], dtype=np.uint64), np.array([r[1] for r in pod_rows], dtype=np.uint32),
            np.array([r[3] for r in pod_rows], dtype=np.uint32),
        ),
        nodes=node_rec,
        n_domains=len(domain_values),
        domain_values=domain_values,
        node_names=[n.name for n in cluster.nodes],
        lws_names=[it.lws.name for it in items],
        group_pod_names=group_pod_names,
    )


# --------------------------------------------------------------------------- #
# DisaggregatedSet
# --------------------------------------------------------------------------- #
@dataclass
class DsItem:
    ds: api.DisaggregatedSet
    revision: str  # ComputeRevision(spec.roles) — the target revision
    children: list = field(default_factory=list)  # api.ChildLWS, List order


@dataclass
class DsTablesHost:
    ds: np.ndarray
    roles: np.ndarray
    revroles: np.ndarray
    role_names: list  # per DS: allRoleNames
    old_revisions: list  # per DS: old revision names in row order


def get_initial_replicas(child: api.ChildLWS) -> int:
    """pkg/utils/disaggregatedset/utils.go:33-46 → value or -1."""
    v = child.annotations.get(api.DSInitialReplicasAnnotationKey)
    if v is None or v == "":
        return -1
    n = atoi(v)
    if n is None or not -(1 << 31) <= n < (1 << 31):  # strconv.ParseInt(value, 10, 32)
        return -1
    return n


def encode_ds(items: Iterable[DsItem]) -> DsTablesHost:
    items = list(items)
    ds_rows, role_rows, rr_rows, names_out, revs_out = [], [], [], [], []
    # one order-preserving rank table for all timestamps
    stamps = sorted({c.creationTimestamp for it in items for c in it.children})
    rank = {s: i + 1 for i, s in enumerate(stamps)}
    for it in items:
        spec_names = [r.name for r in it.ds.roles]
        # GroupByRevision (utils.go:192-211); old revisions in first-seen order
        by_rev: dict[str, dict[str, api.ChildLWS]] = {}
        for c in it.children:
            by_rev.setdefault(c.revision, {})[c.role] = c
        old_revs = [r for r in by_rev if r != it.revision]
        # allRoleNames = spec roles, then removed roles (executor.go:140,189-197); the
        # reference ranges a Go map there — canonical order here is sorted
        old_role_set = {role for r in old_revs for role in by_rev[r]}
        removed = sorted(old_role_set - set(spec_names))
        all_names = spec_names + removed
        n = len(all_names)
        role_base, rev_base = len(role_rows), len(rr_rows)
        for i, name in enumerate(all_names):
            flags, target, surge, unav = 0, 0, 0, 0
            if i < len(spec_names):
                spec = it.ds.roles[i]
                flags |= R.ROLE_IN_SPEC
                target = 1 if spec.replicas is None else spec.replicas
                if spec.rollingUpdate is not None:
                    flags |= R.ROLE_HAS_ROLLING_CONFIG
                    surge, sp, sok = parse_int_or_percent(spec.rollingUpdate.maxSurge)
                    unav, up, uok = parse_int_or_percent(spec.rollingUpdate.maxUnavailable)
                    flags |= (R.ROLE_SURGE_IS_PERCENT if sp else 0) | (R.ROLE_UNAVAIL_IS_PERCENT if up else 0)
                    flags |= (0 if sok else R.ROLE_SURGE_INVALID) | (0 if uok else R.ROLE_UNAVAIL_INVALID)
            role_rows.append((target, surge, unav, flags))
        for rev in old_revs + [it.revision]:
            for name in all_names:
                c = by_rev.get(rev, {}).get(name)
                if c is None:
                    rr_rows.append((0, -1, 0, 0))
                    continue
                flags = R.RR_EXISTS | (rank[c.creationTimestamp] << R.RR_TS_SHIFT)
                if c.replicas is None:
                    flags |= R.RR_REPLICAS_NIL
                rr_rows.append((1 if c.replicas is None else c.replicas, get_initial_replicas(c),
                                c.readyReplicas, flags))
        ds_flags = R.DS_HAS_NEW_REVISION if it.revision in by_rev else 0
        ds_rows.append((R.hash64(it.ds.uid), role_base, n, len(spec_names), rev_base, len(old_revs), ds_flags))
        names_out.append(all_names)
        revs_out.append(old_revs)

    def table(rows, dtype):
        t = R.aligned_empty(len(rows), dtype)
        for i, r in enumerate(rows):
            t[i] = r
        return t

    return DsTablesHost(table(ds_rows, R.DS_REC), table(role_rows, R.DS_ROLE_REC),
                        table(rr_rows, R.DS_REVROLE_REC), names_out, revs_out)


# --------------------------------------------------------------------------- #
# PodGroup MinResources (host arithmetic: stays off the device, DESIGN.md §8)
# --------------------------------------------------------------------------- #
def pod_group_min_resources(leader_requests: Optional[dict], worker_requests: dict, size: int) -> dict:
    """pkg/utils/utils.go:84-103 CalculatePGMinResources over pre-summed per-template request
    vectors (resource name → integer milli-units; `PodRequests` of a single-container template):
    leader (the worker template's when no leader template is given) + (size − 1) × worker."""
    total = dict(worker_requests if leader_requests is None else leader_requests)
    for _ in range(max(int(size) - 1, 0)):  # quotav1.Add: union of the keys, summed
        for name, v in worker_requests.items():
            total[name] = total.get(name, 0) + v
    return total


# --------------------------------------------------------------------------- #
# Placement requests
# --------------------------------------------------------------------------- #
def encode_place_requests(lws: np.ndarray, groups: np.ndarray, ns_of_lws: Optional[np.ndarray] = None) -> np.ndarray:
    """One request per pod group of an exclusive-topology object (vectorised).

    priority  = mix(owner uid hash, group index): a total order that is stable
                across sweeps and shards (smaller wins);
    group_key = per-group salt of the preference hash (the reference's group key is
                sha1("<ns>/<leader pod name>"), pkg/webhooks/pod_webhook.go:180-182 —
                any stable per-group 64-bit value serves the spec);
    leader_node = the group row's leader node (NONE → the engine chooses).
    Only groups whose leader pod exists take part.
    """
    owner = groups["lws_index"].astype(np.int64)
    excl = (lws["flags"][owner] & R.LWS_EXCLUSIVE_TOPOLOGY) != 0
    present = (groups["flags"] & R.GRP_POD_PRESENT) != 0
    sel = np.flatnonzero(excl & present)
    reqs = R.aligned_empty(len(sel), R.PLACE_REQ)
    o = owner[sel]
    gidx = (sel - lws["group_base"][o].astype(np.int64)).astype(np.uint64)
    uid = lws["uid_hash"][o]
    with np.errstate(over="ignore"):
        pr = (uid ^ (gidx * np.uint64(0x9E3779B97F4A7C15))) * np.uint64(0xBF58476D1CE4E5B9)
        pr ^= pr >> np.uint64(31)
        key = (uid + gidx) * np.uint64(0x94D049BB133111EB)
        key ^= key >> np.uint64(29)
    reqs["priority"] = pr
    reqs["group_key"] = key
    reqs["group"] = sel.astype(np.uint32)
    reqs["ns"] = 0 if ns_of_lws is None else ns_of_lws[o]
    reqs["size"] = lws["size"][o]
    reqs["leader_node"] = groups["leader_node"][sel]
    if ns_of_lws is not None and len(reqs):
        # grouped by namespace (stable: group order inside a namespace): the namespaces are independent
        # sub-problems and the engine gives each its own CTA when the table is laid out this way
        order = np.argsort(reqs["ns"], kind="stable")
        grouped = R.aligned_empty(len(reqs), R.PLACE_REQ)
        grouped[:] = reqs[order]
        reqs = grouped
    return reqs


def sub_group_layout(size: int, sub_group_size: int, leader_excluded: bool) -> list:
    """Worker-index ranges of the subgroups of one group → [(first worker index, pods)], following
    getSubGroupIndex (pkg/webhooks/pod_webhook.go:249-255) and the leader rule (:125-135): the leader
    (worker 0) sits in subgroup 0 unless the policy type is LeaderExcluded; when size - 1 is a multiple of
    the subgroup size the leader is an extra pod of subgroup 0."""
    if sub_group_size <= 0 or size <= 0:
        return []
    index_of = (lambda w: (w - 1) // sub_group_size) if (size - 1) % sub_group_size == 0 else (lambda w: w // sub_group_size)
    members: dict[int, list] = {}
    for w in range(size):
        if w == 0:
            if leader_excluded:
                continue
            members.setdefault(0, []).append(0)
        else:
            members.setdefault(index_of(w), []).append(w)
    return [(min(ws), len(ws)) for _, ws in sorted(members.items())]


def encode_subgroup_place_requests(lws: np.ndarray, groups: np.ndarray, pod_ident: np.ndarray, sub_exclusive: np.ndarray,
                                   ns_of_lws: Optional[np.ndarray] = None, n_namespaces: int = 1) -> np.ndarray:
    """Requests for SUBGROUP-exclusive placement (pod_webhook.go:132-134, :153-155: affinity / anti-affinity on
    the subgroup-key label, same shape as the group-level terms): one request per (group, subgroup) of the
    objects flagged in `sub_exclusive` (bool per object: the subgroup-exclusive-topology annotation is set).

    The anti-affinity term selects on the SUBGROUP key label, so subgroup claims only exclude other
    subgroups — never group-level claims, which select on the group key label.  The two label keys are two
    independent exclusivity classes; a class is addressed as its own namespace id:
    ns' = n_namespaces + ns (group-level requests keep ns).  Pass n_namespaces * 2 to the placement call
    when both kinds are in one table.  `group` carries group row | subgroup index << 24.  The first pod of
    the subgroup decides pinning (its node binding, read from the identity column); groups whose pod rows
    are not the regular size-many (pods in worker-index order) are left to the stock path."""
    out = []
    for li in np.flatnonzero(sub_exclusive):
        size, sg = int(lws["size"][li]), int(lws["subgroup_size"][li])
        excluded = bool(int(lws["flags"][li]) & R.LWS_SUBGROUP_LEADER_EXCLUDED)
        layout = sub_group_layout(size, sg, excluded)
        ns = 0 if ns_of_lws is None else int(ns_of_lws[li])
        uid = int(lws["uid_hash"][li])
        base, count = int(lws["group_base"][li]), int(lws["group_count"][li])
        for gi in range(count):
            g = groups[base + gi]
            if not (int(g["flags"]) & R.GRP_POD_PRESENT) or int(g["pod_count"]) != size or (base + gi) >= (1 << 24):
                continue
            for si, (first_w, pods) in enumerate(layout):
                place = int(pod_ident["place"][int(g["pod_base"]) + first_w])
                node = (place >> R.PODID_NODE_SHIFT) if (place & R.PODID_SCHEDULED) else R.NONE
                mix = (uid ^ ((gi * 0x9E3779B97F4A7C15 + si * 0xC2B2AE3D27D4EB4F) & 0xFFFFFFFFFFFFFFFF)) * 0xBF58476D1CE4E5B9 & 0xFFFFFFFFFFFFFFFF
                mix ^= mix >> 31
                key = ((uid + gi * 131 + si) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
                key ^= key >> 29
                out.append((mix, key, (base + gi) | (si << 24), n_namespaces + ns, pods, node))
    reqs = R.aligned_empty(len(out), R.PLACE_REQ)
    for i, row in enumerate(sorted(out, key=lambda r: r[3])):  # grouped by (class, namespace)
        reqs[i] = row
    return reqs
