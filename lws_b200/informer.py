"""Watch events → row patches: the incremental encoder (SURVEY.md §8(f) rank 1).

The reference reads its world through informer-cache ``List`` calls on every reconcile
(pkg/controllers/leaderworkerset_controller.go:421, :584, :598; pod_controller.go:348).  The
engine keeps the same world as resident record tables; this module keeps them current from the
watch stream, so that a reconcile pass is ``lwse_resident_tick(patches)`` instead of a re-encode:

* the tables are laid out in **slots**: every LeaderWorkerSet owns one LWS row and a fixed range of
  group rows, pod rows and placement-request rows with some slack, so an event never moves another
  object.  The tables carry spare rows of every kind (LWS rows included) and spare namespace ids;
* an event marks its object dirty; ``flush()`` re-encodes just the dirty objects with the very
  function the full encoder uses (``encoder.encode_lws`` on the object's slice of the cache — the
  incremental tables therefore mean exactly what a fresh encode means), compares the fresh rows
  with the resident ones and emits one patch segment per table holding only the rows that differ;
* a LeaderWorkerSet ``ADDED`` takes a vacant LWS row and slot ranges (first fit among the ranges
  freed by earlier deletions, otherwise from the spare tail); pods and StatefulSets seen before
  their set (separate informers do not order events between each other) are cached and encoded
  with it.  ``DELETED`` zeroes the object's LWS, group and pod rows (node occupancy stays exact)
  and makes its request rows inert; its rows are free again from the next ``flush()``;
* Node ``ADDED`` takes a vacant node row (freed by an earlier deletion, from the next ``flush()``
  on, otherwise from the ``node_spare`` tail) and a new topology value the next spare domain id;
  ``MODIFIED`` re-encodes the row in place; ``DELETED`` zeroes it (no request can use a zero row).
  Domain ids are not reused before a reload.  Added and deleted nodes change which row a node name
  means, so every object with a pod bound to that name is re-encoded in the same flush: its pods
  become scheduled on the new row, or unscheduled / NODE_NOT_FOUND, and occupancy stays exact.
  The node rows go out as ``TABLE_NODES`` patches;
* an object that outgrows its slots moves to free rows; when the spare LWS rows, slot rows,
  namespace ids, node rows or domain ids run out ``needs_reload`` is set and the caller re-encodes
  everything (``lwse_resident_load`` / ``lwse_upload_nodes``), which lays objects out in
  (namespace, name) order again.

Rows that no object references (slack, vacant rows) are never read for a result: group rows are
reached through ``lws.group_base/count``, pod rows through ``groups.pod_base/count``; unused
placement-request rows are inert (unpinned, size 0).  Reused request rows can carry another
namespace than their neighbours: the request table is then no longer grouped by namespace, and the
engine's resident tick runs the placement round through a namespace index (DESIGN §3.5).
``object_of_lws_row`` / ``object_of_group_row`` route a changed result row back to its object.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import Optional

import numpy as np

from . import api, encoder
from . import records as R


@dataclass
class Slots:
    lws_row: int
    group_base: int
    group_cap: int
    pod_base: int
    pod_cap: int
    req_base: int  # placement request rows = group rows of exclusive objects (same rows as the group range)


@dataclass
class Patches:
    """One tick's row patches, ready for ``Engine.make_tick`` (rows sorted, distinct)."""

    segments: list = field(default_factory=list)  # (table id, rows uint32, values)

    def add(self, table: int, rows: list, values: np.ndarray):
        if rows:
            order = np.argsort(rows, kind="stable")
            r = np.asarray(rows, dtype=np.uint32)[order]
            v = R.aligned_empty(len(r), values.dtype)
            v[:] = values[order]
            self.segments.append((table, r, v))

    def n_rows(self) -> int:
        return sum(len(s[1]) for s in self.segments)


def _slack(n: int) -> int:
    return n + max(2, n // 4)


def _take(free: list, cap: int) -> Optional[int]:
    """First fit in a list of free [base, length] ranges: the base of `cap` rows, or None."""
    for i, (base, n) in enumerate(free):
        if n >= cap:
            if n == cap:
                free.pop(i)
            else:
                free[i] = [base + cap, n - cap]
            return base
    return None


def _give(free: list, base: int, cap: int):
    """Return a range to a free list, merged with its neighbours."""
    free.append([base, cap])
    free.sort()
    merged = [free[0]]
    for b, n in free[1:]:
        if merged[-1][0] + merged[-1][1] == b:
            merged[-1][1] += n
        else:
            merged.append([b, n])
    free[:] = merged


class IncrementalEncoder:
    """Resident tables + the slice of the informer cache they were encoded from."""

    def __init__(self, items: list, cluster: encoder.Cluster, topology_key: Optional[str] = None,
                 namespaces: Optional[dict] = None, spare: float = 0.25, node_spare: int = 0):
        """``node_spare``: node rows and domain ids kept free for nodes and topology values that appear
        later (0: the node table is exactly ``encoder.encode_nodes`` of the cluster's nodes)."""
        self.topology_key = topology_key
        self.nodes = {n.name: n for n in cluster.nodes}  # node name → Node
        rec, self.domain_values, self.node_index = encoder.encode_nodes(cluster.nodes, topology_key)
        self.node_rec = R.aligned_empty(len(rec) + node_spare, R.NODE_REC)
        self.node_rec[: len(rec)] = rec
        self._encoded_nodes = (self.node_rec, self.domain_values, self.node_index)  # (updated in place)
        self.n_domains = len(self.domain_values) + node_spare  # domain capacity: what upload_nodes takes
        self._domain_ids = {v: d for d, v in enumerate(self.domain_values)}
        self._node_end = len(rec)     # node rows below this one are in use or vacated
        self._free_nodes: list = []   # vacated node rows
        self._node_dirty: set = set()  # node rows written since the last flush
        self._node_resident = self.node_rec.copy()
        self._on_node: dict[str, dict] = {}  # node name → {object key: pods bound to that name}
        self.ns_ids = dict(namespaces or {})  # namespace name → dense id (exclusivity scope)
        self.items: dict[tuple, encoder.LwsItem] = {(it.lws.namespace, it.lws.name): it for it in items}
        self.pods: dict[tuple, dict] = {}  # (ns, set name) → {pod name: Pod}; also for sets not (yet) known
        self.sts: dict[tuple, dict] = {}   # (ns, set name) → {sts name: StatefulSet}  (the leader sts lives in the item)
        for p in cluster.pods:
            self.pods.setdefault((p.namespace, p.labels.get(api.SetNameLabelKey)), {})[p.name] = p
            self._bind(p, 1)
        for s in cluster.statefulsets:
            self.sts.setdefault((s.namespace, s.labels.get(api.SetNameLabelKey)), {})[s.name] = s
        self.needs_reload = False
        self.dirty: set = set()
        self._deleted: set = set()  # objects deleted since the last flush whose rows are still resident
        self.moved_keys: set = set()  # (ns, name) whose LWS row the last flush() took, gave back or re-uid'ed
        # ---- first layout: objects in (namespace id, name) order so that the request table is grouped by namespace
        keys = sorted(self.items, key=lambda k: (self._ns_id(k[0]), k))
        fresh = {k: self._encode_object(k) for k in keys}
        self.slots: dict[tuple, Slots] = {}
        g = p = 0
        for i, k in enumerate(keys):
            gcap, pcap = self._caps(k, len(fresh[k].groups), len(fresh[k].pod_state))
            self.slots[k] = Slots(i, g, gcap, p, pcap, g)
            g, p = g + gcap, p + pcap
        self.order = keys
        n_lws = len(keys)
        self.lws = R.aligned_empty(n_lws + max(4, int(n_lws * spare)), R.LWS_REC)
        self.groups = R.aligned_empty(g + max(16, int(g * spare)), R.GROUP_REC)
        self.pod_state = R.aligned_empty(p + max(64, int(p * spare)), R.POD_STATE)
        self.pod_ident = R.aligned_empty(len(self.pod_state), R.POD_IDENT)
        self.reqs = R.aligned_empty(len(self.groups), R.PLACE_REQ)
        self.n_lws, self.g_end, self.p_end, self.r_end = n_lws, g, p, g
        # free rows below the ends (vacated by deletions and relocations): [base, length] ranges
        self._free_lws: list = []
        self._free_groups: list = []
        self._free_pods: list = []
        self._freed: list = []  # (free list, base, length) released by this flush: free from the next one
        self._lws_key: dict[int, tuple] = {}
        self._group_lws = np.full(len(self.groups), -1, dtype=np.int64)  # group row → owning LWS row, -1 = free
        last_ns = max([self._ns_id(k[0]) for k in keys], default=0)
        self.reqs["leader_node"] = R.NONE  # inert rows: unpinned, size 0 — never claim anything;
        self.reqs["ns"] = last_ns          # the spare tail keeps the table grouped by namespace
        for k in keys:
            self._own(k)
            self._write_object(k, fresh[k], None)
        self.n_namespaces = max(1, last_ns + 1, len(self.ns_ids)) + max(4, int(len(self.ns_ids) * spare))

    # ------------------------------------------------------------------ helpers
    def _bind(self, pod: api.Pod, d: int):
        """Count (d = 1) or forget (d = -1) the pod in the node-name → objects map."""
        if pod.nodeName == "":
            return
        objs = self._on_node.setdefault(pod.nodeName, {})
        key = self._set_key(pod)
        n = objs.get(key, 0) + d
        if n > 0:
            objs[key] = n
        else:
            objs.pop(key, None)
            if not objs:
                del self._on_node[pod.nodeName]

    def _ns_id(self, namespace: str) -> int:
        return self.ns_ids.setdefault(namespace, len(self.ns_ids))

    def _wanted_groups(self, key) -> int:
        it = self.items[key]
        want = it.lws.replicas
        surge, is_pct, ok = encoder.parse_int_or_percent(it.lws.rollingUpdate.maxSurge)
        if ok:
            want += -(-surge * it.lws.replicas // 100) if is_pct else surge
        if it.leader_sts is not None:
            want = max(want, it.leader_sts.replicas)
        return max(want, 0)

    def _caps(self, key, ng: int, npod: int) -> tuple:
        """(group rows, pod rows) of a slot for an object with `ng` groups and `npod` pods."""
        gcap = _slack(max(ng, self._wanted_groups(key)))
        size = max(1, self.items[key].lws.size)
        return gcap, max(_slack(npod), gcap * (size + 1))

    def _encode_object(self, key) -> encoder.LwsTables:
        it = self.items[key]
        cl = encoder.Cluster(pods=list(self.pods.get(key, {}).values()),
                             statefulsets=list(self.sts.get(key, {}).values()))  # (the node table: _encoded_nodes)
        return encoder.encode_lws([it], cl, self.topology_key, encoded_nodes=self._encoded_nodes)

    def _object_requests(self, key, t: encoder.LwsTables, sl: Slots) -> np.ndarray:
        """The request rows of the object's slot range (inert where no exclusive group sits)."""
        out = R.aligned_empty(sl.group_cap, R.PLACE_REQ)
        out["leader_node"] = R.NONE
        out["ns"] = self._ns_id(key[0])
        if len(t.lws) and (int(t.lws["flags"][0]) & R.LWS_EXCLUSIVE_TOPOLOGY) and len(t.groups):
            rq = encoder.encode_place_requests(t.lws, t.groups)
            idx = rq["group"].astype(np.int64)  # group rows of this object start at 0 in its own encode
            rq["group"] = idx + sl.group_base
            rq["ns"] = self._ns_id(key[0])
            out[idx] = rq
        return out

    def _put(self, patches: Optional[Patches], table_id: int, table: np.ndarray, base: int, fresh_rows: np.ndarray):
        """Write rows [base, base + n) of a table; with `patches`, emit the rows that changed."""
        n = len(fresh_rows)
        if n == 0:
            return
        cur = table[base: base + n]
        if patches is None:
            cur[:] = fresh_rows
            return
        a = np.ascontiguousarray(cur).view(np.uint8).reshape(n, -1)
        b = np.ascontiguousarray(fresh_rows).view(np.uint8).reshape(n, -1)
        diff = np.flatnonzero((a != b).any(axis=1))
        if len(diff):
            vals = R.aligned_empty(len(diff), table.dtype)
            vals[:] = fresh_rows[diff]
            cur[diff] = vals
            patches._pending.setdefault(table_id, ([], []))
            patches._pending[table_id][0].extend((diff + base).tolist())
            patches._pending[table_id][1].append(vals)

    def _write_object(self, key, t: encoder.LwsTables, patches: Optional[Patches]):
        """Place the object's fresh rows into its slots; with `patches`, emit the rows that changed."""
        sl = self.slots[key]
        ng, npod = len(t.groups), len(t.pod_state)
        if ng > sl.group_cap or npod > sl.pod_cap:
            if not self._relocate(key, ng, npod, patches):
                self.needs_reload = True
                return
            sl = self.slots[key]
        lws_row = t.lws.copy()
        lws_row["group_base"] = sl.group_base
        grp = t.groups.copy()
        grp["lws_index"] = sl.lws_row
        grp["pod_base"] = grp["pod_base"].astype(np.int64) + sl.pod_base
        reqs = self._object_requests(key, t, sl)

        self._put(patches, R.TABLE_LWS, self.lws, sl.lws_row, lws_row)
        self._put(patches, R.TABLE_GROUPS, self.groups, sl.group_base, grp)
        # the pod columns are written over the WHOLE slot range: rows a shrinking object no longer
        # references go back to zero (the engine counts node occupancy over every identity row)
        pst = R.aligned_empty(sl.pod_cap, R.POD_STATE)
        pst[:npod] = t.pod_state
        pid = R.aligned_empty(sl.pod_cap, R.POD_IDENT)
        pid[:npod] = t.pod_ident
        self._put(patches, R.TABLE_POD_STATE, self.pod_state, sl.pod_base, pst)
        self._put(patches, R.TABLE_POD_IDENT, self.pod_ident, sl.pod_base, pid)
        self._put(patches, R.TABLE_PLACE_REQS, self.reqs, sl.req_base, reqs)

    def _alloc(self, gcap: int, pcap: int) -> Optional[tuple]:
        """(group base, pod base) of free ranges — first fit among freed ranges, else the spare tail — or None."""
        g = _take(self._free_groups, gcap)
        if g is None and self.g_end + gcap <= len(self.groups):
            g, self.g_end = self.g_end, self.g_end + gcap
            self.r_end = self.g_end
        if g is None:
            return None
        p = _take(self._free_pods, pcap)
        if p is None and self.p_end + pcap <= len(self.pod_state):
            p, self.p_end = self.p_end, self.p_end + pcap
        if p is None:
            self._freed.append((self._free_groups, g, gcap))
            return None
        return g, p

    def _vacate(self, sl: Slots, ns: int, patches: Optional[Patches], whole: bool):
        """The object's rows stop taking part: pod rows back to zero (occupancy), request rows inert;
        with `whole` (a deletion) its group rows and LWS row too.  The rows are free from the next flush."""
        inert = R.aligned_empty(sl.group_cap, R.PLACE_REQ)
        inert["leader_node"] = R.NONE
        inert["ns"] = ns
        self._put(patches, R.TABLE_PLACE_REQS, self.reqs, sl.req_base, inert)
        self._put(patches, R.TABLE_POD_STATE, self.pod_state, sl.pod_base, R.aligned_empty(sl.pod_cap, R.POD_STATE))
        self._put(patches, R.TABLE_POD_IDENT, self.pod_ident, sl.pod_base, R.aligned_empty(sl.pod_cap, R.POD_IDENT))
        if whole:
            self._put(patches, R.TABLE_GROUPS, self.groups, sl.group_base, R.aligned_empty(sl.group_cap, R.GROUP_REC))
            self._put(patches, R.TABLE_LWS, self.lws, sl.lws_row, R.aligned_empty(1, R.LWS_REC))
            self._lws_key.pop(sl.lws_row, None)
            self._freed.append((self._free_lws, sl.lws_row, 1))
        self._group_lws[sl.group_base: sl.group_base + sl.group_cap] = -1
        self._freed.append((self._free_groups, sl.group_base, sl.group_cap))
        self._freed.append((self._free_pods, sl.pod_base, sl.pod_cap))

    def _own(self, key):
        sl = self.slots[key]
        self._lws_key[sl.lws_row] = key
        self._group_lws[sl.group_base: sl.group_base + sl.group_cap] = sl.lws_row

    def _relocate(self, key, ng: int, npod: int, patches: Optional[Patches]) -> bool:
        """Move an object that outgrew its slots to free rows."""
        sl = self.slots[key]
        gcap, pcap = self._caps(key, ng, npod)
        got = self._alloc(gcap, pcap)
        if got is None:
            return False
        self._vacate(sl, self._ns_id(key[0]), patches, whole=False)
        self.slots[key] = Slots(sl.lws_row, got[0], gcap, got[1], pcap, got[0])
        self._own(key)
        return True

    def _create(self, key, t: encoder.LwsTables) -> bool:
        """Slots for a new object: a vacant LWS row and free ranges.  False: nothing left, reload."""
        if self._ns_id(key[0]) >= self.n_namespaces:
            return False
        row = _take(self._free_lws, 1)
        if row is None and self.n_lws < len(self.lws):
            row, self.n_lws = self.n_lws, self.n_lws + 1
        if row is None:
            return False
        gcap, pcap = self._caps(key, len(t.groups), len(t.pod_state))
        got = self._alloc(gcap, pcap)
        if got is None:
            self._freed.append((self._free_lws, row, 1))
            return False
        self.slots[key] = Slots(row, got[0], gcap, got[1], pcap, got[0])
        self._own(key)
        return True

    # ------------------------------------------------------------------- events
    def _set_key(self, obj):
        return (obj.namespace, obj.labels.get(api.SetNameLabelKey))

    def pod_event(self, kind: str, pod: api.Pod):
        """kind: ADDED | MODIFIED | DELETED (a watch event of the pod informer).  Pods of a set not
        known (yet, or any more) are only cached."""
        key = self._set_key(pod)
        bucket = self.pods.setdefault(key, {})
        old = bucket.get(pod.name)
        if old is not None:
            self._bind(old, -1)
        if kind == "DELETED":
            bucket.pop(pod.name, None)
        else:
            bucket[pod.name] = pod
            self._bind(pod, 1)
        if key in self.items:
            self.dirty.add(key)

    def statefulset_event(self, kind: str, sts: api.StatefulSet):
        key = self._set_key(sts)
        it = self.items.get(key)
        if it is not None and sts.name == it.lws.name and api.GroupIndexLabelKey not in sts.labels:  # the leader StatefulSet
            it.leader_sts = None if kind == "DELETED" else sts
        else:  # (a leader StatefulSet seen before its set waits here too)
            bucket = self.sts.setdefault(key, {})
            if kind == "DELETED":
                bucket.pop(sts.name, None)
            else:
                bucket[sts.name] = sts
        if it is not None:
            self.dirty.add(key)

    def lws_event(self, kind: str, item: encoder.LwsItem):
        """ADDED | MODIFIED | DELETED of a LeaderWorkerSet.  A new object takes spare rows at the next
        ``flush()``; a deleted one gives its rows back there."""
        key = (item.lws.namespace, item.lws.name)
        if kind == "DELETED":
            if self.items.pop(key, None) is not None:
                self.dirty.discard(key)
                if key in self.slots:
                    self._deleted.add(key)
            return
        keep = self.items.get(key)
        if keep is not None:
            item.leader_sts = item.leader_sts if item.leader_sts is not None else keep.leader_sts
        elif item.leader_sts is None:  # a new object: its leader StatefulSet may already be cached
            bucket = self.sts.get(key, {})
            leader = bucket.get(item.lws.name)
            if leader is not None and api.GroupIndexLabelKey not in leader.labels:
                item.leader_sts = bucket.pop(item.lws.name)
        self.items[key] = item
        self.dirty.add(key)

    def node_event(self, kind: str, node: api.Node):
        """ADDED | MODIFIED | DELETED of a Node.  A node's row changes at once (the objects re-encoded in
        this flush see the new table); the rows go out with the next ``flush()``.  MODIFIED keeps the
        row, and with it every object's rows: the device reads capacity, cordon and domain from the row."""
        row = self.node_index.get(node.name)
        if kind == "DELETED":
            if row is None:
                return
            del self.node_index[node.name]
            self.nodes.pop(node.name, None)
            self.node_rec[row] = np.zeros(1, R.NODE_REC)
            self._node_dirty.add(row)
            self._freed.append((self._free_nodes, row, 1))
            self._touch_bound(node.name)
            return
        val = node.labels.get(self.topology_key) if self.topology_key is not None else None
        if val is not None and val not in self._domain_ids and len(self._domain_ids) >= self.n_domains:
            self.needs_reload = True  # no spare domain id
            return
        if row is None:
            row = _take(self._free_nodes, 1)
            if row is None and self._node_end < len(self.node_rec):
                row, self._node_end = self._node_end, self._node_end + 1
            if row is None:
                self.needs_reload = True  # no spare node row
                return
            self.node_index[node.name] = row
            self._touch_bound(node.name)
        self.nodes[node.name] = node
        n_dom = len(self._domain_ids)
        self.node_rec[row] = encoder.encode_node(node, self.topology_key, self._domain_ids)
        if len(self._domain_ids) > n_dom:
            self.domain_values.append(val)
        self._node_dirty.add(row)

    def _touch_bound(self, node_name: str):
        """Objects with a pod bound to `node_name` are re-encoded in the next flush."""
        for key in self._on_node.get(node_name, {}):
            if key in self.items:
                self.dirty.add(key)

    def flush(self) -> Patches:
        """Re-encode the dirty objects → the patch segments of one ``lwse_resident_tick``."""
        patches = Patches()
        patches._pending = {}
        if self._node_dirty:
            rows = np.array(sorted(self._node_dirty), dtype=np.int64)
            a = self.node_rec[rows].view(np.uint8).reshape(len(rows), -1)
            b = self._node_resident[rows].view(np.uint8).reshape(len(rows), -1)
            changed = rows[(a != b).any(axis=1)]
            self._node_resident[changed] = self.node_rec[changed]
            patches.add(R.TABLE_NODES, changed.tolist(), self.node_rec[changed])
            self._node_dirty.clear()
        self.moved_keys = set(self._deleted)
        for key in sorted(self._deleted):
            self._vacate(self.slots.pop(key), self._ns_id(key[0]), patches, whole=True)
        self._deleted.clear()
        for key in sorted(self.dirty):
            t = self._encode_object(key)
            if key not in self.slots:
                if not self._create(key, t):
                    self.needs_reload = True
                    continue
                self.moved_keys.add(key)
            row = self.slots[key].lws_row
            uid = int(self.lws["uid_hash"][row])
            self._write_object(key, t, patches)
            if int(self.lws["uid_hash"][row]) != uid:  # the object was replaced under its name (a new uid)
                self.moved_keys.add(key)
        self.dirty.clear()
        for free, base, n in self._freed:  # rows given back in this flush may be patched in it: reuse from the next
            _give(free, base, n)
        self._freed.clear()
        for table_id in (R.TABLE_LWS, R.TABLE_GROUPS, R.TABLE_POD_STATE, R.TABLE_POD_IDENT, R.TABLE_PLACE_REQS):
            if table_id in patches._pending:
                rows, chunks = patches._pending[table_id]
                patches.add(table_id, rows, np.concatenate(chunks))
        del patches._pending
        return patches

    # ------------------------------------------------------------- what-if
    # Segments and extra rows for ``Engine.resident_place_whatif``, built from the state of the last
    # ``flush()``.  None of them changes the encoder: no namespace id, slot, spare row or node row is
    # taken.  They model node cordons and capacity changes and new exclusive groups; they do not model
    # node deletion or eviction, which move occupancy (the what-if takes no identity patches).
    def _whatif_nodes(self, names, edit) -> tuple:
        rows = np.array(sorted({self.node_index[n] for n in names}), dtype=np.uint32)
        vals = R.aligned_empty(len(rows), R.NODE_REC)
        vals[:] = self._node_resident[rows]
        edit(vals)
        return R.TABLE_NODES, rows, vals

    def whatif_cordon(self, node_names) -> tuple:
        """A NODES segment of the named nodes' resident rows with NODE_SCHEDULABLE cleared."""
        def cordon(v):
            v["flags"] &= ~np.uint16(R.NODE_SCHEDULABLE)
        return self._whatif_nodes(node_names, cordon)

    def whatif_capacity(self, node_name: str, capacity: int) -> tuple:
        """A NODES segment that sets one node's capacity (pods it can hold)."""
        def resize(v):
            v["capacity"] = capacity
        return self._whatif_nodes([node_name], resize)

    @staticmethod
    def _whatif_requests(uid_hash: int, size: int, ns: int, group_indices) -> np.ndarray:
        """Request rows of an exclusive object's groups whose leader pods exist and are not scheduled, with
        the priority and key mix of ``encoder.encode_place_requests`` (the same function computes them)."""
        gidx = np.asarray(list(group_indices), dtype=np.int64)
        if len(gidx) == 0:
            return R.aligned_empty(0, R.PLACE_REQ)
        lws = R.aligned_empty(1, R.LWS_REC)
        lws["uid_hash"], lws["size"], lws["flags"] = uid_hash, size, R.LWS_EXCLUSIVE_TOPOLOGY
        groups = R.aligned_empty(int(gidx.max()) + 1, R.GROUP_REC)
        groups["leader_node"] = R.NONE
        groups["flags"][gidx] = R.GRP_POD_PRESENT
        reqs = encoder.encode_place_requests(lws, groups)
        reqs["ns"] = ns
        return reqs

    def whatif_new_lws(self, item: encoder.LwsItem) -> tuple:
        """Extra rows for a LeaderWorkerSet that is not resident, created with its ``replicas`` groups
        (indices 0 .. replicas-1, leaders not yet scheduled) → (rows, n_namespaces to pass).  A namespace
        the encoder has not seen gets the id the next flush would give it; n_namespaces covers it."""
        t = encoder.encode_lws([item], encoder.Cluster(pods=[], statefulsets=[]), self.topology_key,
                               encoded_nodes=self._encoded_nodes)
        ns = self.ns_ids.get(item.lws.namespace, len(self.ns_ids))
        n_ns = max(self.n_namespaces, ns + 1)
        if not len(t.lws) or not (int(t.lws["flags"][0]) & R.LWS_EXCLUSIVE_TOPOLOGY):
            return R.aligned_empty(0, R.PLACE_REQ), n_ns
        return self._whatif_requests(int(t.lws["uid_hash"][0]), int(t.lws["size"][0]), ns,
                                     range(max(item.lws.replicas, 0))), n_ns

    def whatif_scale(self, key: tuple, replicas: int) -> np.ndarray:
        """Extra rows for the groups a resident object would add when scaled to ``replicas``: indices from
        its current ``replicas`` up (leaders not yet scheduled).  Empty for a scale-down or a
        non-exclusive object."""
        row = self.slots[key].lws_row
        if not (int(self.lws["flags"][row]) & R.LWS_EXCLUSIVE_TOPOLOGY):
            return R.aligned_empty(0, R.PLACE_REQ)
        return self._whatif_requests(int(self.lws["uid_hash"][row]), int(self.lws["size"][row]), self.ns_ids[key[0]],
                                     range(self.items[key].lws.replicas, replicas))

    def whatif_rollout(self, item: encoder.LwsItem) -> tuple:
        """A proposal for ``Engine.resident_rollout_whatif``: ``item`` is what ``lws_event`` would take for
        the edit (with its own ``revision_key`` and ``lws_updated``), encoded with the object's cached pods
        and StatefulSets as the next ``flush()`` would encode it → (LWS row, LWS_REC row).  Nothing in the
        encoder changes.  KeyError for an object that is not resident."""
        key = (item.lws.namespace, item.lws.name)
        sl = self.slots[key]
        if item.leader_sts is None:  # as lws_event: the cached leader StatefulSet
            item = replace(item, leader_sts=self.items[key].leader_sts)
        cl = encoder.Cluster(pods=list(self.pods.get(key, {}).values()),
                             statefulsets=list(self.sts.get(key, {}).values()))
        t = encoder.encode_lws([item], cl, self.topology_key, encoded_nodes=self._encoded_nodes)
        rec = t.lws.copy()
        rec["group_base"] = sl.group_base
        return sl.lws_row, rec[0]

    def rollout_place_query(self, keys=None) -> tuple:
        """The entries of ``Engine.resident_rollout_place`` for every resident exclusive object, or for the named
        ``keys`` ((namespace, name); non-exclusive ones included, which the call flags) → (rows, ns), in key order.
        Nothing in the encoder changes."""
        if keys is None:
            keys = [k for k, sl in self.slots.items()
                    if int(self.lws["flags"][sl.lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY]
        keys = sorted(keys)
        rows = np.array([self.slots[k].lws_row for k in keys], dtype=np.uint32)
        ns = np.array([self.ns_ids[k[0]] for k in keys], dtype=np.uint32)
        return rows, ns

    def rollout_place_proposal(self, item: encoder.LwsItem) -> tuple:
        """``whatif_rollout``'s proposal plus the object's namespace id → (LWS row, LWS_REC row, ns), for
        ``Engine.resident_rollout_place(rows, ns, recs)``.  KeyError for an object that is not resident."""
        row, rec = self.whatif_rollout(item)
        return row, rec, self.ns_ids[item.lws.namespace]

    def rollout_place_report(self, result: dict) -> list:
        """A ``resident_rollout_place`` answer as dicts, one per entry that strands or bumps, in query order:
        ``namespace`` and ``name`` (None for a row no object holds), then the row's fields, its ``records.RPL_*``
        flags named.  Nothing in the encoder changes."""
        names = {sl.lws_row: k for k, sl in self.slots.items()}
        out = []
        for r, row in zip(np.asarray(result["lws_rows"]).tolist(), result["rows"]):
            if not (int(row["flags"]) & (R.RPL_STRANDS | R.RPL_BUMPS)):
                continue
            ns, name = names.get(int(r), (None, None))
            d = {"namespace": ns, "name": name, **{f: int(row[f]) for f in R.ROLLOUT_PLACE.names}}
            d["flags"] = [v for b, v in R.RPL_NAMES.items() if int(row["flags"]) & b]
            out.append(d)
        return out

    def rollout_place_waves_report(self, result: dict) -> dict:
        """A ``resident_rollout_place_waves`` answer by name → {"waves": per opened wave the (namespace, name) of its
        objects in query order, "unplanned": one dict per key that is not planned, in query order, with
        ``namespace``, ``name``, ``status`` (``records.ROLLW_NAMES``) and ``alone`` (``records.RPW_NAMES``)}.  The
        entries come from ``rollout_place_query`` or ``rollout_place_proposal``.  Nothing in the encoder changes."""
        names = {sl.lws_row: k for k, sl in self.slots.items()}
        waves = [[] for _ in range(len(result["waves"]))]
        unplanned = []
        for r, k in zip(np.asarray(result["lws_rows"]).tolist(), result["keys"]):
            key = names.get(int(r), (None, None))
            if int(k["status"]) == R.ROLLW_PLANNED:
                waves[int(k["wave"])].append(key)
                continue
            unplanned.append({"namespace": key[0], "name": key[1], "status": R.ROLLW_NAMES[int(k["status"])],
                              "alone": [v for b, v in R.RPW_NAMES.items() if int(k["alone"]) & b]})
        return {"waves": waves, "unplanned": unplanned}

    def scale_headroom_query(self, keys=None, ceilings=None) -> tuple:
        """The entries of ``Engine.resident_scale_headroom``: ``rollout_place_query``'s (rows, ns) and, per key,
        its ceiling from ``ceilings`` ({(namespace, name): an HPA's maxReplicas}; -1 for a key not in it)
        → (rows, ns, ceilings), in key order.  Nothing in the encoder changes."""
        if keys is None:
            keys = [k for k, sl in self.slots.items()
                    if int(self.lws["flags"][sl.lws_row]) & R.LWS_EXCLUSIVE_TOPOLOGY]
        keys = sorted(keys)
        rows, ns = self.rollout_place_query(keys)
        ceil = np.array([int((ceilings or {}).get(k, -1)) for k in keys], dtype=np.int32)
        return rows, ns, ceil

    def scale_headroom_report(self, result: dict) -> list:
        """A ``resident_scale_headroom`` answer as dicts, one per entry in query order: ``namespace`` and ``name``
        (None for a row no object holds), ``replicas``, ``max_replicas``, ``headroom`` (max_replicas - replicas,
        None when not answered or blocked), ``limit`` ("ceiling", "strands", "bumps", or None when not answered)
        and the row's ``records.SHR_*`` flags named.  Nothing in the encoder changes."""
        names = {sl.lws_row: k for k, sl in self.slots.items()}
        out = []
        for r, row in zip(np.asarray(result["lws_rows"]).tolist(), result["rows"]):
            f = int(row["flags"])
            ns, name = names.get(int(r), (None, None))
            limit = None
            if f & R.SHR_AT_CEILING:
                limit = "ceiling"
            elif f & R.SHR_STRANDS:
                limit = "strands"
            elif f & R.SHR_BUMPS:
                limit = "bumps"
            ok = (f & R.SHR_SOLVED) and not (f & R.SHR_BLOCKED)
            out.append({"namespace": ns, "name": name, "replicas": int(row["replicas"]),
                        "max_replicas": int(row["max_replicas"]),
                        "headroom": int(row["max_replicas"]) - int(row["replicas"]) if ok else None,
                        "limit": limit, "flags": [v for b, v in R.SHR_NAMES.items() if f & b]})
        return out

    def place_explain_report(self, result: dict, extra_groups=None) -> list:
        """A ``resident_place_explain`` answer as dicts, one per row in answer order: ``namespace``, ``name`` and
        ``group`` (the group index; None for a row no object holds), ``row``, the ``records.PEX_*`` flags named,
        and ``message``, one line in the scheduler's style, e.g. ``0/625 domains available: 402 too small, 3
        without a usable node (12 of these would fit with cordoned nodes), 220 held ahead in the namespace (180
        pinned); 2 slots short in rack-17; would take rack-4, held by ns/lws-a group 3`` (the cordoned count covers
        the too-small and the usable-less domains together).  A request row below the encoder's used request rows
        is its group's row (others name no object); extra row i (the last ``len(extra_groups)`` rows of the round)
        is ``extra_groups[i]``, a (namespace, name, group index) — for ``whatif_scale(key, r)``'s rows,
        ``[(*key, int(g)) for g in rows["group"]]``.  Domain ids are named by their topology values.  Nothing in the
        encoder changes."""
        names = {d: v for v, d in self._domain_ids.items()}
        n_res = int(result["round_rows"]) - len(extra_groups or ())

        def who(row):
            row = int(row)
            if row >= n_res:
                return tuple(extra_groups[row - n_res])
            return self.object_of_group_row(int(self.reqs["group"][row])) if row < self.r_end else None

        def dom(d):
            return names.get(int(d), f"domain {int(d)}")

        def holder(row):
            h = who(row)
            return f"{h[0]}/{h[1]} group {h[2]}" if h else f"row {int(row)}"

        out = []
        for e in result["rows"]:
            f = int(e["flags"])
            key = who(e["row"])
            if f & R.PEX_NO_NAMESPACE:
                msg = "no such namespace"
            else:
                avail = int(e["n_own"]) + int(e["n_open"]) + int(e["n_held_later"])
                ahead = int(e["n_held_pinned"]) + int(e["n_held_earlier"])
                parts = [f"{int(e['n_too_small'])} too small",
                         f"{int(e['n_no_usable'])} without a usable node ({int(e['n_fit_uncordoned'])} of these would fit "
                         "with cordoned nodes)",
                         f"{ahead} held ahead in the namespace ({int(e['n_held_pinned'])} pinned)"]
                msg = f"{avail}/{int(result['n_domains'])} domains available: " + ", ".join(parts)
                if int(e["shortfall_domain"]) != R.NONE:
                    n = int(e["shortfall"])
                    msg += f"; {n} slot{'s' if n != 1 else ''} short in {dom(e['shortfall_domain'])}"
                if f & R.PEX_CONFLICT:
                    msg += f"; leader's domain {dom(e['blocker_domain'])} is held by {holder(e['blocker_row'])}"
                elif int(e["blocker_domain"]) != R.NONE:
                    msg += f"; would take {dom(e['blocker_domain'])}, held by {holder(e['blocker_row'])}"
                if f & R.PEX_NO_CLAIM:
                    msg += "; the leader's node has no topology domain"
                if f & R.PEX_BAD_SIZE:
                    msg += "; size below 1"
            out.append({"namespace": key[0] if key else None, "name": key[1] if key else None,
                        "group": key[2] if key else None, "row": int(e["row"]),
                        "flags": [v for b, v in R.PEX_NAMES.items() if f & b], "message": msg})
        return out

    def whatif_drain(self, node_names) -> np.ndarray:
        """The node rows of the named nodes, for ``Engine.resident_drain_whatif`` (sorted, each once)."""
        return np.array(sorted({self.node_index[n] for n in node_names}), dtype=np.uint32)

    def whatif_drain_domains(self, topology_values) -> np.ndarray:
        """The domain ids of the named topology values, for ``Engine.resident_drain_budget(domains=...)``
        (sorted, each once).  A value no node row has carried is a KeyError."""
        unknown = sorted({v for v in topology_values if v not in self._domain_ids})
        if unknown:
            raise KeyError(f"unknown topology values: {unknown}")
        return np.array(sorted({self._domain_ids[v] for v in topology_values}), dtype=np.uint32)

    def drain_budget_report(self, result: dict) -> list:
        """The touched objects of a ``resident_drain_budget`` answer as dicts: ``namespace`` and ``name`` (None
        for a row no object holds), then the row's fields, its ``records.DRAINB_*`` flags named."""
        names = {R.DRAINB_NOT_EVALUATED: "not_evaluated", R.DRAINB_BREACHED: "breached",
                 R.DRAINB_ALREADY_BELOW: "already_below", R.DRAINB_LOSES_AVAILABLE: "loses_available"}
        out = []
        for r in result["rows"]:
            key = self.object_of_lws_row(int(r["lws"]))
            out.append({"namespace": key[0] if key else None, "name": key[1] if key else None,
                        **{f: int(r[f]) for f in R.DRAIN_BUDGET.names if f != "reserved"},
                        "conditions": [n for bit, n in names.items() if int(r["flags"]) & bit]})
        return out

    def drain_place_query(self, result: dict, node_names) -> list:
        """Segments for ``Engine.resident_place_whatif`` that ask where the groups a drain restarts would go:
        a NODES segment that cordons the drained nodes (``whatif_cordon``) and a PLACE_REQS segment that unpins
        (leader_node = NONE) the request rows of the groups ``result`` (a ``resident_drain_whatif`` answer for
        the same nodes) restarts and of the groups whose leader is on a drained node.  A request row is its
        group's row.

        The answer is conservative: the placement what-if never moves occupancy, so the pods of a restarting
        group on nodes that are not drained still count against those nodes."""
        drained = self.whatif_drain(node_names)
        restart = np.uint32(R.GOUT_DELETE_LEADER | R.GOUT_LEADER_DELETING)
        hit = ((result["before"]["flags"] & restart) == 0) & ((result["after"]["flags"] & restart) != 0)
        rows = set(result["rows"][hit].tolist())
        owned = np.flatnonzero(self._group_lws[: len(self.groups)] >= 0)
        rows |= set(owned[np.isin(self.groups["leader_node"][owned], drained)].tolist())
        rows = np.array(sorted(rows), dtype=np.uint32)
        vals = R.aligned_empty(len(rows), R.PLACE_REQ)
        vals[:] = self.reqs[rows]
        vals["leader_node"] = R.NONE
        return [self.whatif_cordon(node_names), (R.TABLE_PLACE_REQS, rows, vals)]

    def drain_place_report(self, rows, scope: str = "nodes") -> list:
        """A ``resident_drain_place_cost`` answer as dicts, one per key: ``node`` (scope ``"nodes"``) or
        ``topology`` (``"domains"``) — the node's name or the topology value, None for a row nobody holds —
        then the row's fields.  Nothing in the encoder changes."""
        if scope == "nodes":
            names = {row: name for name, row in self.node_index.items()}
            field = "node"
        elif scope == "domains":
            names = {d: v for v, d in self._domain_ids.items()}
            field = "topology"
        else:
            raise ValueError(f"unknown scope {scope!r}")
        return [{field: names.get(k), **{f: int(r[f]) for f in R.DRAIN_PLACE_COST.names if f != "reserved"}}
                for k, r in enumerate(rows)]

    def drain_waves_report(self, result: dict, scope: str = "nodes") -> dict:
        """A ``resident_drain_waves`` answer with names: ``waves``, one list per wave of the node names (scope
        ``"nodes"``) or topology values (``"domains"``) in it, in query order, and ``unplanned``, the keys without a
        wave as (name, status) with status ``"breaches_alone"`` or ``"no_wave"``.  A key nobody holds is named
        None.  Nothing in the encoder changes."""
        if scope == "nodes":
            names = {row: name for name, row in self.node_index.items()}
        elif scope == "domains":
            names = {d: v for v, d in self._domain_ids.items()}
        else:
            raise ValueError(f"unknown scope {scope!r}")
        status = {R.DRAINW_BREACHES_ALONE: "breaches_alone", R.DRAINW_NO_WAVE: "no_wave"}
        waves = [[] for _ in range(len(result["waves"]))]
        unplanned = []
        for k in result["keys"]:
            name = names.get(int(k["id"]))
            if int(k["status"]) == R.DRAINW_PLANNED:
                waves[int(k["wave"])].append(name)
            else:
                unplanned.append((name, status[int(k["status"])]))
        return {"waves": waves, "unplanned": unplanned}

    def ds_drain_waves_report(self, result: dict, scope: str = "nodes") -> dict:
        """A ``resident_ds_drain_waves`` answer with names, as ``drain_waves_report``: ``waves``, one list per wave
        of the node names or topology values in it, and ``unplanned``, the keys without a wave as (name, status,
        alone) with ``alone`` the names (``records.DSW_NAMES``) of the verdicts the key triggers by itself.
        Nothing in the encoder changes."""
        base = self.drain_waves_report(result, scope)
        alone = [[n for bit, n in R.DSW_NAMES.items() if int(k["alone"]) & bit]
                 for k in result["keys"] if int(k["status"]) != R.DRAINW_PLANNED]
        base["unplanned"] = [(name, st, a) for (name, st), a in zip(base["unplanned"], alone)]
        return base

    def drain_place_waves_report(self, result: dict, scope: str = "nodes") -> dict:
        """A ``resident_drain_place_waves`` answer with names, as ``drain_waves_report``: ``waves``, one list per
        wave of the node names or topology values in it, and ``unplanned``, the keys without a wave as (name,
        status, alone) with ``alone`` the names (``records.DPW_NAMES``) of the verdicts the key triggers by itself.
        Nothing in the encoder changes."""
        base = self.drain_waves_report(result, scope)
        alone = [[n for bit, n in R.DPW_NAMES.items() if int(k["alone"]) & bit]
                 for k in result["keys"] if int(k["status"]) != R.DRAINW_PLANNED]
        base["unplanned"] = [(name, st, a) for (name, st), a in zip(base["unplanned"], alone)]
        return base

    # ------------------------------------------------------------------ results
    def tables(self):
        """(lws, groups, pod_state, pod_ident, reqs) trimmed to the rows in use (+ spare already laid out)."""
        return (self.lws[: self.n_lws], self.groups[: self.g_end], self.pod_state[: self.p_end],
                self.pod_ident[: self.p_end], self.reqs[: self.r_end])

    def full_tables(self):
        """The whole allocation, spare rows included (what ``resident_load`` / ``resident_place_load``
        should take, so that new objects and relocations stay in range)."""
        return self.lws, self.groups, self.pod_state, self.pod_ident, self.reqs

    def group_row(self, namespace: str, name: str, group_index: int) -> int:
        return self.slots[(namespace, name)].group_base + group_index

    def lws_row(self, namespace: str, name: str) -> int:
        return self.slots[(namespace, name)].lws_row

    def lws_link(self, namespace: str, name: str) -> Optional[tuple]:
        """(LWS row, uid_hash) of a LeaderWorkerSet as the resident table holds it after the last
        ``flush()``, or None when no row holds it: what a DS revision-role row links to
        (``ds_informer.DsIncrementalEncoder(links=...)``).  ``moved_keys`` names the objects for which
        the answer changed in the last ``flush()``: created, deleted, or given a new uid."""
        sl = self.slots.get((namespace, name))
        if sl is None:
            return None
        return sl.lws_row, int(self.lws["uid_hash"][sl.lws_row])

    def node_row(self, name: str) -> Optional[int]:
        """The node-table row of a node, or None for a node the table does not hold."""
        return self.node_index.get(name)

    def object_of_lws_row(self, row: int) -> Optional[tuple]:
        """(namespace, name) of the object an LWS result row belongs to, or None for a vacant row."""
        return self._lws_key.get(int(row))

    def object_of_group_row(self, row: int) -> Optional[tuple]:
        """(namespace, name, group index) of a group result row, or None for a vacant or slack row."""
        row = int(row)
        lr = int(self._group_lws[row]) if 0 <= row < len(self._group_lws) else -1
        key = self._lws_key.get(lr)
        if key is None:
            return None
        gi = row - self.slots[key].group_base
        return (key[0], key[1], gi) if gi < int(self.lws["group_count"][lr]) else None
