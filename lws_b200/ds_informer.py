"""DisaggregatedSet and child-LeaderWorkerSet watch events → DS row patches.

The reference's DS reconciler is a controller of its own: it watches DisaggregatedSets and the
LeaderWorkerSets they own (disaggregatedset_controller.go:273) and never reads pods.  The engine
keeps its three DS tables resident (``Engine.ds_resident_load``) and runs a DS tick of their own
(``Engine.ds_resident_tick``); this module keeps those tables current from the two watch streams:

* the tables are laid out in **slots**: every DS owns one DS row, a range of role rows and a range
  of revision-role rows, each with some slack, so an event never moves another DS;
* an event marks its DS dirty; ``flush()`` re-encodes just the dirty DS with the very function the
  full encoder uses (``encoder.encode_ds([item])``), rebases the rows to the DS's slot ranges and
  emits only the rows that differ from the resident ones.  Encoding one DS on its own gives it
  creation ranks of its own (1, 2, … over its children's timestamps) instead of ranks over every
  DS: the kernel only compares the ranks of one DS with each other (the newest-first revision
  order of scaleDownOld, executor.go:283-302), so its results are the same;
* child LeaderWorkerSets are keyed by (namespace, DS name, role, revision); children seen before
  their DS (separate informers do not order events between each other) are cached and encoded
  with it;
* a DS ``ADDED`` takes a vacant DS row and ranges (first fit among freed ranges, otherwise from the
  spare tail); a DS whose role or revision-role rows outgrow their range moves that range to a
  first-fit one, and the old range is zeroed; ``DELETED`` zeroes the DS row and both ranges (a zero
  DS row is a vacant DS).  Freed rows are reused from the next ``flush()`` on;
* ``needs_reload`` is set only when spare DS rows, role rows or revision-role rows run out: the
  caller then encodes everything again and calls ``Engine.ds_resident_load``.

``object_of_ds_row``, ``role_names`` and ``old_revisions`` map a changed DS row, and its
``revrole_out`` entries (old revision r, role i at ``rev_base + r * n_roles + i``; the target
revision after the old ones), back to the objects.

With ``links=`` (an ``informer.IncrementalEncoder`` of the same engine's LWS tables) the encoder also
keeps ``links``, the ``TABLE_DS_LINKS`` table beside ``revroles``: revision-role row r of a DS links to
the resident row and uid_hash of the LeaderWorkerSet named ``<ds>-<revision>-<role>`` in the DS's
namespace (GenerateName, pkg/utils/disaggregatedset/utils.go:92-94), or holds ``lws_row = NONE``.  The
DS tick then reads linked children's ready counts from the LWS tick on the device (lwse.h,
``lwse_ds_link``).  Link rows follow the revision-role ranges (moved and freed ranges go back to
``NONE``) and are emitted only where they differ.  The engine's load sets every link to ``NONE``: send
``links`` whole with the first DS tick after ``Engine.ds_resident_load``, as the range segment
``(TABLE_DS_LINKS, 0, links, True)``.  After an LWS ``flush()``, ``relink(lws.moved_keys)``
has the next ``flush()`` re-link just the DS whose children took or gave back an LWS row or changed
uid.  When the LWS encoder is rebuilt (its ``needs_reload``, then ``resident_load``), every row and
uid may have changed: rebuild this encoder with ``links=`` the new LWS encoder and send ``links`` whole
again (or ``relink`` every LWS key).  Without ``links=`` no link table exists and nothing emitted
changes.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import api, encoder
from . import records as R
from .informer import Patches, _give, _slack, _take


@dataclass
class DsSlots:
    ds_row: int
    role_base: int
    role_cap: int
    rev_base: int
    rev_cap: int


class DsIncrementalEncoder:
    """Resident DS tables + the DS objects and child LeaderWorkerSets they were encoded from."""

    def __init__(self, items: list, spare: float = 0.25, links=None):
        """``items``: ``encoder.DsItem`` (their children included).  ``spare``: share of spare rows of
        each table (DS rows, role rows, revision-role rows) kept for later objects and growth.
        ``links``: a resolver with ``lws_link(namespace, name) -> (row, uid_hash) | None`` (the LWS
        ``informer.IncrementalEncoder``); it turns on the link table."""
        self.items: dict[tuple, tuple] = {}      # (ns, name) → (DisaggregatedSet, target revision)
        self.children: dict[tuple, dict] = {}    # (ns, DS name) → {(role, revision): ChildLWS}, List order
        for it in items:
            key = (it.ds.namespace, it.ds.name)
            self.items[key] = (it.ds, it.revision)
            bucket = self.children.setdefault(key, {})
            for c in it.children:
                bucket[(c.role, c.revision)] = c
        fresh = {k: self._encode(k) for k in self.items}
        self.slots: dict[tuple, DsSlots] = {}
        r = v = 0
        for i, k in enumerate(self.items):
            rc, vc = _slack(len(fresh[k].roles)), _slack(len(fresh[k].revroles))
            self.slots[k] = DsSlots(i, r, rc, v, vc)
            r, v = r + rc, v + vc
        n = len(self.items)
        self.ds = R.aligned_empty(n + max(4, int(n * spare)), R.DS_REC)
        self.roles = R.aligned_empty(r + max(16, int(r * spare)), R.DS_ROLE_REC)
        self.revroles = R.aligned_empty(v + max(32, int(v * spare)), R.DS_REVROLE_REC)
        self.n_ds, self.role_end, self.rev_end = n, r, v
        self._free_ds: list = []
        self._free_roles: list = []
        self._free_revroles: list = []
        self._freed: list = []  # (free list, base, length) released by this flush: free from the next one
        self._ds_key: dict[int, tuple] = {}
        self._meta: dict[int, tuple] = {}  # DS row → (role names, old revisions)
        self.needs_reload = False
        self.dirty: set = set()
        self._deleted: set = set()
        self.resolver = links
        self.links = None
        if links is not None:
            self.links = R.aligned_empty(len(self.revroles), R.DS_LINK)
            self.links["lws_row"] = R.NONE
            self._link_names: dict[tuple, set] = {}  # DS key → the (ns, LWS name) its rows resolve
            self._linkers: dict[tuple, set] = {}     # (ns, LWS name) → DS keys that resolve it
            self._relink: set = set()
        for k in self.items:
            self._ds_key[self.slots[k].ds_row] = k
            self._write(k, fresh[k], None)

    # ------------------------------------------------------------------ helpers
    def item(self, key) -> encoder.DsItem:
        """The ``encoder.DsItem`` of a DS as the encoder holds it now."""
        ds, rev = self.items[key]
        return encoder.DsItem(ds, rev, list(self.children.get(key, {}).values()))

    def _encode(self, key) -> encoder.DsTablesHost:
        return encoder.encode_ds([self.item(key)])

    @staticmethod
    def _put(patches: Optional[Patches], table_id: int, table: np.ndarray, base: int, fresh_rows: np.ndarray):
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
            rows, chunks = patches._pending.setdefault(table_id, ([], []))
            rows.extend((diff + base).tolist())
            chunks.append(vals)

    def _alloc(self, free: list, end_attr: str, table: np.ndarray, cap: int) -> Optional[int]:
        base = _take(free, cap)
        end = getattr(self, end_attr)
        if base is None and end + cap <= len(table):
            base = end
            setattr(self, end_attr, end + cap)
        return base

    def _write(self, key, t: encoder.DsTablesHost, patches: Optional[Patches]):
        """Place the DS's fresh rows into its slots (moving an outgrown range); with `patches`, emit
        the rows that changed."""
        sl = self.slots[key]
        n, nrr = len(t.roles), len(t.revroles)
        if n > sl.role_cap:
            cap = _slack(n)
            base = self._alloc(self._free_roles, "role_end", self.roles, cap)
            if base is None:
                self.needs_reload = True
                return
            self._put(patches, R.TABLE_DS_ROLES, self.roles, sl.role_base, R.aligned_empty(sl.role_cap, R.DS_ROLE_REC))
            self._freed.append((self._free_roles, sl.role_base, sl.role_cap))
            sl.role_base, sl.role_cap = base, cap
        if nrr > sl.rev_cap:
            cap = _slack(nrr)
            base = self._alloc(self._free_revroles, "rev_end", self.revroles, cap)
            if base is None:
                self.needs_reload = True
                return
            self._put(patches, R.TABLE_DS_REVROLES, self.revroles, sl.rev_base,
                      R.aligned_empty(sl.rev_cap, R.DS_REVROLE_REC))
            self._unlink_range(patches, sl.rev_base, sl.rev_cap)
            self._freed.append((self._free_revroles, sl.rev_base, sl.rev_cap))
            sl.rev_base, sl.rev_cap = base, cap
        row = t.ds.copy()
        row["role_base"], row["rev_base"] = sl.role_base, sl.rev_base
        # whole slot ranges: rows a shrinking DS no longer references go back to zero
        roles = R.aligned_empty(sl.role_cap, R.DS_ROLE_REC)
        roles[:n] = t.roles
        revroles = R.aligned_empty(sl.rev_cap, R.DS_REVROLE_REC)
        revroles[:nrr] = t.revroles
        self._put(patches, R.TABLE_DS, self.ds, sl.ds_row, row)
        self._put(patches, R.TABLE_DS_ROLES, self.roles, sl.role_base, roles)
        self._put(patches, R.TABLE_DS_REVROLES, self.revroles, sl.rev_base, revroles)
        self._meta[sl.ds_row] = (list(t.role_names[0]), list(t.old_revisions[0]))
        if self.links is not None:
            self._put(patches, R.TABLE_DS_LINKS, self.links, sl.rev_base, self._resolve(key))

    def _create(self, key, t: encoder.DsTablesHost) -> bool:
        """Slots for a new DS: a vacant DS row and free ranges.  False: nothing left, reload."""
        row = _take(self._free_ds, 1)
        if row is None and self.n_ds < len(self.ds):
            row, self.n_ds = self.n_ds, self.n_ds + 1
        if row is None:
            return False
        rc, vc = _slack(len(t.roles)), _slack(len(t.revroles))
        r = self._alloc(self._free_roles, "role_end", self.roles, rc)
        v = self._alloc(self._free_revroles, "rev_end", self.revroles, vc) if r is not None else None
        if r is None or v is None:
            self._freed.append((self._free_ds, row, 1))
            if r is not None:
                self._freed.append((self._free_roles, r, rc))
            return False
        self.slots[key] = DsSlots(row, r, rc, v, vc)
        self._ds_key[row] = key
        return True

    def _vacate(self, key, patches: Patches):
        """A deleted DS: its DS row and both ranges back to zero, free from the next flush."""
        sl = self.slots.pop(key)
        self._put(patches, R.TABLE_DS, self.ds, sl.ds_row, R.aligned_empty(1, R.DS_REC))
        self._put(patches, R.TABLE_DS_ROLES, self.roles, sl.role_base, R.aligned_empty(sl.role_cap, R.DS_ROLE_REC))
        self._put(patches, R.TABLE_DS_REVROLES, self.revroles, sl.rev_base, R.aligned_empty(sl.rev_cap, R.DS_REVROLE_REC))
        self._unlink_range(patches, sl.rev_base, sl.rev_cap)
        if self.links is not None:
            self._index_links(key, set())
        self._ds_key.pop(sl.ds_row, None)
        self._meta.pop(sl.ds_row, None)
        self._freed += [(self._free_ds, sl.ds_row, 1), (self._free_roles, sl.role_base, sl.role_cap),
                        (self._free_revroles, sl.rev_base, sl.rev_cap)]

    # -------------------------------------------------------------------- links
    def _unlink_range(self, patches: Optional[Patches], base: int, n: int):
        """Link rows [base, base + n) back to NONE (a moved or freed revision-role range)."""
        if self.links is not None:
            none = R.aligned_empty(n, R.DS_LINK)
            none["lws_row"] = R.NONE
            self._put(patches, R.TABLE_DS_LINKS, self.links, base, none)

    def _index_links(self, key, names: set):
        for lk in self._link_names.pop(key, set()) - names:
            users = self._linkers.get(lk)
            if users is not None:
                users.discard(key)
                if not users:
                    del self._linkers[lk]
        for lk in names:
            self._linkers.setdefault(lk, set()).add(key)
        if names:
            self._link_names[key] = names

    def _resolve(self, key) -> np.ndarray:
        """The link rows of the DS's whole revision-role range, resolved by child name now."""
        sl = self.slots[key]
        names, old = self._meta[sl.ds_row]
        out = R.aligned_empty(sl.rev_cap, R.DS_LINK)
        out["lws_row"] = R.NONE
        ns, ds_name = key
        used = set()
        for r, rev in enumerate(old + [self.items[key][1]]):
            for i, role in enumerate(names):
                lk = (ns, f"{ds_name}-{rev}-{role}")  # GenerateName (utils.go:92-94)
                used.add(lk)
                got = self.resolver.lws_link(*lk)
                if got is not None:
                    out["lws_row"][r * len(names) + i] = got[0]
                    out["lws_uid_hash"][r * len(names) + i] = got[1]
        self._index_links(key, used)
        return out

    def relink(self, lws_keys):
        """(ns, name) of LeaderWorkerSets whose resident row was taken or given back (the LWS
        encoder's ``moved_keys`` after its ``flush()``): the next ``flush()`` re-links the DS whose
        revision-role rows name them."""
        for lk in lws_keys:
            self._relink.update(self._linkers.get(lk, ()))

    # ------------------------------------------------------------------- events
    def ds_event(self, kind: str, ds: api.DisaggregatedSet, revision: str):
        """ADDED | MODIFIED | DELETED of a DisaggregatedSet; ``revision`` is its target revision
        (ComputeRevision(spec.roles), as in ``encoder.DsItem``)."""
        key = (ds.namespace, ds.name)
        if kind == "DELETED":
            if self.items.pop(key, None) is not None:
                self.dirty.discard(key)
                if key in self.slots:
                    self._deleted.add(key)
            return
        self.items[key] = (ds, revision)
        self._deleted.discard(key)  # (deleted and added again in one flush: it keeps its rows)
        self.dirty.add(key)

    def child_event(self, kind: str, namespace: str, ds_name: str, child: api.ChildLWS):
        """ADDED | MODIFIED | DELETED of a LeaderWorkerSet owned by DS ``ds_name``: the child of
        (role, revision).  Children of a DS not known (yet, or any more) are only cached."""
        key = (namespace, ds_name)
        bucket = self.children.setdefault(key, {})
        if kind == "DELETED":
            bucket.pop((child.role, child.revision), None)
        else:
            bucket[(child.role, child.revision)] = child
        if key in self.items:
            self.dirty.add(key)

    def flush(self) -> Patches:
        """Re-encode the dirty DS → the patch segments of one ``Engine.ds_resident_tick``."""
        patches = Patches()
        patches._pending = {}
        for key in sorted(self._deleted):
            self._vacate(key, patches)
        self._deleted.clear()
        for key in sorted(self.dirty):
            t = self._encode(key)
            if key not in self.slots and not self._create(key, t):
                self.needs_reload = True
                continue
            self._write(key, t, patches)
        if self.links is not None:
            for key in sorted(self._relink - self.dirty):
                if key in self.slots and key in self.items:
                    self._put(patches, R.TABLE_DS_LINKS, self.links, self.slots[key].rev_base, self._resolve(key))
            self._relink.clear()
        self.dirty.clear()
        for free, base, n in self._freed:  # rows given back in this flush may be patched in it: reuse from the next
            _give(free, base, n)
        self._freed.clear()
        for table_id in (R.TABLE_DS, R.TABLE_DS_ROLES, R.TABLE_DS_REVROLES, R.TABLE_DS_LINKS):
            if table_id in patches._pending:
                rows, chunks = patches._pending[table_id]
                patches.add(table_id, rows, np.concatenate(chunks))
        del patches._pending
        return patches

    # ------------------------------------------------------------------ results
    def tables(self):
        """(ds, roles, revroles): the whole allocation, spare rows included (what
        ``Engine.ds_resident_load`` should take, so that new DS and moved ranges stay in range)."""
        return self.ds, self.roles, self.revroles

    def ds_row(self, namespace: str, name: str) -> int:
        return self.slots[(namespace, name)].ds_row

    def object_of_ds_row(self, row: int) -> Optional[tuple]:
        """(namespace, name) of the DS a result row belongs to, or None for a vacant row."""
        return self._ds_key.get(int(row))

    def role_names(self, row: int) -> list:
        """allRoleNames of the DS at `row`: spec roles, then removed roles (role_out / revrole_out order)."""
        return self._meta[int(row)][0]

    def old_revisions(self, row: int) -> list:
        """The old revisions of the DS at `row` in revision-role row order (the target revision follows them)."""
        return self._meta[int(row)][1]

    def ds_drain_report(self, result: dict) -> list:
        """The touched DisaggregatedSets of a ``resident_ds_drain`` answer as dicts: ``namespace`` and ``name``
        (None for a row no DS holds), ``rows_touched`` / ``rows_zeroed``, the ``records.DSD_*`` flags named in
        ``conditions``, ``service_lost`` ({"revision": the target revision, "roles": its spec roles the drain
        takes to zero ready replicas}, or None) and ``old_service_lost`` (one {"revision", "roles"} per old
        revision that loses its service; a DS row carries one role mask for all of them, so each lists the
        roles zeroed in any of those revisions)."""
        names = {R.DSD_TOUCHED: "touched", R.DSD_SERVICE_LOST: "service_lost",
                 R.DSD_OLD_SERVICE_LOST: "old_service_lost", R.DSD_STALLS: "stalls", R.DSD_CHANGED: "changed"}
        out = []
        for r in result["rows"]:
            row, flags = int(r["ds"]), int(r["flags"])
            key = self.object_of_ds_row(row)
            roles = self.role_names(row) if key else []
            old = self.old_revisions(row) if key else []

            def named(mask):
                return [role for i, role in enumerate(roles) if (mask >> i) & 1]

            fell = int(r["before"]["ready_revs"]) & ~int(r["after"]["ready_revs"])
            service = None
            if key and flags & R.DSD_SERVICE_LOST:
                service = {"revision": self.items[key][1], "roles": named(int(r["new_zeroed_roles"]))}
            out.append({"namespace": key[0] if key else None, "name": key[1] if key else None,
                        "rows_touched": int(r["rows_touched"]), "rows_zeroed": int(r["rows_zeroed"]),
                        "conditions": [n for bit, n in names.items() if flags & bit],
                        "service_lost": service,
                        "old_service_lost": [{"revision": rev, "roles": named(int(r["old_zeroed_roles"]))}
                                             for i, rev in enumerate(old) if (fell >> i) & 1]})
        return out

    def whatif_rollout(self, ds: api.DisaggregatedSet, revision: str) -> tuple:
        """A proposal for ``Engine.resident_ds_rollout_whatif``: ``ds`` is the edited object and ``revision`` its
        ComputeRevision(spec.roles), as ``ds_event`` would take them.  The edited object is encoded with the
        DS's cached children, the retired target revision's children last in List order, as the next
        ``flush()`` would encode it once the edit lands.  → (DS_PROPOSAL, DS_MAX_ROLES DS_ROLE_REC rows, the
        encoded role rows first): DSP_NEW_REVISION iff ``revision`` is not the current target, DSP_ROLES iff
        the role rows differ from the resident ones.  Nothing in the encoder changes.  KeyError for a DS that
        is not resident; ValueError for an edit that changes allRoleNames or which of them are in the spec (add,
        remove or rename a role, also one whose children remain, or take a removed role back into the spec) or
        whose revision names an old revision that still has children (re-encode and use
        ``Engine.ds_forecast_host`` for those)."""
        key = (ds.namespace, ds.name)
        sl = self.slots[key]
        current = self.items[key][1]
        kids = list(self.children.get(key, {}).values())
        if revision != current and any(c.revision == revision for c in kids):
            raise ValueError(f"{key}: revision {revision} still has children")
        kids = [c for c in kids if c.revision != current] + [c for c in kids if c.revision == current]
        t = encoder.encode_ds([encoder.DsItem(ds, revision, kids)])
        names = self.role_names(sl.ds_row)
        if list(t.role_names[0]) != names:
            raise ValueError(f"{key}: the edit changes the roles {names} to {list(t.role_names[0])}")
        # allRoleNames alone misses a spec role dropped while its children remain (it stays, as a removed role)
        # and a removed role taken back into the spec: the spec / removed split moves, which a proposal keeps
        n_spec = int(self.ds[sl.ds_row]["n_spec_roles"])
        if int(t.ds[0]["n_spec_roles"]) != n_spec:
            raise ValueError(f"{key}: the edit changes the spec roles {names[:n_spec]} to "
                             f"{names[:int(t.ds[0]['n_spec_roles'])]}")
        n = len(names)
        roles = R.aligned_empty(R.DS_MAX_ROLES, R.DS_ROLE_REC)
        roles[:n] = t.roles
        flags = R.DSP_NEW_REVISION if revision != current else 0
        if roles[:n].tobytes() != self.roles[sl.role_base: sl.role_base + n].tobytes():
            flags |= R.DSP_ROLES
        p = np.zeros(1, R.DS_PROPOSAL)
        p[0] = (sl.ds_row, flags)
        return p[0], roles

    def whatif_of(self, answer: dict, i: int, namespace: str, name: str) -> dict:
        """Proposal i of a ``resident_ds_rollout_whatif`` answer on the named DS, as ``forecast_of`` names a
        forecast, plus ``now`` (the DS_OUT row) and per role its ``next`` (old, new) from ``now_roles``.  A
        template edit adds the retired target revision as the last old revision (bit len(old_revisions) of
        drained_revs / ready_revs)."""
        names = self.role_names(self.ds_row(namespace, name))
        n, base = len(names), i * R.DS_MAX_ROLES
        out = self._named(answer["ds"][i], answer["roles"][base: base + n], answer.get("steps"), names)
        out["now"] = answer["now"][i]
        for j, role in enumerate(names):
            r = answer["now_roles"][base + j]
            out["roles"][role]["next"] = (int(r["next_old"]), int(r["next_new"]))
        return out

    def forecast_of(self, forecast: dict, namespace: str, name: str) -> dict:
        """One DS's rollout forecast (``Engine.ds_resident_forecast`` over ``tables()``), by name:
        the flags, cycle and step counts, and per role name its peak replicas, availability floor,
        final old / new counts and trajectory [(old, new), ...] (empty without trajectory rows, or
        when the DS's rows did not fit)."""
        row = self.ds_row(namespace, name)
        role_base = int(self.ds[row]["role_base"])
        names = self.role_names(row)
        return self._named(forecast["ds"][row], forecast["roles"][role_base: role_base + len(names)],
                           forecast.get("steps"), names)

    @staticmethod
    def _named(fc, role_rows, steps, names) -> dict:
        """A forecast row and its role rows, by role name (``forecast_of``, ``whatif_of``)."""
        n, base, n_steps = len(names), int(fc["step_base"]), int(fc["n_steps"])
        have = steps is not None and not fc["flags"] & R.DSF_TRUNCATED and base + n_steps * n <= len(steps)
        roles = {}
        for i, role in enumerate(names):
            r = role_rows[i]
            traj = ([(int(steps[base + s * n + i]["next_old"]), int(steps[base + s * n + i]["next_new"]))
                     for s in range(n_steps)] if have else [])
            roles[role] = {"peak_replicas": int(r["peak_replicas"]), "floor_available": int(r["floor_available"]),
                           "final_old": int(r["final_old"]), "final_new": int(r["final_new"]), "trajectory": traj}
        return {"flags": int(fc["flags"]), "cycles": int(fc["cycles"]), "n_steps": n_steps, "roles": roles}
