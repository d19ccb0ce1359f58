"""Links from DS revision-role rows to resident child LeaderWorkerSets (LWSE_TABLE_DS_LINKS): the rule
the linked DS tick applies, written once more for the oracle comparisons; a seeded world with both
encoders; and size-1 child LeaderWorkerSet tables for the revision-role rows of a synthetic DS table."""
from __future__ import annotations

import numpy as np

from ds_world import DsWorld
from lws_b200 import api, ds_informer, encoder, informer
from lws_b200 import records as R

LOUT_NO_UPDATE = R.LOUT_IRREGULAR | R.LOUT_BAD_TABLE | R.LOUT_RUP_ERROR | R.LOUT_STATUS_ERROR


def linked_revroles(revroles, links, lws=None, lws_out=None):
    """The revision-role rows as the linked DS tick reads them (lwse.h, lwse_ds_link).  Row r with link
    (L, U) takes lws_out[L].ready_replicas when r has RR_EXISTS, LWS results exist (``lws`` and
    ``lws_out`` given: the resident LWS table and the results of its last sweep), L < len(lws),
    lws[L].uid_hash == U and lws_out[L].flags has none of IRREGULAR, BAD_TABLE, RUP_ERROR, STATUS_ERROR;
    otherwise its own ready_replicas.  → (rows, rows that took the LWS value, linked rows that fell back),
    the counts over every row (the engine counts the rows its DS rows reach)."""
    rr = revroles.copy()
    L = links["lws_row"].astype(np.int64)
    linked = L != R.NONE
    ok = linked & ((rr["flags"] & R.RR_EXISTS) != 0)
    if lws is None or lws_out is None:
        ok[:] = False
    else:
        ok &= L < len(lws)
        at = np.where(ok, L, 0)
        if len(lws):
            ok &= lws["uid_hash"][at] == links["lws_uid_hash"]
            ok &= (lws_out["flags"][at] & LOUT_NO_UPDATE) == 0
            rr["ready_replicas"] = np.where(ok, lws_out["ready_replicas"][at], rr["ready_replicas"])
    return rr, int(ok.sum()), int((linked & ~ok).sum())


def none_links(n: int) -> np.ndarray:
    links = R.aligned_empty(n, R.DS_LINK)
    links["lws_row"] = R.NONE
    return links


# --------------------------------------------------------------------------------------------------
# size-1 children of a synthetic DS table
# --------------------------------------------------------------------------------------------------
def child_lws_tables(revroles, rng, p_ready=0.9, spare=0):
    """One size-1 LeaderWorkerSet per existing revision-role row (groups = its replicas, one running
    leader pod per group, ready with probability ``p_ready``), plus ``spare`` empty LWS rows at the end.
    → (lws, groups, pod_state, pod_ident, links): links[r] names row r's child."""
    ex = np.flatnonzero(revroles["flags"] & R.RR_EXISTS)
    n = len(ex) + spare
    reps = np.zeros(n, np.int64)
    reps[: len(ex)] = np.maximum(revroles["replicas"][ex], 0)
    base = np.concatenate([[0], np.cumsum(reps)[:-1]]) if n else np.zeros(0, np.int64)
    G = int(reps.sum())
    lws = R.aligned_empty(n, R.LWS_REC)
    lws["rev_hash"] = rng.integers(1, 2**63, size=n, dtype=np.int64).astype(np.uint64)
    lws["size"] = 1
    lws["flags"] = R.LWS_STS_EXISTS | R.LWS_ANNOT_VALID
    lws["replicas"] = reps
    lws["max_surge"] = 1
    lws["sts_replicas"] = reps
    lws["sts_replicas_annotation"] = reps
    lws["uid_hash"] = rng.integers(1, 2**63, size=n, dtype=np.int64).astype(np.uint64)
    lws["group_base"] = base
    lws["group_count"] = reps
    owner = np.repeat(np.arange(n), reps)
    g = R.aligned_empty(G, R.GROUP_REC)
    g["leader_rev_hash"] = lws["rev_hash"][owner]
    g["wsts_rev_hash"] = lws["rev_hash"][owner]
    g["leader_uid_hash"] = rng.integers(1, 2**31, size=G).astype(np.uint32)
    g["leader_node"] = R.NONE
    g["pod_base"] = np.arange(G)
    g["pod_count"] = 1
    g["lws_index"] = owner
    flags = np.full(G, R.GRP_POD_PRESENT | R.GRP_POD_NAME_MATCH | R.GRP_POD_RUNNING | R.GRP_WSTS_LABEL_NAME_MATCH
                    | R.GRP_WSTS_FOUND | R.GRP_WSTS_REV_SETTLED | R.GRP_REVISION_EXISTS, np.uint32)
    flags |= np.where(rng.random(G) < p_ready, R.GRP_POD_READY, 0).astype(np.uint32)
    g["flags"] = flags
    pst = R.aligned_empty(G, R.POD_STATE)
    pst[:] = (R.POD_PHASE_RUNNING | (R.POD_OWNER_POD << R.POD_OWNER_SHIFT) | R.POD_OWNER_NAME_MATCH
              | R.POD_IS_LEADER)
    pid = R.pod_ident_table(g["leader_rev_hash"], g["leader_uid_hash"], R.PODID_NAME_OK)
    links = none_links(len(revroles))
    links["lws_row"][ex] = np.arange(len(ex))
    links["lws_uid_hash"][ex] = lws["uid_hash"][: len(ex)]
    return lws, g, pst, pid, links


def flip_ready(groups, rng, share):
    """Rows and values of a group patch that flips leader-pod readiness of ``share`` of the groups."""
    rows = np.unique(rng.choice(len(groups), size=max(1, int(len(groups) * share)), replace=False)).astype(np.uint32)
    v = groups[rows].copy()
    v["flags"] ^= np.uint32(R.GRP_POD_READY)
    return rows, v


# --------------------------------------------------------------------------------------------------
# both encoders on one seeded world
# --------------------------------------------------------------------------------------------------
def fresh_links(ds_enc, lws_enc, key) -> np.ndarray:
    """The link rows of a DS's revision-role range, resolved by name now: ``<ds>-<revision>-<role>`` in
    the DS's namespace, over the roles and old revisions of a fresh ``encode_ds``."""
    sl = ds_enc.slots[key]
    t = encoder.encode_ds([ds_enc.item(key)])
    names, old = t.role_names[0], t.old_revisions[0]
    out = none_links(sl.rev_cap)
    for r, rev in enumerate(old + [ds_enc.items[key][1]]):
        for i, role in enumerate(names):
            got = lws_enc.lws_link(key[0], f"{key[1]}-{rev}-{role}")
            if got is not None:
                out[r * len(names) + i] = (got[1], got[0], 0)
    return out


class LinkWorld:
    """A DsWorld plus the child LeaderWorkerSets as objects of an LWS encoder: created (often under a
    child's name, with a new uid each time) and deleted, so LWS rows are taken and reused."""

    def __init__(self, seed: int):
        self.ds = DsWorld(seed)
        self.rng = np.random.default_rng(seed + 1000)
        self.serial = 0
        self.lws: dict[tuple, encoder.LwsItem] = {}
        for name in self._child_names()[::2]:
            self.lws[name] = self._item(*name)
        nodes = [api.Node("n0", {"zone": "z0"}, capacity=64)]
        self.lws_enc = informer.IncrementalEncoder(list(self.lws.values()), encoder.Cluster(nodes=nodes),
                                                   topology_key="zone", namespaces={"a": 0, "b": 1}, spare=4.0)
        self.cap = len(self.lws) + 6
        self.ds_enc = ds_informer.DsIncrementalEncoder(self.ds.initial_items(), spare=1.0, links=self.lws_enc)

    def _child_names(self):
        out = []
        for key in sorted(self.ds.items):
            for (role, rev) in sorted(self.ds.children.get(key, {})):
                out.append((key[0], f"{key[1]}-{rev}-{role}"))
        return out

    def _item(self, ns, name):
        self.serial += 1
        lws = api.LeaderWorkerSet(name=name, namespace=ns, uid=f"uid-{self.serial}", replicas=1, size=1)
        return encoder.LwsItem(lws=lws, revision_key="rev-1")

    def step(self):
        u = self.rng.random()
        if u < 0.45:
            self.ds.step(self.ds_enc)
        elif u < 0.75 and len(self.lws) < self.cap:  # a child (or some other LWS) is created
            names = [n for n in self._child_names() if n not in self.lws]
            if not names or self.rng.random() < 0.2:
                names = [(["a", "b"][int(self.rng.integers(0, 2))], f"other-{int(self.rng.integers(0, 4))}")]
            key = names[int(self.rng.integers(0, len(names)))]
            if key not in self.lws:
                self.lws[key] = self._item(*key)
                self.lws_enc.lws_event("ADDED", self.lws[key])
        elif self.lws:  # deleted: its row is reused by a later create
            keys = sorted(self.lws)
            key = keys[int(self.rng.integers(0, len(keys)))]
            self.lws_enc.lws_event("DELETED", self.lws.pop(key))


# --------------------------------------------------------------------------------------------------
# the executor flows of ds_sim with children that are resident LeaderWorkerSets
# --------------------------------------------------------------------------------------------------
def _child_object(ns, name, replicas, ready):
    """A size-1 LeaderWorkerSet with ``replicas`` groups, each a running leader pod; the first ``ready``
    of them ready.  → (LwsItem, pods)."""
    rev = "rev-1"
    lws = api.LeaderWorkerSet(name=name, namespace=ns, replicas=replicas, size=1,
                              rollingUpdate=api.RollingUpdateConfiguration(0, 1, 0))
    sts = api.StatefulSet(name=name, namespace=ns, replicas=replicas, partition=0,
                          labels={api.SetNameLabelKey: name, api.RevisionKey: rev},
                          annotations={api.ReplicasAnnotationKey: str(replicas)})
    pods = [api.Pod(name=f"{name}-{g}", namespace=ns, phase="Running", readyCondition=g < ready,
                    labels={api.SetNameLabelKey: name, api.GroupIndexLabelKey: str(g),
                            api.WorkerIndexLabelKey: "0", api.RevisionKey: rev})
            for g in range(replicas)]
    return encoder.LwsItem(lws=lws, revision_key=rev, leader_sts=sts), pods


class FlowLoop:
    """Many ``ds_sim.DsSim`` flows of one engine, each child LeaderWorkerSet an object of the LWS tables
    (size 1, one leader pod per replica, as many pods ready as the sim's readyReplicas).  One loop
    iteration (``tick``) is what an operator runs: the watch events since the last iteration go to both
    encoders, one LWS tick, one DS tick; then each sim reconciles on the DS tick's results.

    ``linked``: the DS revision-role rows link to the children; the DS encoder never sees a ready count
    (its children carry readyReplicas = 0), so readiness reaches the DS tick only through the links.
    Unlinked: the DS encoder learns readyReplicas from the status the LWS tick computed, written back
    and delivered as a child MODIFIED event in the next iteration (the status write and its watch event
    are the round trip a link removes)."""

    def __init__(self, engine, sims, linked: bool):
        from ds_sim import DsSim  # noqa: F401  (the sims this loop drives)

        self.engine, self.sims, self.linked = engine, sims, linked
        self.name_of = {}  # (sim index, role, revision) → LWS name
        self.child_of = {}  # (ns, LWS name) → (sim index, role, revision)
        self.pods: dict[tuple, list] = {}  # (ns, LWS name) → the pods sent
        self.lws_snap: dict[tuple, tuple] = {}  # (ns, LWS name) → (replicas, ready) sent
        self.status: dict[tuple, int] = {}  # (sim, role, rev) → readyReplicas the DS encoder has seen
        self.inbox: dict[tuple, int] = {}  # status writes of this iteration, delivered in the next
        items, pods = [], []
        for i, s in enumerate(sims):
            for c in s.children:
                self.status[(i, c.role, c.revision)] = c.readyReplicas
                key, item, ps = self._object(i, s, c)
                items.append(item)
                pods += ps
        self.lws_enc = informer.IncrementalEncoder(items, encoder.Cluster(pods=pods), None, spare=2.0)
        ds_items = [encoder.DsItem(s.ds, s.revision, [self._ds_child(i, c) for c in s.children])
                    for i, s in enumerate(sims)]
        self.ds_enc = ds_informer.DsIncrementalEncoder(ds_items, spare=1.0,
                                                       links=self.lws_enc if linked else None)
        self.ds_snap = [{(c.role, c.revision): self._ds_view(i, c) for c in s.children} for i, s in enumerate(sims)]
        engine.resident_load(*self.lws_enc.full_tables()[:4])
        engine.resident_tick(engine.make_tick(()))
        engine.ds_resident_load(*self.ds_enc.tables())
        self.res = engine.ds_resident_tick([(R.TABLE_DS_LINKS, 0, self.ds_enc.links, True)] if linked else [])
        self.lws_ticks = self.ds_ticks = 0

    def _object(self, i, s, c):
        ns, name = s.ds.namespace, f"{s.ds.name}-{c.revision}-{c.role}"  # GenerateName (utils.go:92-94)
        self.name_of[(i, c.role, c.revision)] = name
        self.child_of[(ns, name)] = (i, c.role, c.revision)
        replicas = 1 if c.replicas is None else c.replicas
        ready = min(c.readyReplicas, replicas)
        item, pods = _child_object(ns, name, replicas, ready)
        self.pods[(ns, name)] = pods
        self.lws_snap[(ns, name)] = (replicas, ready)
        return (ns, name), item, pods

    def _ds_child(self, i, c):
        ready = 0 if self.linked else self.status.get((i, c.role, c.revision), 0)
        return api.ChildLWS(c.role, c.revision, c.replicas, ready, c.creationTimestamp, dict(c.annotations))

    def _ds_view(self, i, c):
        return (c.replicas, c.creationTimestamp, tuple(sorted(c.annotations.items())),
                0 if self.linked else self.status.get((i, c.role, c.revision), 0))

    def _sync(self):
        """The watch events since the last iteration, to both encoders."""
        for k, v in self.inbox.items():
            self.status[k] = v
        self.inbox = {}
        lws_enc, ds_enc = self.lws_enc, self.ds_enc
        for i, s in enumerate(self.sims):
            ns, ds_name = s.ds.namespace, s.ds.name
            now = {(c.role, c.revision): c for c in s.children}
            for (role, rev) in list(self.ds_snap[i]):
                if (role, rev) not in now:  # deleted (cleanupDrainedLWS)
                    key = (ns, self.name_of[(i, role, rev)])
                    item, _ = _child_object(ns, key[1], 0, 0)
                    lws_enc.lws_event("DELETED", item)
                    for p in self.pods.pop(key):
                        lws_enc.pod_event("DELETED", p)
                    del self.lws_snap[key]
                    ds_enc.child_event("DELETED", ns, ds_name, api.ChildLWS(role, rev))
                    del self.ds_snap[i][(role, rev)]
            for (role, rev), c in now.items():
                key = (ns, f"{ds_name}-{rev}-{role}")
                replicas = 1 if c.replicas is None else c.replicas
                want = (replicas, min(c.readyReplicas, replicas))
                if self.lws_snap.get(key) != want:  # created, scaled, or its pods' readiness changed
                    new = key not in self.lws_snap
                    old = {p.name: p for p in self.pods.get(key, [])}
                    _, item, pods = self._object(i, s, c)
                    lws_enc.lws_event("ADDED" if new else "MODIFIED", item)
                    for p in pods:
                        lws_enc.pod_event("MODIFIED" if p.name in old else "ADDED", p)
                    names = {p.name for p in pods}
                    for n, p in old.items():
                        if n not in names:
                            lws_enc.pod_event("DELETED", p)
                view = self._ds_view(i, c)
                if self.ds_snap[i].get((role, rev)) != view:
                    kind = "ADDED" if (role, rev) not in self.ds_snap[i] else "MODIFIED"
                    ds_enc.child_event(kind, ns, ds_name, self._ds_child(i, c))
                    self.ds_snap[i][(role, rev)] = view

    def tick(self):
        """One loop iteration: watch events in, one LWS tick, one DS tick."""
        self._sync()
        p = self.lws_enc.flush()
        assert not self.lws_enc.needs_reload
        got = self.engine.resident_tick(self.engine.make_tick(p.segments))
        self.lws_ticks += 1
        if not self.linked:  # updateConditions → Status().Update: delivered as a watch event next iteration
            for row, out in zip(got["lws_rows"], got["lws_out"]):
                obj = self.lws_enc.object_of_lws_row(int(row))
                if obj is not None and obj in self.child_of:
                    self.inbox[self.child_of[obj]] = int(out["ready_replicas"])
        else:
            self.ds_enc.relink(self.lws_enc.moved_keys)
        p = self.ds_enc.flush()
        assert not self.ds_enc.needs_reload
        self.res = self.engine.ds_resident_tick(p.segments)
        self.ds_ticks += 1

    def sweep_for(self, sim):
        def sweep(t):
            enc = self.ds_enc
            d = enc.ds_row(sim.ds.namespace, sim.ds.name)
            assert enc.role_names(d) == t.role_names[0] and enc.old_revisions(d) == t.old_revisions[0]
            row = enc.ds[d]
            rb, n, vb = int(row["role_base"]), int(row["n_roles"]), int(row["rev_base"])
            nrr = (int(row["n_old_revs"]) + 1) * n
            return (self.res["ds_out"][d: d + 1].copy(), self.res["role_out"][rb: rb + n].copy(),
                    self.res["revrole_out"][vb: vb + nrr].copy())
        return sweep


def steps_of(history):
    """(rollout steps, loop iterations they took): the reconciles after the first whose decisions changed
    a child, and the number of loop iterations from the first reconcile to the last such one."""
    changes = [k for k in range(1, len(history)) if history[k] != history[k - 1]]
    return len(changes), (changes[-1] if changes else 0)
