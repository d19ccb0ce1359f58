"""A seeded stream of DisaggregatedSet and child-LeaderWorkerSet watch events, and the checks that the
DS encoder's patched tables mean what a fresh ``encoder.encode_ds`` of the same objects means."""
from __future__ import annotations

import numpy as np

import oracle
from lws_b200 import api, encoder
from lws_b200 import records as R

DS_TABLES = {R.TABLE_DS: 0, R.TABLE_DS_ROLES: 1, R.TABLE_DS_REVROLES: 2}


class DsWorld:
    """The objects as the API server holds them; every change comes out as the watch event it causes."""

    def __init__(self, seed: int, n_ds: int = 6):
        self.rng = np.random.default_rng(seed)
        self.clock = 1000.0
        self.items: dict[tuple, tuple] = {}   # (ns, name) → (DisaggregatedSet, target revision)
        self.children: dict[tuple, dict] = {}  # (ns, name) → {(role, revision): ChildLWS}
        self.revno: dict[tuple, int] = {}
        self.next_name = 0
        for _ in range(n_ds):
            key, ds = self._new_ds()
            self.items[key] = (ds, "r0")
            self.children[key] = {}
            for role in ds.roles:
                self._child(key, role.name, "r0")

    def _new_ds(self):
        ns = ["a", "b"][int(self.rng.integers(0, 2))]
        name = f"ds-{self.next_name}"
        self.next_name += 1
        n = int(self.rng.integers(2, 5))
        roles = [self._role(f"role{i}") for i in range(n)]
        self.revno[(ns, name)] = 0
        return (ns, name), api.DisaggregatedSet(name, ns, roles=roles)

    def _role(self, name):
        rng = self.rng
        replicas = None if rng.random() < 0.1 else int(rng.integers(0, 6))
        ru = None
        if rng.random() < 0.6:
            surge = [1, 2, "25%", "x"][int(rng.integers(0, 4))]
            unav = [0, 1, "50%"][int(rng.integers(0, 3))]
            ru = api.RollingUpdateConfiguration(maxSurge=surge, maxUnavailable=unav)
        return api.DisaggregatedRoleSpec(name, replicas, ru)

    def _child(self, key, role, rev):
        rng = self.rng
        self.clock += float(rng.integers(0, 2))  # equal stamps happen
        ann = {}
        if rng.random() < 0.3:
            ann[api.DSInitialReplicasAnnotationKey] = ["3", "", "x", "0"][int(rng.integers(0, 4))]
        replicas = None if rng.random() < 0.1 else int(rng.integers(0, 6))
        c = api.ChildLWS(role, rev, replicas, int(rng.integers(0, 6)), self.clock, ann)
        self.children.setdefault(key, {})[(role, rev)] = c
        return c

    def item(self, key) -> encoder.DsItem:
        ds, rev = self.items[key]
        return encoder.DsItem(ds, rev, list(self.children.get(key, {}).values()))

    def initial_items(self):
        return [self.item(k) for k in self.items]

    def step(self, enc):
        """One random change, handed to the encoder as its watch event."""
        rng = self.rng
        u = rng.random()
        keys = sorted(self.items)
        if u < 0.08 or not keys:  # a new DS; sometimes its children arrive first
            key, ds = self._new_ds()
            early = rng.random() < 0.5
            kids = [self._child(key, r.name, "r0") for r in ds.roles if rng.random() < 0.7]
            if early:
                for c in kids:
                    enc.child_event("ADDED", key[0], key[1], c)
            self.items[key] = (ds, "r0")
            enc.ds_event("ADDED", ds, "r0")
            if not early:
                for c in kids:
                    enc.child_event("ADDED", key[0], key[1], c)
            return
        key = keys[int(rng.integers(0, len(keys)))]
        ds, rev = self.items[key]
        if u < 0.13:  # deleted (its children go with it, as the garbage collector deletes them)
            del self.items[key]
            enc.ds_event("DELETED", ds, rev)
            for c in list(self.children.pop(key, {}).values()):
                enc.child_event("DELETED", key[0], key[1], c)
            return
        if u < 0.25:  # a spec change: new target revision; sometimes a role removed or added
            roles = list(ds.roles)
            if len(roles) > 2 and rng.random() < 0.3:
                roles.pop(int(rng.integers(0, len(roles))))
            elif len(roles) < 6 and rng.random() < 0.3:
                roles.append(self._role(f"role{len(roles) + int(rng.integers(0, 3))}"))
                if len({r.name for r in roles}) < len(roles):
                    roles.pop()
            roles = [self._role(r.name) if rng.random() < 0.5 else r for r in roles]
            self.revno[key] += 1
            rev = f"r{self.revno[key]}"
            ds = api.DisaggregatedSet(ds.name, ds.namespace, uid=ds.uid, roles=roles)
            self.items[key] = (ds, rev)
            enc.ds_event("MODIFIED", ds, rev)
            return
        kids = self.children.setdefault(key, {})
        if u < 0.45 or not kids:  # a child of the target revision (or an older one) appears
            revs = [rev] + sorted({r for (_, r) in kids})
            names = [r.name for r in ds.roles] + ["gone"]
            c = self._child(key, names[int(rng.integers(0, len(names)))], revs[int(rng.integers(0, len(revs)))])
            enc.child_event("ADDED", key[0], key[1], c)
            return
        ck = sorted(kids)[int(rng.integers(0, len(kids)))]
        c = kids[ck]
        if u < 0.55:
            del kids[ck]
            enc.child_event("DELETED", key[0], key[1], c)
            return
        c = api.ChildLWS(c.role, c.revision, c.replicas, c.readyReplicas, c.creationTimestamp, dict(c.annotations))
        if rng.random() < 0.6:  # the common event: a status update
            c.readyReplicas = int(rng.integers(0, 6))
        else:
            c.replicas = None if rng.random() < 0.15 else int(rng.integers(0, 6))
        kids[ck] = c
        enc.child_event("MODIFIED", key[0], key[1], c)


def apply_patches(mirror, patches):
    for table, rows, values in patches.segments:
        mirror[DS_TABLES[table]][rows] = values


def _dense_ranks(revroles: np.ndarray) -> np.ndarray:
    """The creation-rank bits of one DS's revision-role rows, renumbered 1, 2, … in order."""
    rr = revroles.copy()
    flags = rr["flags"].astype(np.uint64)
    exists = (flags & R.RR_EXISTS) != 0
    ts = flags >> R.RR_TS_SHIFT
    uniq = np.unique(ts[exists])
    dense = np.searchsorted(uniq, ts) + 1
    low = flags & ((1 << R.RR_TS_SHIFT) - 1)
    rr["flags"] = np.where(exists, low | (dense.astype(np.uint64) << R.RR_TS_SHIFT), flags).astype(np.uint32)
    return rr


def per_ds(ds, roles, revroles, d):
    """(DS row with its bases zeroed, role rows, revision-role rows with dense ranks) of DS row d."""
    row = ds[d: d + 1].copy()
    rb, n, vb, v = int(row["role_base"][0]), int(row["n_roles"][0]), int(row["rev_base"][0]), int(row["n_old_revs"][0])
    row["role_base"], row["rev_base"] = 0, 0
    return row, roles[rb: rb + n], _dense_ranks(revroles[vb: vb + (v + 1) * n])


def outputs_of_ds(ds, outs, d):
    ds_out, role_out, rr_out = outs
    rb, n, vb, v = (int(ds["role_base"][d]), int(ds["n_roles"][d]), int(ds["rev_base"][d]), int(ds["n_old_revs"][d]))
    return ds_out[d].tobytes(), role_out[rb: rb + n].tobytes(), rr_out[vb: vb + (v + 1) * n].tobytes()


def check_against_fresh(world: DsWorld, enc, mirror, where, got_outputs=None):
    """The mirror (the resident tables with every patch applied) against a fresh encode of the same
    objects, DS by DS: the same rows (creation ranks made dense per DS) and the same oracle results.
    ``got_outputs``: the engine's output tables for the mirror, checked against the oracle too."""
    keys = sorted(world.items)
    assert sorted(enc.items) == keys, where
    fresh = encoder.encode_ds([world.item(k) for k in keys])
    want = oracle.sweep_ds(fresh.ds, fresh.roles, fresh.revroles)
    got = oracle.sweep_ds(*mirror)
    owned = set()
    for i, key in enumerate(keys):
        d = enc.ds_row(*key)
        owned.add(d)
        assert enc.object_of_ds_row(d) == key, where
        a, b = per_ds(*mirror, d), per_ds(fresh.ds, fresh.roles, fresh.revroles, i)
        for x, y, what in zip(a, b, ("ds", "roles", "revroles")):
            assert x.tobytes() == y.tobytes(), f"{where}: {key} {what}"
        assert outputs_of_ds(mirror[0], got, d) == outputs_of_ds(fresh.ds, want, i), f"{where}: {key} oracle"
        assert enc.role_names(d) == fresh.role_names[i] and enc.old_revisions(d) == fresh.old_revisions[i], where
        if got_outputs is not None:
            assert outputs_of_ds(mirror[0], got_outputs, d) == outputs_of_ds(mirror[0], got, d), f"{where}: {key} engine"
    for d in range(len(mirror[0])):
        if d not in owned:
            assert enc.object_of_ds_row(d) is None, where
            assert mirror[0][d].tobytes() == bytes(R.DS_REC.itemsize), where
