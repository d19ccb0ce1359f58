"""A random watch-event stream that also adds, changes and deletes Nodes (tests/test_informer_nodes.py,
tests/test_gpu_node_events.py), on top of LeaderWorkerSet creation and deletion: capacity changes,
cordons, relabels to an existing or a new topology value, pods bound to nodes that do not exist yet.
Also the by-name view of a node table, since a fresh encode numbers rows and domains differently."""
import copy

import numpy as np

from lifecycle_world import LifecycleWorld
from lws_b200 import api
from lws_b200 import records as R


class NodeWorld(LifecycleWorld):
    """LifecycleWorld.step plus Node events."""

    def __init__(self, items, cluster, seed=1, p_node=0.25, **kw):
        super().__init__(items, cluster, seed, **kw)
        self.nodes = list(cluster.nodes)
        self.p_node = p_node
        self.n_new = 0  # names node-new-<k> handed out so far
        self.n_zones = 1 + max(int(n.labels["zone"][1:]) for n in self.nodes if "zone" in n.labels)

    def node_names(self):
        return {n.name for n in self.nodes}

    def future_name(self):
        """A node name that does not exist yet but may be added later."""
        return f"node-new-{self.n_new + int(self.rng.integers(0, 3))}"

    def node_event(self, enc, kind=None, name=None, node=None):
        rng = self.rng
        kind = kind if kind is not None else str(rng.choice(["ADDED", "MODIFIED", "MODIFIED", "DELETED"]))
        if kind == "ADDED":
            if node is None:
                name = name if name is not None else f"node-new-{self.n_new}"
                self.n_new += 1
                labels = {} if rng.random() < 0.1 else {"zone": f"z{int(rng.integers(0, self.n_zones + 1))}"}
                node = api.Node(name=name, labels=labels, capacity=int(rng.integers(1, 20)), schedulable=rng.random() < 0.9)
            if node.labels.get("zone") == f"z{self.n_zones}":
                self.n_zones += 1
            if node.name in self.node_names():
                return None
            self.nodes.append(node)
            enc.node_event("ADDED", node)
            return node
        if not self.nodes:
            return None
        i = int(rng.integers(0, len(self.nodes))) if name is None else [n.name for n in self.nodes].index(name)
        if kind == "DELETED":
            node = self.nodes.pop(i)
            enc.node_event("DELETED", node)
            return node
        node = copy.deepcopy(self.nodes[i])
        c = rng.random()
        if c < 0.4:
            node.capacity = int(rng.integers(0, 24))
        elif c < 0.7:
            node.schedulable = not node.schedulable
        elif c < 0.85:
            node.labels = {"zone": f"z{int(rng.integers(0, self.n_zones))}"}  # an existing value
        elif c < 0.95:
            node.labels = {"zone": f"z{self.n_zones}"}  # a new value
            self.n_zones += 1
        else:
            node.labels = {}
        self.nodes[i] = node
        enc.node_event("MODIFIED", node)
        return node

    def bind_to_future_node(self, enc):
        """A pod re-bound to a node that does not exist yet (its scheduler saw the Node first)."""
        if not self.pods:
            return
        key = list(self.pods)[int(self.rng.integers(0, len(self.pods)))]
        p = copy.deepcopy(self.pods[key])
        p.nodeName = self.future_name()
        self.pods[key] = p
        enc.pod_event("MODIFIED", p)

    def step(self, enc):
        r = self.rng.random()
        if r < self.p_node:
            self.serial += 1
            self.node_event(enc)
        elif r < self.p_node + 0.05:
            self.serial += 1
            self.bind_to_future_node(enc)
        else:
            super().step(enc)


def nodes_by_name(rec, names, domain_values):
    """{node name: (topology hash, domain label value or None, capacity, flags)} of a node table."""
    out = {}
    for name, row in names.items():
        r = rec[row]
        d = int(r["domain_id"])
        out[name] = (int(r["topo_value_hash"]), domain_values[d] if d != R.NONE else None, int(r["capacity"]), int(r["flags"]))
    return out


def occupancy_by_name(pod_ident, n_rows, names):
    occ = R.occupancy_of(pod_ident, n_rows)
    return {name: int(occ[row]) for name, row in names.items()}
