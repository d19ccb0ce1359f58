"""A random watch-event stream that also creates and deletes LeaderWorkerSets (tests/test_informer_lifecycle.py,
tests/test_gpu_lifecycle.py): new namespaces, delete and re-create under the same name, pods delivered
before their set, exclusive and non-exclusive objects."""
import copy

from informer_world import World
from lws_b200 import api, encoder


def new_object(rng, name, ns, n_nodes, exclusive, size=None, replicas=None, topology_key="zone"):
    """(item, pods, worker statefulsets) of one running LeaderWorkerSet, as make_world builds them."""
    size = int(rng.choice([1, 2, 3])) if size is None else size
    replicas = int(rng.choice([1, 2, 3])) if replicas is None else replicas
    ann = {api.ExclusiveKeyAnnotationKey: topology_key} if exclusive else {}
    lws = api.LeaderWorkerSet(name=name, namespace=ns, replicas=replicas, size=size, annotations=ann,
                              rollingUpdate=api.RollingUpdateConfiguration(0, 1, 0))
    rev = "rev-1"
    sts = api.StatefulSet(name=name, namespace=ns, replicas=replicas, partition=0,
                          labels={api.SetNameLabelKey: name, api.RevisionKey: rev},
                          annotations={api.ReplicasAnnotationKey: str(replicas)})
    pods, stss = [], []
    for g in range(replicas):
        node = f"node-{int(rng.integers(0, n_nodes))}" if rng.random() < 0.7 else ""
        leader = api.Pod(name=f"{name}-{g}", namespace=ns, phase="Running", readyCondition=True, nodeName=node,
                         labels={api.SetNameLabelKey: name, api.GroupIndexLabelKey: str(g),
                                 api.WorkerIndexLabelKey: "0", api.RevisionKey: rev})
        pods.append(leader)
        if size > 1:
            w = api.StatefulSet(name=leader.name, namespace=ns, replicas=size - 1, availableReplicas=size - 1,
                                currentRevision="a", updateRevision="a",
                                labels={api.SetNameLabelKey: name, api.GroupIndexLabelKey: str(g), api.RevisionKey: rev},
                                ownerReferences=[api.OwnerReference("Pod", leader.name, leader.uid)])
            stss.append(w)
            for wi in range(1, size):
                pods.append(api.Pod(name=f"{leader.name}-{wi}", namespace=ns, phase="Running", readyCondition=True,
                                    labels={api.SetNameLabelKey: name, api.GroupIndexLabelKey: str(g),
                                            api.WorkerIndexLabelKey: str(wi), api.RevisionKey: rev},
                                    ownerReferences=[api.OwnerReference("StatefulSet", w.name, w.uid)], nodeName=node))
    return encoder.LwsItem(lws=lws, revision_key=rev, leader_sts=sts), pods, stss


class LifecycleWorld(World):
    """World.step plus LeaderWorkerSet creation and deletion."""

    def __init__(self, items, cluster, seed=1, p_create=0.12, p_delete=0.08, new_namespaces=2, names=6):
        super().__init__(items, cluster, seed)
        self.p_create, self.p_delete = p_create, p_delete
        self.namespaces = sorted({k[0] for k in self.items}) + [f"ns-new-{j}" for j in range(new_namespaces)]
        self.names = [f"lws-c{j}" for j in range(names)]  # a small pool: deleted names come back

    def create(self, enc, ns=None, name=None, exclusive=None, size=None, replicas=None):
        rng = self.rng
        ns = ns if ns is not None else str(rng.choice(self.namespaces))
        free = [n for n in self.names if (ns, n) not in self.items]
        if name is None and not free:
            return None
        name = name if name is not None else str(rng.choice(free))
        exclusive = bool(rng.random() < 0.6) if exclusive is None else exclusive
        item, pods, stss = new_object(rng, name, ns, len(self.nodes), exclusive, size, replicas)
        early = rng.random() < 0.5  # pods and worker sets reach the encoder before their set
        if early:
            self._deliver(enc, pods, stss)
        self.items[(ns, name)] = item
        enc.lws_event("ADDED", copy.deepcopy(item))
        if not early:
            self._deliver(enc, pods, stss)
        return (ns, name)

    def _deliver(self, enc, pods, stss):
        for s in stss:
            self.stss[(s.namespace, s.name)] = s
            enc.statefulset_event("ADDED", s)
        for p in pods:
            kind = "MODIFIED" if (p.namespace, p.name) in self.pods else "ADDED"
            self.pods[(p.namespace, p.name)] = p
            enc.pod_event(kind, p)

    def delete(self, enc, key=None):
        rng = self.rng
        if len(self.items) <= 1:
            return None
        key = key if key is not None else list(self.items)[int(rng.integers(0, len(self.items)))]
        item = self.items.pop(key)
        enc.lws_event("DELETED", item)
        # the garbage collector removes (some of) the pods and worker sets now, the rest later
        for pk in [k for k, p in self.pods.items() if (p.namespace, p.labels.get(api.SetNameLabelKey)) == key]:
            if rng.random() < 0.7:
                enc.pod_event("DELETED", self.pods.pop(pk))
        for sk in [k for k, s in self.stss.items() if (s.namespace, s.labels.get(api.SetNameLabelKey)) == key]:
            enc.statefulset_event("DELETED", self.stss.pop(sk))
        return key

    def step(self, enc):
        r = self.rng.random()
        if r < self.p_create:
            self.serial += 1
            self.create(enc)
        elif r < self.p_create + self.p_delete:
            self.serial += 1
            self.delete(enc)
        else:
            super().step(enc)
