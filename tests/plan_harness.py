"""Shared by the planner-loop tests (cae_plan_removals): the host loop on the CPU oracle, the same loop as one engine call,
both reduced to one comparable outcome, and hand-worked clusters."""
import copy

from kubernetes_autoscaler_b200 import drain as dr
from kubernetes_autoscaler_b200 import planner
from kubernetes_autoscaler_b200.encode import Encoder, encode
from kubernetes_autoscaler_b200.objects import BuildTestPod, LabelSelector, NodeInfo, PodDisruptionBudget, Requirement, WithLabels
from kubernetes_autoscaler_b200.removal import RemovalSimulator
from test_removal_batch import OracleSimulator, _ds, _node, _rs


def _outcome(entries, left, sim, cluster, persist):
    out = dict(results=entries, pdb_left=list(left), hints=dict(sim.hints.current), old=dict(sim.hints.old),
               last_index=sim.last_index)
    if persist:
        out["cluster"] = [(ni.node.name, [(p.name, p.node_name) for p in ni.pods]) for ni in cluster]
    return out


def _byte_of(bytes_by_name):
    return lambda p: bytes_by_name[(p.namespace, p.name)]


def loop_plan(cluster, cands, dest, persist, bytes_by_name, pdbs=(), limit=-1, atomic=None, kube_system=None, last_index=0,
              hints=None):
    """categorize_nodes on the CPU oracle."""
    cluster = copy.deepcopy(cluster)
    sim = OracleSimulator()
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    rs = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    entries, left = planner.categorize_nodes(rs, cands, dest, _byte_of(bytes_by_name), pdbs, limit, atomic, kube_system)
    return _outcome(entries, left, sim, cluster, persist)


def engine_plan(eng, cluster, cands, dest, persist, bytes_by_name, pdbs=(), limit=-1, atomic=None, kube_system=None,
                last_index=0, hints=None, log_cap=None):
    """categorize_nodes_engine after a cae_load of the cluster."""
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    cluster = copy.deepcopy(cluster)
    encoder = Encoder()
    eng.load(encode(cluster, [], [], encoder=encoder))
    sim = plp.HintingSimulator(eng)
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    rs = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    entries, left = planner.categorize_nodes_engine(rs, encoder, cands, dest, _byte_of(bytes_by_name), pdbs, limit, atomic,
                                                    kube_system, log_cap=log_cap)
    return _outcome(entries, left, sim, cluster, persist)


def bytes_of_cluster(cluster, now=0.0):
    """drain.drain_byte of every pod, by (namespace, name)."""
    return {(p.namespace, p.name): dr.drain_byte(p, now) for ni in cluster for p in ni.pods}


def everywhere(cluster):
    return {ni.node.name: True for ni in cluster}


# ---- hand-worked clusters ------------------------------------------------------------------------------------------------
def shared_pdb_cluster():
    """Two candidates, each with one `web` pod under one PDB, and a roomy destination."""
    a = NodeInfo(_node("A", 1000), [_rs(BuildTestPod("a1", 100, 1000, WithLabels({"app": "web"})), "rs-web")])
    b = NodeInfo(_node("B", 1000), [_rs(BuildTestPod("b1", 100, 1000, WithLabels({"app": "web"})), "rs-web")])
    c = NodeInfo(_node("C", 4000), [_rs(BuildTestPod("c1", 100, 1000), "rs-c")])
    return [a, b, c]


def web_pdb(allowed=1, selector=LabelSelector({"app": "web"})):
    return PodDisruptionBudget("web", "default", selector, allowed)


def kube_system_cluster():
    """A kube-system pod on A; B is a plain node."""
    p = _rs(BuildTestPod("dns", 100, 1000, WithLabels({"k8s-app": "dns"})), "rs-dns")
    p.namespace = "kube-system"
    a = NodeInfo(_node("A", 1000), [_ds(BuildTestPod("a-ds", 10, 10)), p])
    b = NodeInfo(_node("B", 4000), [])
    return [a, b]


def dns_pdb(allowed=1):
    return PodDisruptionBudget("dns", "kube-system", LabelSelector(match_expressions=[Requirement("k8s-app", "Exists")]), allowed)


def pdb_before_static_cluster():
    """A: a pod its PDB blocks at position 1, then a not-safe-to-evict pod at position 2."""
    x = _rs(BuildTestPod("x", 100, 1000), "rs-x")
    w = _rs(BuildTestPod("w", 100, 1000, WithLabels({"app": "web"})), "rs-web")
    y = _rs(BuildTestPod("y", 100, 1000), "rs-y")
    y.annotations[dr.SAFE_TO_EVICT_KEY] = "false"
    return [NodeInfo(_node("A", 1000), [x, w, y]), NodeInfo(_node("B", 4000), [])]


def limit_cluster(n=5):
    """n small candidates and one big destination."""
    cl = [NodeInfo(_node("N%d" % i, 1000), [_rs(BuildTestPod("q%d" % i, 100, 1000), "rs-q")]) for i in range(n)]
    return cl + [NodeInfo(_node("BIG", 8000), [])]


def chain_pdb_cluster():
    """A's web pod fits only on B; B is a later candidate: the moved-in pod is checked and counted again."""
    a = NodeInfo(_node("A", 1000), [_rs(BuildTestPod("a1", 600, 1000, WithLabels({"app": "web"})), "rs-web")])
    b = NodeInfo(_node("B", 1000), [])
    c = NodeInfo(_node("C", 700), [])
    return [a, b, c]


def random_pdbs(rng, cluster, n):
    """n PDBs over the cluster's namespaces: nil, {}, matchLabels, In / Gt / Lt expressions (some on values no pod holds),
    budgets 0..3."""
    nss = sorted({p.namespace for ni in cluster for p in ni.pods} | {"default", "nowhere"})
    apps = sorted({p.labels.get("app", "") for ni in cluster for p in ni.pods} - {""}) + ["zzz"]
    out = []
    for b in range(n):
        k = rng.random()
        if k < 0.1:
            sel = None
        elif k < 0.2:
            sel = LabelSelector()
        elif k < 0.6:
            sel = LabelSelector({"app": rng.choice(apps)})
        elif k < 0.75:
            sel = LabelSelector(match_expressions=[Requirement("app", "In", rng.sample(apps, min(2, len(apps))))])
        elif k < 0.9:
            sel = LabelSelector(match_expressions=[Requirement("tier", rng.choice(["Gt", "Lt"]), [str(rng.randint(0, 9))])])
        else:
            sel = LabelSelector(match_expressions=[Requirement("app", "NotIn", ["zzz%d" % b])])
        out.append(PodDisruptionBudget("pdb%d" % b, rng.choice(nss), sel, rng.randint(0, 3)))
    return out


def random_bytes(rng, cluster):
    """Random drain bytes: mostly MOVE / UNDEFINED, some SKIP, BLOCK and late reasons; DaemonSet pods SKIP."""
    out = {}
    for ni in cluster:
        for p in ni.pods:
            if p.owner_kind == "DaemonSet":
                out[(p.namespace, p.name)] = dr.SKIP
                continue
            k = rng.random()
            out[(p.namespace, p.name)] = (dr.MOVE if k < 0.35 else dr.UNDEFINED if k < 0.8 else dr.SKIP if k < 0.88
                                          else dr.UNDEFINED | rng.randint(4, 5) << 4 if k < 0.94 else dr.BLOCK | rng.randint(1, 15) << 4)
    return out


def label_tiers(rng, cluster):
    """A numeric `tier` label on some pods (for Gt / Lt selectors)."""
    for ni in cluster:
        for p in ni.pods:
            if rng.random() < 0.5:
                p.labels = dict(p.labels, tier=str(rng.randint(0, 9)))
    return cluster

