"""TEST HARNESS (not product code) for the ProvisioningRequest capacity batch: the two arms and the hand-worked cases.

The reference arm is CapacityChecker.CheckCapacity, the loop of single TrySchedulePods calls with Fork / Commit / Revert on
a copy of the cluster, run on the CPU oracle: it encodes the cluster again for every request, so it shares none of the
device's batch bookkeeping.  The outcome is compared whole: found flags, the node of every pod placed in its request's
simulation, every hint, lastIndex and the cluster with the kept placements."""
import copy

from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo, WithLabels
from kubernetes_autoscaler_b200.provreq import CapacityChecker, PodSet, ProvisioningRequest

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


class OracleSimulator(plp.HintingSimulator):
    """The placement loop on the CPU oracle."""

    def _run(self, x, breakOnFailure):
        from oracle import pyoracle
        return pyoracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, self.last_index, breakOnFailure)


def _outcome(found, cluster, chk):
    sim = chk.schedulingSimulator
    return dict(found=found, assigned=dict(chk.assigned), hints=dict(sim.hints.current), last_index=sim.last_index,
                cluster=[(ni.node.name, [(p.namespace, p.name, p.node_name) for p in ni.pods]) for ni in cluster])


def run(sim, cluster, booked, requests, batch, last_index=0, hints=None, namespaces=()):
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    chk = CapacityChecker(copy.deepcopy(cluster), schedulingSimulator=sim, namespaces=namespaces)
    fn = chk.CheckCapacityBatch if batch else chk.CheckCapacity
    found, after = fn(booked, requests, want_cluster=True)
    return _outcome(found, after, chk)


def oracle_loop(cluster, booked, requests, **kw):
    return run(OracleSimulator(), cluster, booked, requests, False, **kw)


def node(name, cpu=1000, mem=1 << 30, zone=None, pods=110, unschedulable=False):
    n = BuildTestNode(name, cpu, mem)
    n.labels = {HOST: name}
    n.allocatable["pods"] = n.capacity["pods"] = pods
    if zone:
        n.labels[ZONE] = zone
    n.unschedulable = unschedulable
    return n


def pr(name, *sets, ns="default"):
    """A request of pod sets (template, count)."""
    return ProvisioningRequest(name, [PodSet(t, c) for t, c in sets], namespace=ns)


def tmpl(cpu, mem=1000, app="job", **fields):
    p = BuildTestPod("t", cpu, mem, WithLabels({"app": app}))
    for k, v in fields.items():
        setattr(p, k, v)
    return p


# ---- the hand-worked cases: (cluster, booked, requests, kw, expected found flags) ----------------------------------------
def case_compete():
    """Two requests want the same free capacity: the first is found, the second is not."""
    cl = [NodeInfo(node("a", 1000)), NodeInfo(node("b", 1000))]
    return cl, [], [pr("r1", (tmpl(600), 2)), pr("r2", (tmpl(600), 2))], {}, [True, False]


def case_revert_frees_room():
    """r1 places one pod, then fails: reverted, so r2 fits into the room r1 briefly took."""
    cl = [NodeInfo(node("a", 1000))]
    return cl, [], [pr("r1", (tmpl(700), 2)), pr("r2", (tmpl(900), 1))], {}, [False, True]


def case_booking():
    """Booked pods take capacity first and a partly placed booking keeps what it placed: of the four 400m booked pods
    three fit (two on a, one on b), the fourth does not; then a 500m check finds no room, a 150m one does."""
    cl = [NodeInfo(node("a", 1000)), NodeInfo(node("b", 1000), [BuildTestPod("res", 500, 1000)])]
    booked = [pr("old", (tmpl(400), 4))]
    return cl, booked, [pr("r1", (tmpl(500), 1)), pr("r2", (tmpl(150), 1))], {}, [False, True]


def case_empty():
    """A request with no pods is found (0 placed == 0 asked); so is one whose pod set has count 0."""
    cl = [NodeInfo(node("a", 100))]
    return cl, [], [pr("r0"), pr("r1", (tmpl(600), 0)), pr("r2", (tmpl(600), 1))], {}, [True, True, False]


def case_unschedulable():
    """An unschedulable node is never a destination."""
    cl = [NodeInfo(node("a", 4000, unschedulable=True)), NodeInfo(node("b", 1000))]
    return cl, [], [pr("r1", (tmpl(600), 2)), pr("r2", (tmpl(600), 1))], {}, [False, True]


def case_hints_survive_revert():
    """r1 places its first pod on b (the hint), then fails: the hint set there survives the Revert."""
    cl = [NodeInfo(node("a", 1000)), NodeInfo(node("b", 1000))]
    hints = {("default", "r1-0-0"): "b"}
    return cl, [], [pr("r1", (tmpl(900), 3)), pr("r2", (tmpl(900), 2))], dict(hints=hints), [False, True]


def case_last_index():
    """lastIndex moves through a reverted request; r0 has no pods and r2 fits nowhere, so neither scan moves it."""
    cl = [NodeInfo(node(n, 1000)) for n in "abcd"]
    return (cl, [], [pr("r0"), pr("r1", (tmpl(300), 5), (tmpl(900), 4)), pr("r2", (tmpl(5000), 1)), pr("r3", (tmpl(300), 2))],
            dict(last_index=7), [True, False, False, True])


CASES = [case_compete, case_revert_frees_room, case_booking, case_empty, case_unschedulable, case_hints_survive_revert,
         case_last_index]
