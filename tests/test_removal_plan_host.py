"""The planner's removal loop on the host (planner.categorize_nodes over the CPU oracle), the drainability rules and the
PDB tracker it uses (drain.py), and the ABI of cae_plan_removals."""
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200 import drain as dr
from kubernetes_autoscaler_b200.objects import BuildTestPod, LabelSelector, PodDisruptionBudget, Requirement, WithLabels
from plan_harness import (bytes_of_cluster, chain_pdb_cluster, dns_pdb, everywhere, kube_system_cluster, limit_cluster,
                          loop_plan, pdb_before_static_cluster, shared_pdb_cluster, web_pdb)


def _pod(**kw):
    p = BuildTestPod("p", 100, 1000)
    p.owner_uid, p.owner_kind = "rs", "ReplicaSet"
    for k, v in kw.items():
        setattr(p, k, v)
    return p


# ---- drain bytes: one known answer per rule, in rules.Default's order ------------------------------------------------
def test_drain_byte_per_rule():
    now = 1000.0
    assert dr.drain_byte(_pod(annotations={"kubernetes.io/config.mirror": "x"}), now) == dr.SKIP               # mirror
    assert dr.drain_byte(_pod(deletion_timestamp=0.0, termination_grace_period_seconds=30), now) == dr.SKIP    # long-terminating
    assert dr.drain_byte(_pod(), now, lister_reason=lambda p, r: dr.MIN_REPLICAS_REACHED if r == "replicacount" else 0) \
        == dr.BLOCK | dr.MIN_REPLICAS_REACHED << 4                                                             # replica count
    assert dr.drain_byte(_pod(owner_kind="DaemonSet"), now) == dr.SKIP                                         # daemonset
    assert dr.drain_byte(_pod(owner_uid="", annotations={dr.SAFE_TO_EVICT_KEY: "true"}), now) == dr.MOVE       # safe-to-evict
    assert dr.drain_byte(_pod(owner_uid="", phase="Succeeded", restart_policy="Never"), now) == dr.MOVE        # terminal
    assert dr.drain_byte(_pod(owner_uid="", phase="Succeeded", restart_policy="OnFailure"), now) == dr.MOVE
    assert dr.drain_byte(_pod(owner_uid="", phase="Failed"), now) == dr.MOVE
    assert dr.drain_byte(_pod(owner_uid="", phase="Succeeded"), now) == dr.BLOCK | dr.NOT_REPLICATED << 4        # Always restarts
    assert dr.drain_byte(_pod(owner_uid=""), now) == dr.BLOCK | dr.NOT_REPLICATED << 4                         # replicated
    assert dr.drain_byte(_pod(owner_kind="CustomThing"), now) == dr.BLOCK | dr.NOT_REPLICATED << 4
    assert dr.drain_byte(_pod(owner_kind="CustomThing"), now, dr.DrainOptions(skip_nodes_with_custom_controller_pods=False)) \
        == dr.UNDEFINED
    assert dr.drain_byte(_pod(), now, lister_reason=lambda p, r: dr.CONTROLLER_NOT_FOUND if r == "replicated" else 0) \
        == dr.BLOCK | dr.CONTROLLER_NOT_FOUND << 4
    assert dr.drain_byte(_pod(namespace="kube-system"), now) == dr.UNDEFINED                                   # system: late, by PDBs
    assert dr.drain_byte(_pod(annotations={dr.SAFE_TO_EVICT_KEY: "false"}), now) == dr.UNDEFINED | dr.NOT_SAFE_TO_EVICT << 4
    assert dr.drain_byte(_pod(local_storage=True), now) == dr.UNDEFINED | dr.LOCAL_STORAGE << 4                # local storage
    assert dr.drain_byte(_pod(local_storage=True), now, dr.DrainOptions(skip_nodes_with_local_storage=False)) == dr.UNDEFINED
    assert dr.drain_byte(_pod(), now) == dr.UNDEFINED                                                          # pdb: by budgets


def test_get_pods_to_move_system_and_pdb():
    p = _pod(namespace="kube-system", labels={"k8s-app": "dns"})
    q = _pod(labels={"app": "web"})
    q.name = "q"
    by = {id(p): dr.UNDEFINED, id(q): dr.UNDEFINED}
    t = dr.RemainingPdbTracker([])
    assert dr.GetPodsToMove([q, p], lambda x: by[id(x)], t, "kube-system") == ([], (1, dr.KUBE_SYSTEM))
    assert dr.GetPodsToMove([q, p], lambda x: by[id(x)], t, None) == ([q, p], None)
    t = dr.RemainingPdbTracker([dns_pdb(1), PodDisruptionBudget("w", "default", LabelSelector({"app": "web"}), 0)])
    assert dr.GetPodsToMove([p], lambda x: by[id(x)], t, "kube-system") == ([p], None)
    assert dr.GetPodsToMove([p, q], lambda x: by[id(x)], t, "kube-system") == ([], (1, dr.NOT_ENOUGH_PDB))


def test_tracker():
    web = [_pod(labels={"app": "web"}) for _ in range(3)]
    pdbs = [PodDisruptionBudget("a", "default", LabelSelector({"app": "web"}), 2),
            PodDisruptionBudget("nil", "default", None, 5),
            PodDisruptionBudget("all", "default", LabelSelector(), 4),
            PodDisruptionBudget("other-ns", "prod", LabelSelector(), 4),
            PodDisruptionBudget("gt", "default", LabelSelector(match_expressions=[Requirement("tier", "Gt", ["3"])]), 1)]
    t = dr.RemainingPdbTracker(pdbs)
    assert t.MatchingPdbs(web[0]) == [0, 2]
    tiered = _pod(labels={"tier": "7"})
    assert t.MatchingPdbs(tiered) == [2, 4]
    assert t.MatchingPdbs(_pod(labels={"tier": "x7"})) == [2]
    assert t.CanRemovePods(web[:2]) == (True, 0, None)
    assert t.CanRemovePods([web[0]]) == (True, 1, None)
    ok, slack, blocking = t.CanRemovePods(web)
    assert (ok, slack, blocking) == (False, -1, web[2])
    assert t.CanRemovePods([]) == (True, 2 ** 31 - 1, None)
    t.RemovePods(web[:2])
    assert t.remaining == [0, 5, 2, 4, 1]


# ---- the loop on the oracle, hand-worked --------------------------------------------------------------------------------
@pytest.mark.parametrize("persist", [False, True])
def test_shared_pdb(oracle, persist):
    cl = shared_pdb_cluster()
    by = bytes_of_cluster(cl)
    got = loop_plan(cl, ["A", "B"], everywhere(cl), persist, by, [web_pdb(1)])
    assert got["results"][0][:2] == ("remove", "A") and got["results"][0][4] == 0
    assert got["results"][1] == ("blocked", "B", 0, dr.NOT_ENOUGH_PDB)
    assert got["pdb_left"] == [0]
    got = loop_plan(cl, ["A", "B"], everywhere(cl), persist, by, [])
    assert [r[0] for r in got["results"]] == ["remove", "remove"]
    assert got["results"][1][4] == 2 ** 31 - 1


def test_kube_system(oracle):
    cl = kube_system_cluster()
    by = bytes_of_cluster(cl)
    got = loop_plan(cl, ["A"], everywhere(cl), True, by, [], kube_system="kube-system")
    assert got["results"] == [("blocked", "A", 1, dr.KUBE_SYSTEM)]
    got = loop_plan(cl, ["A"], everywhere(cl), True, by, [dns_pdb(1)], kube_system="kube-system")
    assert got["results"] == [("remove", "A", ["dns"], ["a-ds"], 0)] and got["pdb_left"] == [0]
    got = loop_plan(cl, ["A"], everywhere(cl), True, by, [dns_pdb(0)], kube_system="kube-system")
    assert got["results"] == [("blocked", "A", 1, dr.NOT_ENOUGH_PDB)]
    got = loop_plan(cl, ["A"], everywhere(cl), True, by, [], kube_system=None)
    assert got["results"][0][0] == "remove"


def test_pdb_ahead_of_static_block(oracle):
    cl = pdb_before_static_cluster()
    by = bytes_of_cluster(cl)
    got = loop_plan(cl, ["A"], everywhere(cl), False, by, [web_pdb(0)])
    assert got["results"] == [("blocked", "A", 1, dr.NOT_ENOUGH_PDB)]
    got = loop_plan(cl, ["A"], everywhere(cl), False, by, [web_pdb(1)])
    assert got["results"] == [("blocked", "A", 2, dr.NOT_SAFE_TO_EVICT)]


def test_limit_and_atomic(oracle):
    cl = limit_cluster()
    by = bytes_of_cluster(cl)
    cands = ["N0", "N1", "N2", "N3", "N4"]
    got = loop_plan(cl, cands, everywhere(cl), True, by, [], limit=2, atomic=[0, 1, 1, 0, 0])
    assert [r[0] for r in got["results"]] == ["remove"] * 4 + ["not_simulated"]
    got = loop_plan(cl, cands, everywhere(cl), True, by, [], limit=0)
    assert [r[0] for r in got["results"]] == ["not_simulated"] * 5


def test_no_persist_removed_node_is_no_destination(oracle):
    cl = shared_pdb_cluster()
    by = bytes_of_cluster(cl)
    # without the loop's destination deletion C would take A's pod and then C's own pod could move to A
    got = loop_plan(cl, ["A", "C"], {"A": True, "B": False, "C": True}, False, by, [])
    assert got["results"][0][0] == "remove"
    assert got["results"][1] == ("unremovable", "C", "NoPlaceToMovePods")


def test_moved_in_pod_checked_and_counted_again(oracle):
    cl = chain_pdb_cluster()
    by = bytes_of_cluster(cl)
    got = loop_plan(cl, ["A", "B"], everywhere(cl), True, by, [web_pdb(2)])
    assert got["results"][0][:3] == ("remove", "A", ["a1"]) and got["results"][1][:3] == ("remove", "B", ["a1"])
    assert got["pdb_left"] == [0]
    got = loop_plan(cl, ["A", "B"], everywhere(cl), True, by, [web_pdb(1)])
    assert got["results"][1] == ("blocked", "B", 0, dr.NOT_ENOUGH_PDB)


# ---- ABI ----------------------------------------------------------------------------------------------------------------
def test_header_symbol_and_struct():
    assert "cae_plan_removals" in capi.declared_functions()
    names = [n for n, _ in capi.cae_removal_plan._fields_]
    assert names[0] == "abi_version"
    for f in ("n_cand", "cand_node", "dest_ok", "unneeded_limit", "atomic", "n_res", "drain", "hint_node", "sim_class",
              "kube_system_ns", "n_pdb", "pdb_namespace", "pdb_allowed", "pdb_sel_kind", "pdb_req_off", "req_key", "req_op",
              "req_val_off", "req_vals", "num_new_values", "value_is_int", "value_int"):
        assert f in names, f
    assert capi.CONST["CAE_REMOVAL_BLOCKED"] == 3 and capi.CONST["CAE_REMOVAL_NOT_SIMULATED"] == 4
    assert capi.CONST["CAE_BLOCK_KUBE_SYSTEM"] == 16 and capi.CONST["CAE_BLOCK_NOT_ENOUGH_PDB"] == 17
    restype, args = capi.signatures(capi._SRC)["cae_plan_removals"]
    assert len(args) == 11
