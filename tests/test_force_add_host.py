"""Host side of cae_force_add_pods: EncodedObjects.apply_force_add states the same snapshot as a fresh encode() of the
object world with the pods moved onto their NodeInfos (compared through the oracle: reasons, estimates, filter
assignments — not ids; the resident lists, which ids do not hide, are compared entry by entry), the new_index map, emptied
groups are kept, and malformed lists are rejected."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200.encode import encode

from test_node_delta_host import _encoder, _same_results, _world


def _move(cluster, groups, moves):
    """The object world after ForceAddPod of groups[g].pods[i] onto cluster[r] for (g, i, r) in `moves`, in that order.
    Emptied groups stay (with no pods)."""
    gone = set()
    for g, i, r in moves:
        q = groups[g].pods[i].clone()
        q.node_name = cluster[r].node.name
        cluster[r].pods.append(q)
        gone.add((g, i))
    for g, grp in enumerate(groups):
        grp.pods = [p for i, p in enumerate(grp.pods) if (g, i) not in gone]
    return cluster, groups


def _indices(enc0, moves):
    go = enc0.arrays["group_off"]
    return [int(go[g]) + i for g, i, _ in moves], [r for _, _, r in moves]


MOVES = {
    "a few": [(0, 2, 1), (3, 0, 1), (1, 4, 5), (0, 0, 1), (2, 5, 0)],
    "a whole group": [(1, i, 2) for i in range(5)] + [(3, 8, 2)],
    "everything": [(g, i, (g + i) % 6) for g, n in enumerate((7, 5, 6, 9)) for i in range(n)],
}


@pytest.mark.parametrize("name", sorted(MOVES))
def test_apply_force_add_matches_fresh_encode(oracle, name):
    moves = MOVES[name]
    cluster, templates, groups = _world()
    _, enc0 = _encoder(cluster, templates, groups)
    pods, nodes = _indices(enc0, moves)
    after, new_index = enc0.apply_force_add(pods, nodes)
    # the map: moved pods -1, the others numbered in their old order
    assert (new_index[pods] == -1).all() and after.P == enc0.P - len(moves)
    kept = np.flatnonzero(new_index >= 0)
    assert np.array_equal(new_index[kept], np.arange(after.P))
    assert np.array_equal(after.arrays["pend_spec"], enc0.arrays["pend_spec"][kept])
    # groups are kept, emptied ones included
    assert after.E == enc0.E
    sizes = np.diff(enc0.arrays["group_off"]) - np.bincount([g for g, _, _ in moves], minlength=enc0.E)
    assert np.array_equal(np.diff(after.arrays["group_off"]), sizes)
    if name != "a few":
        assert (sizes == 0).any()
    # every row's list is its old list followed by its arrivals in list order, spec ids unchanged
    off0, spec0, off1, spec1 = (x.arrays[k] for x in (enc0, after) for k in ("node_pod_off", "node_pod_spec"))
    for r in range(len(off0) - 1):
        arrivals = [int(enc0.arrays["pend_spec"][p]) for p, n in zip(pods, nodes) if n == r]
        assert list(spec1[off1[r]:off1[r + 1]]) == list(spec0[off0[r]:off0[r + 1]]) + arrivals
    # and the whole snapshot answers like a re-encode of the moved object world
    cluster, groups = _move(cluster, groups, moves)
    _same_results(oracle, after, encode(cluster, templates, groups))


def test_apply_force_add_of_nothing_and_twice(oracle):
    cluster, templates, groups = _world()
    _, enc0 = _encoder(cluster, templates, groups)
    same, idx = enc0.apply_force_add([], [])
    assert np.array_equal(idx, np.arange(enc0.P)) and same.P == enc0.P
    _same_results(oracle, same, enc0)
    first, i1 = enc0.apply_force_add(*_indices(enc0, MOVES["a few"][:3]))
    rest = [(g, i, r) for g, i, r in MOVES["a few"][3:]]
    pods, nodes = _indices(enc0, rest)
    second, _ = first.apply_force_add(i1[pods], nodes)          # the caller's indices follow new_index
    both, _ = enc0.apply_force_add(*_indices(enc0, MOVES["a few"]))
    for k in ("pend_spec", "group_off", "node_pod_off", "node_pod_spec"):
        assert np.array_equal(second.arrays[k], both.arrays[k])


@pytest.mark.parametrize("pods,nodes", [([0, 0], [1, 2]), ([-1], [0]), ([27], [0]), ([0], [6]), ([0], [-1]), ([0, 1], [0])],
                         ids=["twice", "negative pod", "pod past P", "a template row", "negative node", "lengths"])
def test_apply_force_add_rejects(pods, nodes):
    cluster, templates, groups = _world()
    _, enc0 = _encoder(cluster, templates, groups)
    assert enc0.P == 27 and enc0.struct.num_cluster_nodes == 6
    with pytest.raises(ValueError):
        enc0.apply_force_add(pods, nodes)


def test_header_declares_the_call():
    assert "cae_force_add_pods" in capi.declared_functions()
