"""TEST HARNESS for the engine's documented limits on the pod-state plugins (DESIGN.md): at most 8 distinct topology keys,
12 topology counters per dynamic class and 64 distinct host-port sets among pending pods.  The worlds here sit exactly at
those limits, and the `past` variants one step beyond them; `derive` mirrors the host derivation (api.cu plan_static /
plan_dynamic, dyn_kernels.cu's EXIST activity) so a test without the GPU can show that the inputs reach their cases.

Every world is built through the string-world object model from a fixed seed."""
import random

import numpy as np

from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, HostPort, LabelSelector, NodeInfo, PodAffinityTerm,
                                                Requirement, Toleration, TopologySpreadConstraint, makePodEquivalenceGroup)

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"
# the eight keys: hostname; zone; pool; rack (a value per cluster node, one per template); row (cluster nodes only); tmpl
# (templates only, Dc = 0); sparse (a third of the nodes, half the templates); region (template-only values beside shared ones)
KEYS = [HOST, ZONE, "pool", "rack", "row", "tmpl", "sparse", "region"]
NOHOST_KEYS = [ZONE, "pool", "rack", "row", "tmpl", "sparse", "region", "aisle"]
EXTRA_KEY = "extra"
MAX_KEYS, MAX_Q, MAX_PORT_SETS = 8, 12, 64
Q_PTS, Q_AFF, Q_ANTI, Q_EXIST = 0, 1, 2, 3
APPS = ["a", "b", "c", "d", "e"]


def _node(name, labels, cpu=4000, mem=8 << 30, pods=110):
    n = BuildTestNode(name, cpu, mem)
    n.labels = dict(labels)
    n.allocatable["pods"] = n.capacity["pods"] = pods
    return n


def cluster_labels(i, rng, keys):
    lb = {HOST: "c%04d" % i, ZONE: "z%d" % (i % 3), "pool": rng.choice(["p1", "p2"]), "rack": "r%04d" % i,
          "row": "w%d" % (i % 4), "region": rng.choice(["east", "west"]), "aisle": "a%d" % (i % 5)}
    if rng.random() < 1 / 3:
        lb["sparse"] = "s%d" % (i % 2)
    return {k: v for k, v in lb.items() if k in keys or k == HOST}


def template_labels(t, keys):
    lb = {HOST: "t%d" % t, ZONE: "z%d" % (t % 3), "pool": "p%d" % (1 + t % 2), "rack": "tr%d" % t, "tmpl": "T%d" % (t % 2),
          "region": ["east", "mars", "west", "moon"][t % 4], "aisle": "ta%d" % t}
    if t % 2 == 0:
        lb["sparse"] = "s%d" % (t % 4 // 2)
    return {k: v for k, v in lb.items() if k in keys or k == HOST}


def anti_resident(name, app, keys, target):
    """A resident with a required anti-affinity term on each of `keys` against app `target`."""
    p = BuildTestPod(name, 50, 1 << 24)
    p.labels = {"app": app}
    p.owner_uid, p.owner_kind = "rs-" + app, "ReplicaSet"
    p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": target}), k) for k in keys]
    return p


def port_sets():
    """64 host-port lists.  Compact ids 0, 31, 32 and 63 share TCP 7000 (wildcard against specific IPs: every pair of them
    conflicts); every other list is its own ports, with multi-port lists and TCP, UDP and SCTP."""
    out = []
    for i in range(MAX_PORT_SETS):
        proto = ["TCP", "UDP", "SCTP"][i % 3]
        own = [HostPort(8000 + i, proto, ["", "10.0.0.1", "0.0.0.0", "10.0.0.2"][i % 4])]
        if i % 5 == 0:
            own.append(HostPort(9000 + i, ["UDP", "SCTP", "TCP"][i % 3], ""))
        fam = {0: [HostPort(7000, "TCP", "")], 31: [HostPort(7000, "TCP", "10.0.0.1")],
               32: [HostPort(7000, "", "0.0.0.0"), HostPort(7001, "UDP", "10.0.0.9")], 63: [HostPort(7000, "TCP", "10.0.0.1"), HostPort(7002, "SCTP", "")]}
        out.append(fam.get(i, []) + own)
    return out


def _sel(rng, app):
    return LabelSelector({"app": app}) if rng.random() < 0.8 else LabelSelector(match_expressions=[Requirement("app", "In", [app, rng.choice(APPS)])])


def _pts(rng, key, app):
    return TopologySpreadConstraint(rng.randint(1, 3), key, _sel(rng, app), min_domains=rng.choice([None, None, 2, 5]),
                                    when_unsatisfiable=rng.choice(["DoNotSchedule", "DoNotSchedule", "ScheduleAnyway"]),
                                    node_affinity_policy=rng.choice([None, "Honor", "Ignore"]),
                                    node_taints_policy=rng.choice([None, "Honor", "Ignore"]))


# (own PTS, own AFF, own ANTI) per pending class; with the 8 EXIST counters of the resident anti terms:
# 12 = 2 + 1 + 1 + 8, 12 = 4 + 8, 12 with EXIST counters inactive (app d: no term selects it), and 9..11, 8
MIXES = [(2, 1, 1), (4, 0, 0), (2, 2, 0), (1, 0, 0), (1, 1, 1), (0, 0, 3), (0, 0, 0), (2, 0, 1)]


def pending_protos(seed, keys, n=MAX_PORT_SETS, ports=True):
    """n pending pod prototypes: prototype i carries port set i (ids follow first appearance) and counters mix i % 8."""
    rng = random.Random(seed)
    sets = port_sets()
    out = []
    for i in range(n):
        app = "d" if MIXES[i % len(MIXES)] == (2, 2, 0) else rng.choice(APPS)
        p = BuildTestPod("q%02d" % i, rng.choice([20, 50, 100, 250]), rng.choice([1 << 24, 1 << 26, 1 << 28]))
        p.labels = {"app": app}
        p.owner_uid, p.owner_kind = "rs-q%02d" % i, "ReplicaSet"
        np_, na, nn = MIXES[i % len(MIXES)]
        ks = rng.sample(keys, 4)
        p.topology_spread = [_pts(rng, ks[j], rng.choice([app, app, rng.choice(APPS)])) for j in range(np_)]
        p.pod_affinity = [PodAffinityTerm(_sel(rng, rng.choice([app, "ra", "rb"])), rng.choice(keys)) for _ in range(na)]
        p.pod_anti_affinity = [PodAffinityTerm(_sel(rng, rng.choice(APPS)), rng.choice(keys)) for _ in range(nn)]
        if ports:
            p.host_ports = list(sets[i])
        out.append(p)
    return out


def with_extra(protos, what):
    """One more prototype, last: the 9th key (a spread key no other pod uses), the 13th counter (5 own counters) or the
    65th host-port set."""
    p = BuildTestPod("q-extra", 30, 1 << 24)
    p.labels = {"app": "e"}
    p.owner_uid, p.owner_kind = "rs-extra", "ReplicaSet"
    if what == "key":
        p.topology_spread = [TopologySpreadConstraint(1, EXTRA_KEY, LabelSelector({"app": "e"}))]
    elif what == "counter":
        p.topology_spread = [TopologySpreadConstraint(1, k, LabelSelector({"app": "e"})) for k in (ZONE, "pool", "rack")]
        p.pod_affinity = [PodAffinityTerm(LabelSelector({"app": "ra"}), ZONE)]
        p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": "e"}), "row")]
    else:
        p.host_ports = [HostPort(6500, "UDP", "10.1.1.1")]
    return protos + [p]


def world(seed, nodes=40, templates=5, host=True, protos=None, group_pods=5):
    """(cluster, templates, groups, caps) at the limits: 8 keys (with or without the hostname key), every pending class with
    the 8 EXIST counters of the residents' anti terms, 64 port sets among the pending groups."""
    keys = KEYS if host else NOHOST_KEYS
    rng = random.Random(seed)
    cluster = []
    for i in range(nodes):
        ni = NodeInfo(_node("c%04d" % i, cluster_labels(i, rng, keys), cpu=rng.choice([2000, 4000, 8000]),
                            pods=rng.choice([8, 30, 110])), [])
        cluster.append(ni)
    # residents: anti terms on the first four keys against app a on two nodes of zone z0, on the last four against app b
    # elsewhere; the DaemonSet pod of every other template holds terms on all eight keys against app c.  ra-0 is the first
    # pod spec with terms, so its term order is the key order: the hostname key lands in slot 3, not 0
    for j, i in enumerate([0, 3]):
        if i < nodes:
            cluster[i].pods.append(anti_resident("ra-%d" % j, "ra", keys[1:4] + keys[:1], "a"))
    for j in range(min(nodes, 6)):
        i = (5 + 7 * j) % nodes
        cluster[i].pods.append(anti_resident("rb-%d" % j, "rb", keys[4:], "b"))
    for i in range(nodes):
        if rng.random() < 0.5:
            p = BuildTestPod("w-%d" % i, 100, 1 << 26)
            p.labels = {"app": rng.choice(APPS)}
            p.owner_uid, p.owner_kind = "rs-w", "ReplicaSet"
            cluster[i].pods.append(p)
    ds = anti_resident("ds", "dsa", keys, "c")
    ds.owner_uid, ds.owner_kind = "ds", "DaemonSet"
    ds.tolerations = [Toleration("", "Exists", "", "")]
    tmpl = [NodeInfo(_node("t%d" % t, template_labels(t, keys), cpu=[2000, 4000, 8000][t % 3], pods=[30, 110][t % 2]),
                     [ds] if t % 2 == 0 else []) for t in range(templates)]
    protos = pending_protos(seed, keys) if protos is None else protos
    groups = [makePodEquivalenceGroup(p, 1 + (i * 7 + seed) % group_pods) for i, p in enumerate(protos)]
    return cluster, tmpl, groups


def removal_world(seed, nodes=40, host=True, protos=None):
    """The same cluster with the pending prototypes as residents (one bound pod each, set i on node i % nodes), so that the
    pods a removal batch moves reach the limits; six roomy empty nodes last."""
    cluster, _, _ = world(seed, nodes, 0, host)
    rng = random.Random(seed ^ 0xE7)
    cluster += [NodeInfo(_node("c%04d" % (nodes + i), cluster_labels(nodes + i, rng, KEYS if host else NOHOST_KEYS), cpu=64000, pods=250), [])
                for i in range(6)]
    keys = KEYS if host else NOHOST_KEYS
    protos = pending_protos(seed, keys) if protos is None else protos
    for i, p in enumerate(protos):
        q = p.clone()
        q.name = "m%02d" % i
        cluster[i % nodes].pods.append(q)
    return cluster


# ---- the derivation mirror --------------------------------------------------------------------------------------------------
def _labels_of(a, ls):
    return {int(a["ls_key"][j]): int(a["ls_val"][j]) for j in range(a["ls_off"][ls], a["ls_off"][ls + 1])}


def derive(enc, exist_active=None):
    """What plan_static / plan_dynamic derive from `enc`: the topology keys (in order), Dc and D per key, whether each is the
    hostname key, the counter kinds of each dynamic class, and the compact id of every pending port list.
    exist_active(spec, key): the EXIST activity rule, when the caller can judge it (see `exist_rule`)."""
    a, s = enc.arrays, enc.struct
    S, N, T = s.num_podspecs, s.num_cluster_nodes, s.num_templates
    pend = np.zeros(S, bool)
    pend[np.asarray(a["pend_spec"], np.int64)] = True
    used = pend.copy()
    used[np.asarray(a["node_pod_spec"][:a["node_pod_off"][N + T]], np.int64)] = True
    rng_ = lambda off, l: range(int(a[off][l]), int(a[off][l + 1]))
    keys, exist = [], []
    for sp in range(S):
        if not used[sp]:
            continue
        for t in rng_("aff_off", a["ps_anti_list"][sp]):
            k = int(a["aterm_key"][t])
            keys += [k] if k not in keys else []
            exist += [k] if k not in exist else []
        if pend[sp]:
            for c in rng_("pts_off", a["ps_pts_list"][sp]):
                keys += [int(a["pts_key"][c])] if int(a["pts_key"][c]) not in keys else []
            for t in rng_("aff_off", a["ps_aff_list"][sp]):
                keys += [int(a["aterm_key"][t])] if int(a["aterm_key"][t]) not in keys else []
    rows = [_labels_of(a, int(a["node_labelset"][r])) for r in range(N + T)]
    dc, dall = [], []
    for k in keys:
        cv = {r[k] for r in rows[:N] if k in r}
        tv = {r[k] for r in rows[N:] if k in r} - cv
        dc.append(len(cv))
        dall.append(len(cv) + len(tv))
    classes = {}
    for sp in range(S):
        if not pend[sp]:
            continue
        pl, fl, al = int(a["ps_pts_list"][sp]), int(a["ps_aff_list"][sp]), int(a["ps_anti_list"][sp])
        kinds = [Q_PTS] * len(rng_("pts_off", pl)) + [Q_AFF] * len(rng_("aff_off", fl)) + [Q_ANTI] * len(rng_("aff_off", al))
        if not kinds and not exist:
            continue
        q = [(kd, None) for kd in kinds] + [(Q_EXIST, k) for k in exist]
        active = [True] * len(kinds) + [exist_active(sp, k) if exist_active else True for k in exist]
        classes[sp] = dict(kinds=[kd for kd, _ in q], active=active)
    pc, npc = {}, 0
    for sp in range(S):
        p = int(a["ps_port_list"][sp])
        if pend[sp] and a["port_off"][p + 1] > a["port_off"][p] and p not in pc:
            pc[p] = npc
            npc += 1
    return dict(keys=keys, K=len(keys), Dc=dc, D=dall, is_host=[k == s.hostname_key for k in keys], classes=classes,
                port_id=pc, n_port_sets=npc, hostname_key=s.hostname_key)


def exist_rule(cluster, templates, pending):
    """The EXIST activity of dyn_qmeta_kernel on the objects: counter (class of pod p, key k) is active when some pod in the
    snapshot has an anti term on k whose selector matches p (every term here is in the pod's own namespace, "default")."""
    terms = [t for ni in list(cluster) + list(templates) for q in ni.pods for t in q.pod_anti_affinity]
    terms += [t for q in pending for t in q.pod_anti_affinity]

    def match(sel, labels):
        if sel is None:
            return False
        if any(labels.get(k) != v for k, v in sel.match_labels.items()):
            return False
        for r in sel.match_expressions:
            assert r.operator == "In"
            if labels.get(r.key) not in r.values:
                return False
        return True
    return lambda pod, key: any(t.topology_key == key and match(t.label_selector, pod.labels) for t in terms)


def port_conflict(x, y):
    """HostPortInfo.CheckConflict of two lists."""
    w = lambda ip: ip in ("", "0.0.0.0")
    pr = lambda p: p.protocol or "TCP"
    return any(a.host_port == b.host_port and pr(a) == pr(b) and (w(a.host_ip) or w(b.host_ip) or a.host_ip == b.host_ip)
               for a in x for b in y)
