"""Deterministic synthetic snapshots for the BASELINE.json configs (SURVEY.md §8d).

Generator = splitmix64 streams, seed ``0xCA5CA1E0 + config_index``.  Tables are built at the
integer level (``TableBuilder``) — there are no strings to intern in a synthetic snapshot, the ids
stand for them (key 0 = kubernetes.io/hostname, 1 = zone, 2 = pool, 3 = instance-type, 4 = app,
5 = tier, 6.. = taint keys).

Distributions: pods in E = P/100 equivalence groups with Zipf(1.1) replica counts; cpu in
{50,100,250,500,1000,2000,4000} m (20/25/20/15/10/7/3 %), mem = cpu x {1,2,4,8} MiB, 10 % of the
groups ask for nvidia.com/gpu in {1,2,4,8}; 32 namespaces; labels app=<group>, tier in 4.
Templates: vCPU in {2,..,96}, allocatable = capacity - reserved, 110 pods, 2 DaemonSet pods, 15 % GPU
templates, labels hostname/zone(16)/pool(8)/instance-type.  C2+: 16 taints (8 keys x 2 values), 0-2
NoSchedule taints per template, tolerations per group (10 % wildcard Exists), 20 % of the groups
carry a 1-2 key nodeSelector.  C3+: 30 % of the groups have one DoNotSchedule spread constraint and
the snapshot holds `cluster_nodes` nodes x 30 resident pods.  C4+: 10 % self anti-affinity on
hostname, 5 % required affinity to another group on zone.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from .encode import EncodedObjects, TableBuilder

MiB = 1 << 20
GiB = 1 << 30
K_HOST, K_ZONE, K_POOL, K_ITYPE, K_APP, K_TIER, K_TAINT0 = 0, 1, 2, 3, 4, 5, 6
RES_GPU = 3


@dataclass
class Config:
    index: int
    pods: int
    templates: int
    taints: bool = False
    spread: bool = False
    affinity: bool = False
    cluster_nodes: int = 0
    pods_per_node: int = 30
    name: str = ""


CONFIGS = {
    1: Config(1, 1_000, 50, name="C1 1000 pods x 50 templates, NodeResourcesFit only"),
    2: Config(2, 100_000, 1_000, taints=True, name="C2 100k pods x 1000 templates, resources + taints/tolerations"),
    3: Config(3, 100_000, 5_000, taints=True, spread=True, cluster_nodes=2000,
              name="C3 100k pods x 5000 templates, + PodTopologySpread"),
    4: Config(4, 500_000, 5_000, taints=True, spread=True, affinity=True, cluster_nodes=2000,
              name="C4 500k pods x 5000 templates, + InterPodAffinity"),
    5: Config(5, 1_000_000, 10_000, taints=True, spread=True, affinity=True, cluster_nodes=2000,
              name="C5 1M pods x 10000 templates, full predicate set"),
}


class SplitMix64:
    """Vectorised splitmix64 stream."""

    def __init__(self, seed: int) -> None:
        self.state = np.uint64(seed & 0xFFFFFFFFFFFFFFFF)

    def next(self, n: int) -> np.ndarray:
        with np.errstate(over="ignore"):
            idx = np.arange(1, n + 1, dtype=np.uint64)
            z = self.state + idx * np.uint64(0x9E3779B97F4A7C15)
            self.state = z[-1] if n else self.state
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            return z ^ (z >> np.uint64(31))

    def uniform(self, n: int) -> np.ndarray:
        return (self.next(n) >> np.uint64(11)).astype(np.float64) / float(1 << 53)

    def randint(self, n: int, hi: int) -> np.ndarray:
        return (self.next(n) % np.uint64(hi)).astype(np.int64)

    def choice(self, n: int, values, weights) -> np.ndarray:
        cdf = np.cumsum(np.asarray(weights, dtype=np.float64))
        cdf /= cdf[-1]
        return np.asarray(values)[np.searchsorted(cdf, self.uniform(n), side="right").clip(0, len(values) - 1)]


RESERVED = {2: 70, 4: 80, 8: 90, 16: 110, 32: 150, 64: 230, 96: 310}
# the resource dims of generate(dims=...) (CAE_MAX_RES of them), the unit of their request values, the requests of the
# DaemonSet pods every node holds, and the default number of distinct request values per active dim
DIMS = ("cpu", "memory", "ephemeral-storage", "example.com/r0", "example.com/r1", "example.com/r2", "example.com/r3",
        "example.com/r4")
DIM_UNIT = (50, 64 * MiB, GiB, 1, 1, 1, 1, 1)
DS_REQ = [100, 200 * MiB, 0, 0, 0, 0, 0, 0]
DIM_CARD = 3


def generate(config: int = 2, pods: Optional[int] = None, templates: Optional[int] = None,
             cluster_nodes: Optional[int] = None, taints: Optional[bool] = None,
             spread: Optional[bool] = None, affinity: Optional[bool] = None,
             seed: Optional[int] = None, dims=None) -> EncodedObjects:
    """dims = None: the requests of the module docstring (cpu, memory, nvidia.com/gpu as dim 3).  Otherwise the dims the
    pending pods request, out of the 8 of ``DIMS``: a sequence of dim indices (DIM_CARD distinct values each), or a mapping
    dim -> number of distinct request values.  Then a second stream draws every request and the allocatable of the active
    dims (the first draws are unchanged), and there are at least as many groups as the largest count."""
    cfg = CONFIGS[config]
    P = cfg.pods if pods is None else pods
    T = cfg.templates if templates is None else templates
    NC = cfg.cluster_nodes if cluster_nodes is None else cluster_nodes
    use_taints = cfg.taints if taints is None else taints
    use_spread = cfg.spread if spread is None else spread
    use_aff = cfg.affinity if affinity is None else affinity
    rng = SplitMix64((0xCA5CA1E0 + cfg.index) if seed is None else seed)
    card = None if dims is None else (dict(dims) if isinstance(dims, dict) else {int(a): DIM_CARD for a in dims})
    b = TableBuilder(num_res=4 if card is None else len(DIMS))
    b.hostname_key = K_HOST
    b.unschedulable_taint_key = -1
    for ns in range(32):
        b.declare_namespace(ns, 0, False)

    # value id spaces (all label values are opaque ids; none parses as an int)
    V_ZONE0, V_POOL0, V_ITYPE0, V_TIER0, V_TAINTV0 = 0, 16, 24, 48, 52
    V_APP0 = 64
    E = max(1, P // 100)
    if card:
        E = max(E, max(card.values()))
    V_HOST0 = V_APP0 + E
    b.declare_value(V_HOST0 + T + NC + 1, None)

    # ---- groups ------------------------------------------------------------------------------
    w = 1.0 / np.arange(1, E + 1, dtype=np.float64) ** 1.1
    counts = np.maximum(1, np.floor(P * w / w.sum()).astype(np.int64))
    diff = P - int(counts.sum())
    i = 0
    while diff != 0:  # hand the rounding remainder to the head groups
        step = 1 if diff > 0 else -1
        if counts[i % E] + step >= 1:
            counts[i % E] += step
            diff -= step
        i += 1
    perm = rng.next(E).argsort()  # which group is big is random, not tied to its id
    counts = counts[perm]
    cpu = rng.choice(E, [50, 100, 250, 500, 1000, 2000, 4000], [20, 25, 20, 15, 10, 7, 3]).astype(np.int64)
    mem = cpu * rng.choice(E, [1, 2, 4, 8], [1, 1, 1, 1]).astype(np.int64) * MiB
    gpu = np.where(rng.uniform(E) < 0.10, rng.choice(E, [1, 2, 4, 8], [1, 1, 1, 1]), 0).astype(np.int64)
    ns_of = rng.randint(E, 32)
    tier = rng.randint(E, 4)
    u_tol = rng.uniform(E)
    tol_bits = rng.next(E)
    u_sel = rng.uniform(E)
    sel_pool = rng.randint(E, 8)
    sel_zone = rng.randint(E, 16)
    u_pts = rng.uniform(E)
    pts_kind = rng.randint(E, 2)
    pts_skew_h = rng.choice(E, [1, 2], [1, 1])
    pts_skew_z = rng.choice(E, [1, 2, 5], [1, 1, 1])
    pts_mind = rng.choice(E, [1, 3], [1, 1])
    u_aff = rng.uniform(E)
    aff_other = rng.randint(E, max(E, 1))
    if card is not None:   # request of group g in dim a: DIM_UNIT[a] x (1 + level), every level of a dim used once E allows
        rd = SplitMix64(((0xCA5CA1E0 + cfg.index) if seed is None else seed) ^ 0xD1B54A32D192ED03)
        dim_req = np.zeros((E, len(DIMS)), np.int64)
        for a, d in sorted(card.items()):
            lvl = rd.randint(E, d)
            n = min(E, d)
            lvl[:n] = rd.next(n).argsort()
            dim_req[:, a] = DIM_UNIT[a] * (1 + lvl)

    taint_ids = [(K_TAINT0 + k, V_TAINTV0 + v) for k in range(8) for v in range(2)]
    group_spec: List[int] = []
    for g in range(E):
        ls = b.labelset([(K_APP, V_APP0 + g), (K_TIER, V_TIER0 + int(tier[g]))])
        tols = []
        if use_taints:
            if u_tol[g] < 0.10:
                tols.append((-1, 1, -1, 0))  # wildcard: empty key + Exists tolerates everything
            else:
                for i, (k, v) in enumerate(taint_ids):
                    if (int(tol_bits[g]) >> i) & 1:
                        tols.append((k, 0, v, 1))  # key=value:NoSchedule
        naff = -1
        if use_taints and u_sel[g] < 0.20:
            reqs = [(K_POOL, 0, (V_POOL0 + int(sel_pool[g]),))]
            if u_sel[g] < 0.07:
                reqs.append((K_ZONE, 0, (V_ZONE0 + int(sel_zone[g]),)))
            naff = b.node_affinity(b.selector(reqs), False, [])
        pts = 0
        anti = 0
        aff = 0
        own_sel = b.selector([(K_APP, 0, (V_APP0 + g,))]) if (use_spread or use_aff) else 0
        if use_spread and u_pts[g] < 0.30:
            if pts_kind[g] == 0:
                pts = b.pts_list([(int(pts_skew_h[g]), K_HOST, own_sel, int(pts_mind[g]), 1, 0)])
            else:
                pts = b.pts_list([(int(pts_skew_z[g]), K_ZONE, own_sel, int(pts_mind[g]), 1, 0)])
        if use_aff:
            nothing = b.nothing_selector()
            if u_aff[g] < 0.10:
                anti = b.affinity_list([(own_sel, K_HOST, (int(ns_of[g]),), nothing)])
            elif u_aff[g] < 0.15:
                og = int(aff_other[g])
                osel = b.selector([(K_APP, 0, (V_APP0 + og,))])
                aff = b.affinity_list([(osel, K_ZONE, (int(ns_of[og]),), nothing)])
        req = [int(cpu[g]), int(mem[g]), 0, int(gpu[g])] if card is None else dim_req[g].tolist()
        group_spec.append(b.podspec(int(ns_of[g]), ls, req, b.toleration_list(tols), naff, -1, 0, pts, aff, anti))

    # ---- DaemonSet pods (kube-system = namespace 31, no labels anyone selects) --------------------
    ds_ls = b.labelset([(K_TIER, V_TIER0 + 3)])
    ds_tol = b.toleration_list([(-1, 1, -1, 0)])
    ds_spec = [b.podspec(31, ds_ls, DS_REQ[:4], ds_tol), b.podspec(31, ds_ls, DS_REQ[:4], ds_tol)]

    # ---- nodes ----------------------------------------------------------------------------------
    def node_shape(n: int, r: SplitMix64):
        vcpu = r.choice(n, [2, 4, 8, 16, 32, 64, 96], [1] * 7).astype(np.int64)
        mem_per = r.choice(n, [2, 4, 8], [1, 1, 1]).astype(np.int64)
        is_gpu = r.uniform(n) < 0.15
        ngpu = np.where(is_gpu, r.choice(n, [1, 4, 8], [1, 1, 1]), 0).astype(np.int64)
        return vcpu, mem_per, ngpu, r.randint(n, 16), r.randint(n, 8), r.uniform(n), r.next(n)

    def add_nodes(n: int, first_host: int, is_template: bool, resident: Optional[np.ndarray]):
        vcpu, mem_per, ngpu, zone, pool, u_t, tbits = node_shape(n, rng)
        if card is not None:   # allocatable of an active dim: 1/2 .. 2x its largest request, on top of the DaemonSet pods
            dim_alloc = np.zeros((n, len(DIMS)), np.int64)
            for a, d in sorted(card.items()):
                dim_alloc[:, a] = DS_REQ[a] + DIM_UNIT[a] * (d // 2 + rd.randint(n, 2 * d - d // 2 + 1))
        for i in range(n):
            v = int(vcpu[i])
            cap_cpu = v * 1000
            cap_mem = v * int(mem_per[i]) * GiB
            alloc_cpu = cap_cpu - RESERVED[v] - (i % 7)  # a few milli-cores of jitter: distinct allocatable
            alloc_mem = cap_mem - cap_mem // 20 - (i % 11) * MiB
            ls = b.labelset([(K_HOST, V_HOST0 + first_host + i), (K_ZONE, V_ZONE0 + int(zone[i])),
                             (K_POOL, V_POOL0 + int(pool[i])), (K_ITYPE, V_ITYPE0 + (v % 24))])
            tl = []
            if use_taints:
                nt = 0 if u_t[i] < 0.5 else (1 if u_t[i] < 0.85 else 2)
                for j in range(nt):
                    k, val = taint_ids[(int(tbits[i]) >> (8 * j)) % 16]
                    tl.append((k, val, 1))
            pods = list(ds_spec)
            if resident is not None:
                pods += [group_spec[int(x)] for x in resident[i]]
            alloc = [alloc_cpu, alloc_mem, 0, int(ngpu[i])]
            if card is not None:
                alloc = [alloc_cpu, alloc_mem] + [0] * (len(DIMS) - 2)
                for a in card:
                    alloc[a] = int(dim_alloc[i, a])
            args = dict(name=first_host + i, labelset=ls, taint_list=b.taint_list(tl), unschedulable=False,
                        alloc=alloc, allowed_pods=110, cap_cpu=cap_cpu,
                        cap_mem=cap_mem, has_alloc_cpu=True, has_alloc_mem=True, pod_specs=pods)
            (b.template if is_template else b.cluster_node)(**args)

    if NC:
        resident = rng.randint(NC * cfg.pods_per_node, E).reshape(NC, cfg.pods_per_node)
        add_nodes(NC, 0, False, resident)
    add_nodes(T, NC, True, None)

    # ---- pending pods, group-major ------------------------------------------------------------------
    for g in range(E):
        b.group(np.full(int(counts[g]), group_spec[g], np.int32))
    return b.finish()


def node_churn(enc: EncodedObjects, seed: int, n_dirty: int, bind: float = 0.3, evict: float = 0.3, move: float = 0.15,
               cordon: float = 0.15, taint: float = 0.3, alloc: float = 0.25, relabel: float = 0.25):
    """A deterministic random tick of cluster-node churn against a snapshot of ``generate`` (its key / value layout):
    ``n_dirty`` distinct cluster rows, each changed with the given probabilities —
      bind     pods of pending groups are bound to the node (every group keeps at least one pending pod, so the pending
               delta still applies);
      evict    resident pods finish;   move  resident pods move to another dirty node;
      cordon   the node is cordoned / uncordoned;
      taint    the node switches to an existing taint list or to a new one (some with a new value);
      alloc    allocatable and allowed pods change, sometimes below what the residents request (negative free);
      relabel  the node switches to a label set with the same hostname and zone but another pool (sometimes a new value)
               and instance type, which nodeSelectors read.
    Returns (delta, pending): the NodeDelta and ``enc`` with the bound pods removed from the pending rows.
    ``pending.apply_node_delta(delta)`` is the snapshot after the tick."""
    from .encode import NodeDelta
    a, s = enc.arrays, enc.struct
    N = s.num_cluster_nodes
    rng = SplitMix64(0x5EED0000 + seed)
    n_dirty = min(n_dirty, N)
    rows = np.sort(rng.next(N).argsort()[:n_dirty]) if n_dirty else np.zeros(0, np.int64)
    off, spec = a["node_pod_off"], a["node_pod_spec"]
    lists = [list(spec[off[r]:off[r + 1]]) for r in rows]
    go = a["group_off"]
    left = np.diff(go).astype(np.int64)            # pending pods per group after the binds
    gspec = np.where(left > 0, a["pend_spec"][np.minimum(go[:-1], max(len(a["pend_spec"]) - 1, 0))], -1) if len(go) > 1 else []
    nv, nl, nt = s.num_values, s.num_labelsets, s.num_taint_lists
    new_vals: List[int] = []
    new_ls: dict = {}
    new_tl: dict = {}

    def new_value() -> int:
        new_vals.append(len(new_vals))
        return nv + len(new_vals) - 1

    def labels_of(ls: int) -> dict:
        return {int(k): int(v) for k, v in zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]],
                                               a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]])}

    u = rng.uniform(8 * max(n_dirty, 1)).reshape(-1, 8)
    r8 = rng.next(8 * max(n_dirty, 1)).reshape(-1, 8)
    lsets, tlists, unsched, allocs, allowed = [], [], [], [], []
    for i, r in enumerate(rows):
        ui, ri = u[i], [int(x) for x in r8[i]]
        pods = lists[i]
        if ui[0] < evict and pods:
            for _ in range(1 + ri[0] % 3):
                if pods:
                    pods.pop(ri[1] % len(pods))
        if ui[1] < move and pods and n_dirty > 1:
            j = (i + 1 + ri[2] % (n_dirty - 1)) % n_dirty
            lists[j].append(pods.pop(ri[3] % len(pods)))
        if ui[2] < bind and len(left):
            for k in range(1 + ri[4] % 4):
                g = (ri[5] + 7919 * k) % len(left)
                if left[g] >= 2:
                    left[g] -= 1
                    pods.append(int(gspec[g]))
        unsched.append(int(a["node_unschedulable"][r]) ^ int(ui[3] < cordon))
        tl = int(a["node_taint_list"][r])
        if ui[4] < taint:
            if ri[6] % 3 == 0:   # a new list: one or two NoSchedule / NoExecute taints, sometimes on a new value
                key = (K_TAINT0 + ri[6] % 8, new_value() if ri[7] % 4 == 0 else 52 + (ri[6] >> 3) % 2, 1 + 2 * ((ri[6] >> 5) % 2))
                ent = (key,) if (ri[6] >> 7) % 2 else (key, (K_TAINT0 + (ri[6] >> 9) % 8, 52, 1))
                ent = tuple(sorted(set(ent)))
                tl = new_tl.setdefault(ent, nt + len(new_tl))
            else:
                tl = ri[6] % nt
        tlists.append(tl)
        al = a["node_alloc"][r].copy()
        ap = int(a["node_allowed_pods"][r])
        if ui[5] < alloc:
            al[0] = max(1, int(al[0] * (0.5 + ui[6])))
            al[1] = max(1, int(al[1] * (0.5 + ui[7])))
            ap = int(ri[0] % 121)
            if ri[1] % 5 == 0:
                al[0] = 1           # residents request more than the node has: negative free
        allocs.append(al)
        allowed.append(ap)
        ls = int(a["node_labelset"][r])
        if ui[6] < relabel:
            lab = labels_of(ls)
            if K_POOL in lab:
                lab[K_POOL] = new_value() if ri[2] % 10 == 0 else 16 + ri[2] % 8
            if K_ITYPE in lab:
                lab[K_ITYPE] = 24 + ri[3] % 24
            key = tuple(sorted(lab.items()))
            ls = new_ls.setdefault(key, nl + len(new_ls))
        lsets.append(ls)
    # about one dirty row in four ends at or past its pod limit (pod slots 0 .. -3): a kubelet whose max-pods is lowered
    # keeps the pods it runs
    for i, p in enumerate(lists):
        if int(r8[i][7]) % 8 < 2:
            allowed[i] = max(0, len(p) - (int(r8[i][7]) >> 3) % 4)
    ls_items = sorted(new_ls.items(), key=lambda kv: kv[1])
    tl_items = sorted(new_tl.items(), key=lambda kv: kv[1])
    ls_off, tl_off = [0], [0]
    for k, _ in ls_items:
        ls_off.append(ls_off[-1] + len(k))
    for k, _ in tl_items:
        tl_off.append(tl_off[-1] + len(k))
    pod_off = [0]
    for p in lists:
        pod_off.append(pod_off[-1] + len(p))
    delta = NodeDelta(
        value_is_int=[0] * len(new_vals), value_int=[0] * len(new_vals),
        ls_off=ls_off, ls_key=[kk for k, _ in ls_items for kk, _v in k], ls_val=[v for k, _ in ls_items for _k, v in k],
        taint_off=tl_off, taint_key=[e[0] for k, _ in tl_items for e in k], taint_val=[e[1] for k, _ in tl_items for e in k],
        taint_effect=[e[2] for k, _ in tl_items for e in k],
        row=rows, labelset=lsets, taint_list=tlists, unschedulable=unsched,
        alloc=np.asarray(allocs, np.int64).reshape(len(rows), -1), allowed_pods=allowed, pod_off=pod_off,
        pod_spec=[x for p in lists for x in p])
    keep = np.concatenate([np.arange(go[g], go[g] + left[g]) for g in range(len(left))]) if len(left) else np.zeros(0, np.int64)
    new_go = np.concatenate([[0], np.cumsum(left)]).astype(np.int32)
    pending = enc.with_pending(a["pend_spec"][keep.astype(np.int64)], new_go)
    return delta, pending


def node_scale(enc: EncodedObjects, seed: int, n_remove: int, n_add: int, n_dirty: int = 0):
    """A deterministic random tick that changes the cluster-node list of a snapshot of ``generate``: ``n_remove`` random
    cluster rows leave, ``n_add`` nodes shaped like the generator's cluster nodes join, and ``n_dirty`` other rows change
    as in ``node_churn`` (same seed).  Every added node has a new hostname value; about one in four has a new zone value
    (a domain appears); when ``n_remove`` allows, the removals include every node of the smallest zone (a domain
    disappears).  Residents of the added nodes are drawn from the specs resident at the load; about one added node in four
    allows no more pods than it holds.
    Returns (churn, pending): the NodeChurn and ``enc`` with the pods bound by the dirty rows removed from the pending rows.
    ``pending.apply_node_churn(churn)`` is the snapshot after the tick."""
    from .encode import NodeChurn, NodeDelta
    a, s = enc.arrays, enc.struct
    N = s.num_cluster_nodes
    delta, pending = node_churn(enc, seed, n_dirty) if n_dirty else (None, enc)
    dirty = set(int(r) for r in delta.arrays["row"]) if delta is not None else set()
    rng = SplitMix64(0x5CA1E000 + seed)
    # removals: the smallest zone first (when it fits), then random clean rows
    zone = np.full(N, -1, np.int64)
    for r in range(N):
        ls = int(a["node_labelset"][r])
        for i in range(a["ls_off"][ls], a["ls_off"][ls + 1]):
            if a["ls_key"][i] == K_ZONE:
                zone[r] = a["ls_val"][i]
    clean = [r for r in range(N) if r not in dirty]
    n_remove = min(n_remove, len(clean))
    removed: List[int] = []
    zones, counts = np.unique(zone[zone >= 0], return_counts=True)
    if len(zones):
        z = int(zones[int(np.argmin(counts))])
        members = [r for r in range(N) if zone[r] == z]
        if members and all(r not in dirty for r in members) and len(members) <= n_remove:
            removed = members
    rest = [r for r in clean if r not in set(removed)]
    order = rng.next(len(rest)).argsort() if rest else np.zeros(0, np.int64)
    removed = sorted(removed + [rest[int(i)] for i in order[:n_remove - len(removed)]])
    # dictionary tails: those of the dirty rows, then new hostname / zone values and the added nodes' label sets
    nv0 = s.num_values + (delta.struct.num_new_values if delta is not None else 0)
    nl0 = s.num_labelsets + (delta.struct.num_new_labelsets if delta is not None else 0)
    nt = s.num_taint_lists + (delta.struct.num_new_taint_lists if delta is not None else 0)
    new_zone = nv0 + n_add          # one new zone value shared by the nodes that take it
    vcpu = rng.choice(max(n_add, 1), [2, 4, 8, 16, 32, 64, 96], [1] * 7).astype(np.int64)
    mem_per = rng.choice(max(n_add, 1), [2, 4, 8], [1, 1, 1]).astype(np.int64)
    ngpu = np.where(rng.uniform(max(n_add, 1)) < 0.15, rng.choice(max(n_add, 1), [1, 4, 8], [1, 1, 1]), 0).astype(np.int64)
    u = rng.uniform(max(n_add, 1))
    zr, pr, tr, nres = (rng.randint(max(n_add, 1), h) for h in (16, 8, max(nt, 1), 31))
    resident_pool = a["node_pod_spec"]
    name0 = int(a["node_name"].max()) + 1 if len(a["node_name"]) else 0
    ls_items, names, tls, allocs, allowed, pod_off, pod_spec = [], [], [], [], [], [0], []
    for j in range(n_add):
        v = int(vcpu[j])
        z = new_zone if u[j] < 0.25 else int(zr[j])
        ls_items.append(((K_HOST, nv0 + j), (K_ZONE, z), (K_POOL, 16 + int(pr[j])), (K_ITYPE, 24 + v % 24)))
        names.append(name0 + j)
        tls.append(int(tr[j]) if nt else 0)
        cap_mem = v * int(mem_per[j]) * GiB
        allocs.append([v * 1000 - RESERVED[v], cap_mem - cap_mem // 20, 0, int(ngpu[j])])
        k = int(nres[j]) if len(resident_pool) else 0
        pods = [int(resident_pool[i]) for i in rng.randint(k, len(resident_pool))] if k else []
        pod_spec.extend(pods)
        pod_off.append(len(pod_spec))
        allowed.append(110)
    # about one added node in four joins at or past its pod limit (pod slots 0 .. -3), as one whose max-pods is set below
    # what it already runs
    under = rng.randint(max(n_add, 1), 16)
    for j in range(n_add):
        if under[j] < 4:
            allowed[j] = max(0, (pod_off[j + 1] - pod_off[j]) - int(under[j]))
    n_new_vals = n_add + (1 if n_add else 0)
    ls_off = list(delta.arrays["ls_off"]) if delta is not None else [0]
    for it in ls_items:
        ls_off.append(ls_off[-1] + len(it))
    changed_arrays = dict(delta.arrays) if delta is not None else {}
    changed_arrays.update(
        value_is_int=np.concatenate([changed_arrays.get("value_is_int", np.zeros(0, np.uint8)), np.zeros(n_new_vals, np.uint8)]),
        value_int=np.concatenate([changed_arrays.get("value_int", np.zeros(0, np.int64)), np.zeros(n_new_vals, np.int64)]),
        ls_off=ls_off,
        ls_key=np.concatenate([changed_arrays.get("ls_key", np.zeros(0, np.int32)), [k for it in ls_items for k, _ in it]]),
        ls_val=np.concatenate([changed_arrays.get("ls_val", np.zeros(0, np.int32)), [v for it in ls_items for _, v in it]]))
    changed = NodeDelta(**changed_arrays)
    alloc = np.zeros((n_add, len(a["node_alloc"][0]) if len(a["node_alloc"]) else 8), np.int64)
    if n_add:
        alloc[:, :4] = np.asarray(allocs, np.int64)
    churn = NodeChurn(changed, removed=removed, name=names, labelset=[nl0 + j for j in range(n_add)], taint_list=tls,
                      unschedulable=np.zeros(n_add, np.uint8), alloc=alloc, allowed_pods=allowed, pod_off=pod_off,
                      pod_spec=pod_spec)
    return churn, pending


def _template_rows(enc: EncodedObjects, ts) -> dict:
    """The cae_template_delta row columns of templates ``ts`` of ``enc`` as they are."""
    a, N = enc.arrays, enc.struct.num_cluster_nodes
    rows = [N + int(t) for t in ts]
    off, spec = a["node_pod_off"], a["node_pod_spec"]
    out = {nm: [a["node_" + nm][r] for r in rows] for nm in ("name", "labelset", "taint_list", "unschedulable", "allowed_pods",
                                                             "cap_cpu", "cap_mem", "has_alloc_cpu", "has_alloc_mem")}
    out["alloc"] = [a["node_alloc"][r].copy() for r in rows]
    out["pods"] = [list(spec[off[r]:off[r + 1]]) for r in rows]
    return out


def _template_delta(enc: EncodedObjects, tails: dict, removed, changed, rows: dict):
    from .encode import MAX_RES, NodeDelta, TemplateDelta
    po = [0]
    for p in rows["pods"]:
        po.append(po[-1] + len(p))
    nrow = len(rows["name"])
    cols = {nm: rows[nm] for nm in ("name", "labelset", "taint_list", "unschedulable", "allowed_pods", "cap_cpu", "cap_mem",
                                    "has_alloc_cpu", "has_alloc_mem")}
    return TemplateDelta(NodeDelta(**tails), removed=sorted(removed), changed=sorted(changed), pod_off=po,
                         pod_spec=[x for p in rows["pods"] for x in p],
                         alloc=np.asarray(rows["alloc"], np.int64).reshape(nrow, MAX_RES), **cols)


def template_churn(enc: EncodedObjects, seed: int, n_change: int, n_remove: int, n_add: int):
    """A deterministic random tick of node-group template churn against a snapshot of ``generate``: ``n_remove`` random
    templates go away, ``n_change`` others change and ``n_add`` new ones (copies of random templates under a new name and
    pool) are appended.  A changed template gets a new name (the provider's random suffix) and, by turns, a zone value of
    another template (the first changed one a zone value no row had: a new domain), another taint list, other allocatable
    and allowed pods; an added one every third time a new zone value too.  DaemonSet pods stay those of the source.
    Returns the encode.TemplateDelta; ``enc.apply_template_delta(delta)`` is the snapshot after the tick."""
    a, s = enc.arrays, enc.struct
    N, T = s.num_cluster_nodes, s.num_templates
    rng = SplitMix64(0x7E3A0000 + seed)
    perm = rng.next(T).argsort() if T else np.zeros(0, np.int64)
    n_remove = min(n_remove, T)
    n_change = min(n_change, T - n_remove)
    removed = [int(t) for t in perm[:n_remove]]
    changed = sorted(int(t) for t in perm[n_remove:n_remove + n_change])
    src = changed + ([int(x) for x in rng.randint(n_add, T)] if T else [])
    n_add = len(src) - len(changed)
    rows = _template_rows(enc, src)
    nv, nl, nt = s.num_values, s.num_labelsets, s.num_taint_lists
    new_vals, new_ls = [], {}
    zones = []
    for r in range(N, N + T):
        ls = int(a["node_labelset"][r])
        zones += [int(v) for k, v in zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]],
                                         a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]]) if k == K_ZONE]
    name0 = int(a["node_name"].max()) + 1 if len(a["node_name"]) else 0
    r8 = rng.next(8 * max(len(src), 1)).reshape(-1, 8)
    u = rng.uniform(4 * max(len(src), 1)).reshape(-1, 4)
    for i in range(len(src)):
        ri = [int(x) for x in r8[i]]
        ls = int(rows["labelset"][i])
        lab = {int(k): int(v) for k, v in zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]],
                                              a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]])}
        rows["name"][i] = name0 + i
        new_zone = (i == 0 and n_change > 0) or (i >= len(changed) and ri[0] % 3 == 0)
        if new_zone:
            new_vals.append(0)
            lab[K_ZONE] = nv + len(new_vals) - 1
        elif zones and (i >= len(changed) or ri[1] % 2 == 0):
            lab[K_ZONE] = zones[ri[2] % len(zones)]
        if i >= len(changed) or ri[3] % 3 == 0:
            lab[K_POOL] = 16 + ri[4] % 8
        key = tuple(sorted(lab.items()))
        rows["labelset"][i] = new_ls.setdefault(key, nl + len(new_ls))
        if i < len(changed) and ri[5] % 2 == 0 and nt:
            rows["taint_list"][i] = ri[6] % nt
        if i < len(changed) and u[i][0] < 0.5:
            rows["alloc"][i][0] = max(1, int(rows["alloc"][i][0] * (0.5 + u[i][1])))
            rows["alloc"][i][1] = max(1, int(rows["alloc"][i][1] * (0.5 + u[i][2])))
            # one time in four at or past the DaemonSet pods it holds: every pod fails NodeResourcesFit there
            rows["allowed_pods"][i] = int(ri[7] % 121) if ri[7] % 4 else max(0, len(rows["pods"][i]) - (ri[7] >> 2) % 2)
    ls_items = sorted(new_ls.items(), key=lambda kv: kv[1])
    ls_off = [0]
    for k, _ in ls_items:
        ls_off.append(ls_off[-1] + len(k))
    tails = dict(value_is_int=[0] * len(new_vals), value_int=[0] * len(new_vals), ls_off=ls_off,
                 ls_key=[kk for k, _ in ls_items for kk, _v in k], ls_val=[v for k, _ in ls_items for _k, v in k])
    return _template_delta(enc, tails, removed, changed, rows)


def daemonset_rollout(enc: EncodedObjects, seed: int):
    """A DaemonSet created or rolled out: every template's DaemonSet pod list changes (every other template loses its
    first pod, the others gain one pod of a spec already on a template or resident).  Returns the encode.TemplateDelta
    with every template changed."""
    a, s = enc.arrays, enc.struct
    N, T = s.num_cluster_nodes, s.num_templates
    rng = SplitMix64(0xDA350000 + seed)
    rows = _template_rows(enc, range(T))
    pool = sorted(set(int(x) for x in a["node_pod_spec"]))
    pick = rng.randint(max(T, 1), max(len(pool), 1))
    for t in range(T):
        pods = rows["pods"][t]
        if t % 2 and pods:
            pods.pop(0)
        elif pool:
            pods.append(pool[int(pick[t])])
        if t % 5 == 4:   # a template whose DaemonSet pods now fill its pod limit
            rows["allowed_pods"][t] = len(pods)
    return _template_delta(enc, {}, [], range(T), rows)


def pod_churn(enc: EncodedObjects, seed: int, arrive: int, leave: int):
    """A deterministic random tick of workload churn against a snapshot of ``generate``: ``leave`` random pending groups
    finish, and ``arrive`` new workloads come, each a new spec copied from a random pending spec with a new cpu request
    (every third one also a new memory request) and 1..8 pending pods.  Returns the encode.PodDelta (no new dictionary
    entries: the copies reuse the label sets, constraints and lists of their originals)."""
    from .encode import PodDelta
    rng = SplitMix64(0x90D5 ^ (seed * 0x9E3779B9))
    a, S = enc.arrays, enc.struct.num_podspecs
    go = a["group_off"]
    E = len(go) - 1
    gone = set(int(x) for x in rng.randint(leave, max(E, 1))) if E else set()
    groups = [a["pend_spec"][go[g]:go[g + 1]] for g in range(E) if g not in gone]
    pending = np.unique(a["pend_spec"]) if len(a["pend_spec"]) else np.arange(S)
    src = pending[rng.randint(arrive, len(pending))] if len(pending) else np.zeros(arrive, np.int64)
    cols = {nm: a[nm][src] for nm in ("ps_namespace", "ps_labelset", "ps_tol_list", "ps_naff", "ps_node_name", "ps_port_list",
                                      "ps_pts_list", "ps_aff_list", "ps_anti_list", "ps_terminating", "ps_hostname_spread")}
    req = a["ps_req"][src].copy()
    req[:, 0] += 1 + rng.randint(arrive, 997)
    req[::3, 1] += 1 << 20
    sizes = 1 + rng.randint(arrive, 8)
    groups += [np.full(int(sizes[i]), S + i, np.int32) for i in range(arrive)]
    off = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
    return PodDelta(ps_req=req, group_off=off, pend_spec=np.concatenate(groups) if groups else [], **cols)


def node_group_families(config: int, templates: int, family: int, seed: int = 0, groups: Optional[int] = None):
    """Object-level node groups for cae_similar_node_groups: ``templates`` node groups in families of ``family`` zones of
    one instance type (the usual layout under --balance-similar-node-groups), and the pending groups of config ``config``'s
    pod shapes (E = pods / 100 groups unless ``groups`` is given, one pod each: only the exemplars matter here).
    Inside a family the allocatable cpu / memory carry a small jitter, and one member in six a jitter past the 5 % ratios;
    memory capacity varies within, and one member in eight past, the 1.5 % ratio; one member in five carries an extra
    taint, so that similar groups differ in schedulable sets, as they do for the pods (5 %) that select one zone.  Families
    differ in instance type, pool and DaemonSet requests.  Returns (templates {id: NodeInfo}, pod groups,
    [NodeGroupInfo])."""
    from .estimator import NodeGroupInfo
    from .objects import LABEL_ZONE, LABEL_HOSTNAME, Node, NodeInfo, Pod, PodEquivalenceGroup, Taint, Toleration
    cfg = CONFIGS[config]
    E = max(1, cfg.pods // 100) if groups is None else groups
    rng = SplitMix64(0x51A11A ^ (seed * 0x9E3779B9) ^ config)
    nfam = (templates + family - 1) // family
    f_vcpu = rng.choice(nfam, [2, 4, 8, 16, 32, 64, 96], [1] * 7)
    f_mem = rng.choice(nfam, [2, 4, 8], [1, 1, 1])
    f_gpu = np.where(rng.uniform(nfam) < 0.15, rng.choice(nfam, [1, 4, 8], [1, 1, 1]), 0)
    f_pool, f_ds, f_taint = rng.randint(nfam, 8), rng.randint(nfam, 5), rng.randint(nfam, 6)
    u_far, u_cap, u_taint = rng.uniform(templates), rng.uniform(templates), rng.uniform(templates)
    jit, mem_jit = rng.randint(templates, 1000), rng.randint(templates, 1000)
    mx = 1 + rng.randint(templates, 20)
    size = (rng.uniform(templates) * (mx + 1)).astype(np.int64).clip(0, mx)
    infos: dict = {}
    ngs = []
    for t in range(templates):
        f, z = t // family, t % family
        v, gpu = int(f_vcpu[f]), int(f_gpu[f])
        cap_cpu, cap_mem = v * 1000, v * int(f_mem[f]) * GiB
        far = u_far[t] < 1 / 6
        scale = (0.08 + 0.04 * jit[t] / 1000) if far else 0.02 * jit[t] / 1000       # fraction of the allocatable taken off
        alloc_cpu = int((cap_cpu - RESERVED[v]) * (1 - scale))
        alloc_mem = int((cap_mem - cap_mem // 20) * (1 - scale))
        if u_cap[t] < 1 / 8:
            cap_mem = int(cap_mem * (1.02 + 0.01 * mem_jit[t] / 1000))
        else:
            cap_mem = int(cap_mem * (1 - 0.01 * mem_jit[t] / 1000))
        alloc = {"cpu": alloc_cpu, "memory": alloc_mem, "pods": 110}
        cap = {"cpu": cap_cpu, "memory": cap_mem, "pods": 110}
        if gpu:
            alloc["nvidia.com/gpu"] = cap["nvidia.com/gpu"] = gpu
        taints = []
        if f_taint[f] < 2:
            taints.append(Taint("dedicated", "team-%d" % f_taint[f]))
        if u_taint[t] < 0.2:
            taints.append(Taint("maintenance", "soon"))
        name = "ng-%05d" % t
        node = Node(name + "-template", labels={LABEL_HOSTNAME: name + "-template", LABEL_ZONE: "zone-%d" % z,
                                                "pool": "pool-%d" % f_pool[f], "instance-type": "it-%d-%d-%d" % (v, f_mem[f], gpu)},
                    taints=taints, allocatable=alloc, capacity=cap)
        ds = [Pod("%s-ds-%d" % (name, i), namespace="kube-system",
                  requests={"cpu": 100 + 20 * int(f_ds[f]), "memory": (200 + 50 * int(f_ds[f])) * MiB},
                  tolerations=[Toleration(operator="Exists")]) for i in range(2)]
        infos[name] = NodeInfo(node, ds)
        ngs.append(NodeGroupInfo(name, int(mx[t]), int(size[t])))
    cpu = rng.choice(E, [50, 100, 250, 500, 1000, 2000, 4000], [20, 25, 20, 15, 10, 7, 3]).astype(np.int64)
    mem = cpu * rng.choice(E, [1, 2, 4, 8], [1, 1, 1, 1]).astype(np.int64) * MiB
    gpu = np.where(rng.uniform(E) < 0.10, rng.choice(E, [1, 2, 4, 8], [1, 1, 1, 1]), 0)
    u_tol, u_sel, sel = rng.uniform(E), rng.uniform(E), rng.randint(E, 16)
    pgs = []
    for g in range(E):
        req = {"cpu": int(cpu[g]), "memory": int(mem[g])}
        if gpu[g]:
            req["nvidia.com/gpu"] = int(gpu[g])
        tols = []
        if u_tol[g] < 0.3:
            tols.append(Toleration("dedicated", "Equal", "team-%d" % (g % 2), "NoSchedule"))
        if u_tol[g] < 0.1:
            tols.append(Toleration("maintenance", "Exists"))
        node_sel = {}
        if u_sel[g] < 0.05:
            node_sel[LABEL_ZONE] = "zone-%d" % (sel[g] % family)
        elif u_sel[g] < 0.15:
            node_sel["pool"] = "pool-%d" % (sel[g] % 8)
        pgs.append(PodEquivalenceGroup([Pod("p-%d" % g, namespace="ns-%d" % (g % 32), labels={"app": "a%d" % g}, requests=req,
                                            tolerations=tols, node_selector=node_sel)]))
    return infos, pgs, ngs
