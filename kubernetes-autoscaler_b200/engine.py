"""Python binding of the engine's C ABI (``include/caengine.h``) — what the cgo shim does in Go.

There is no CPU path here: if ``libcaengine.so`` or a CUDA device is missing every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import numpy as np

from . import capi
from .encode import DaemonSetInputs, EligibilityInputs, EncodedObjects, PriceInputs, RemovalPlan, ResidentRemovals, SimilarityInputs


class EngineError(RuntimeError):
    pass


class EngineUnsupported(EngineError):
    """Status > 0: the input uses something the engine refuses; the caller must use the stock path."""


def _vp(a: Optional[np.ndarray]):
    """The array's data as a void*, NULL for None."""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _opt(a, dtype) -> Optional[np.ndarray]:
    """A contiguous array of `dtype`, None for None (a NULL argument)."""
    return None if a is None else np.ascontiguousarray(a, dtype)


class PinnedArray:
    """numpy view over page-locked memory from cae_host_alloc."""

    def __init__(self, lib, shape, dtype) -> None:
        self._lib = lib
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self._ptr = lib.cae_host_alloc(max(self.nbytes, 16))
        if not self._ptr:
            raise EngineError("cae_host_alloc failed")
        buf = (C.c_uint8 * max(self.nbytes, 1)).from_address(self._ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def close(self) -> None:
        if self._ptr:
            self.array = None
            self._lib.cae_host_free(self._ptr)
            self._ptr = None

    def __del__(self) -> None:
        try:
            self.close()
        except Exception:
            pass


def shard_pods(P: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Block partition of the pending pods for the dense pass; shard starts are multiples of 32 so the
    template-major bit rows of the ranks concatenate word by word (must match pod_shard in csrc/api.cu)."""
    b = (P * rank // world_size) // 32 * 32
    e = P * (rank + 1) // world_size
    if rank + 1 < world_size:
        e = e // 32 * 32
    return b, e


def shard_templates(T: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Block partition of the templates for the pack: rows of other ranks stay zero, so a sum
    all-reduce of node_count|pod_count assembles the result."""
    return T * rank // world_size, T * (rank + 1) // world_size


class Engine:
    def __init__(self, device: int = 0, rank: int = 0, world_size: int = 1, want_reasons: bool = False,
                 pods_presharded: bool = False, feature_gates: Optional[int] = None) -> None:
        self.lib = capi.load_engine_lib()
        cfg = capi.cae_config()
        cfg.abi_version = capi.CONST["CAE_ABI_VERSION"]
        cfg.device, cfg.rank, cfg.world_size, cfg.want_reasons = device, rank, world_size, int(want_reasons)
        self.rank, self.world_size, self.want_reasons = rank, world_size, want_reasons
        self.pods_presharded = pods_presharded
        # the scheduler feature gates as the Go side would report them; default = the values the engine implements
        gates = capi.CONST["CAE_GATE_NODE_INCLUSION_POLICY_IN_PTS"] | capi.CONST["CAE_GATE_MATCH_LABEL_KEYS_IN_PTS"] \
            if feature_gates is None else int(feature_gates)
        cfg.flags = capi.CONST["CAE_CFG_GATES_REPORTED"] | (capi.CONST["CAE_CFG_PODS_PRESHARDED"] if pods_presharded else 0)
        cfg.feature_gates = gates
        h = C.c_void_p()
        self._check(self.lib.cae_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self.enc: Optional[EncodedObjects] = None
        self._pinned = {}

    # ---- plumbing ---------------------------------------------------------------------------
    def _check(self, rc: int) -> None:
        if rc == 0:
            return
        msg = (self.lib.cae_last_error() or b"").decode()
        if rc > 0:
            raise EngineUnsupported(msg)
        raise EngineError("caengine status %d: %s" % (rc, msg))

    def _applied(self, rc: int) -> bool:
        """A delta call's status: False on 2 ("use a full load"; the engine is unchanged), True on 0, raises otherwise."""
        if rc == 2:
            return False
        self._check(rc)
        return True

    def close(self) -> None:
        if getattr(self, "h", None):
            for p in self._pinned.values():
                p.close()
            self._pinned = {}
            self.lib.cae_destroy(self.h)
            self.h = None

    def __del__(self) -> None:
        try:
            self.close()
        except Exception:
            pass

    def _pin(self, name: str, shape, dtype) -> np.ndarray:
        cur = self._pinned.get(name)
        if cur is None or cur.array.shape != tuple(shape) or cur.array.dtype != np.dtype(dtype):
            if cur is not None:
                cur.close()
            cur = PinnedArray(self.lib, tuple(shape), dtype)
            self._pinned[name] = cur
        return cur.array

    # ---- shards -------------------------------------------------------------------------------
    def pod_shard(self, P: int) -> Tuple[int, int]:
        if self.pods_presharded:   # the loaded objects hold this rank's pods only
            return 0, P
        return shard_pods(P, self.rank, self.world_size)

    def template_shard(self, T: int) -> Tuple[int, int]:
        return shard_templates(T, self.rank, self.world_size)

    # ---- API ------------------------------------------------------------------------------------
    def load(self, enc: EncodedObjects) -> None:
        self.enc = enc
        self._check(self.lib.cae_load(self.h, enc.ptr()))

    def load_pending(self, enc: EncodedObjects) -> bool:
        """The per-tick delta (cae_load_pending): only the pending-pod rows of `enc` travel; nodes, templates and pod specs
        must be the ones of the last load().  Returns False when the engine answers "use a full load" (status 2)."""
        ok = self._applied(self.lib.cae_load_pending(self.h, enc.P, _vp(enc.arrays["pend_spec"]), enc.E,
                                                     _vp(enc.arrays["group_off"])))
        if ok:
            self.enc = enc
        return ok

    def load_nodes(self, delta) -> bool:
        """The per-tick delta of the cluster nodes (cae_load_nodes): new rows of existing cluster nodes plus the dictionary
        tails they need (encode.NodeDelta).  Returns False when the engine answers "use a full load" (status 2); the engine
        is unchanged then."""
        return self._applied(self.lib.cae_load_nodes(self.h, delta.ptr()))

    def load_node_churn(self, churn) -> bool:
        """The per-tick delta of the cluster-node list (cae_load_node_churn): removed and added cluster nodes plus the
        dirty rows of the survivors (encode.NodeChurn).  Returns False when the engine answers "use a full load" (status 2);
        the engine is unchanged then."""
        return self._applied(self.lib.cae_load_node_churn(self.h, churn.ptr()))

    def add_upcoming_nodes(self, up) -> bool:
        """The scale-up's upcoming nodes as copies of their templates (cae_add_upcoming_nodes), applied with the loop's
        node churn in one rebuild (encode.UpcomingNodes).  Returns False when the engine answers "use a full load" (status
        2); the engine is unchanged then."""
        return self._applied(self.lib.cae_add_upcoming_nodes(self.h, up.ptr()))

    def load_templates(self, delta, enc: Optional[EncodedObjects] = None) -> bool:
        """The per-tick delta of the node-group templates (cae_load_templates): removed, changed and added templates plus
        the dictionary tails they need (encode.TemplateDelta).  Returns False when the engine answers "use a full load"
        (status 2); the engine is unchanged then.  `enc`: the objects the engine now holds
        (EncodedObjects.apply_template_delta), kept as this engine's shapes (the template count changes)."""
        ok = self._applied(self.lib.cae_load_templates(self.h, delta.ptr()))
        if ok and enc is not None:
            self.enc = enc
        return ok

    def load_pods(self, delta, enc: Optional[EncodedObjects] = None) -> int:
        """The per-tick delta of the pod specs (cae_load_pods): new pod specs with the dictionary tails they need and the
        complete new pending list (encode.PodDelta).  Returns the status: 0 applied, 1 a limit of the engine (use the stock
        path), 2 a table would overflow (use a full load); the engine is unchanged unless 0.  `enc`: the objects the engine
        now holds (EncodedObjects.apply_pod_delta), kept as this engine's shapes."""
        rc = self.lib.cae_load_pods(self.h, delta.ptr())
        if rc in (1, 2):
            return rc
        self._check(rc)
        if enc is not None:
            self.enc = enc
        return 0

    def force_add_pods(self, pods: Sequence[int], nodes: Sequence[int], enc: Optional[EncodedObjects] = None):
        """ClusterSnapshot.ForceAddPod for a list of pending pods (cae_force_add_pods): pending pod pods[i] becomes a
        resident of cluster row nodes[i] and leaves the pending list, e.g. what filter_schedulable assigned.  Returns
        new_index [P before the call] int32 (-1 = moved), or False when the engine answers "use a full load" (status 2);
        the engine is unchanged then.  `enc`: the objects the engine now holds (EncodedObjects.apply_force_add), kept as
        this engine's shapes."""
        pd, nd = np.ascontiguousarray(pods, np.int32), np.ascontiguousarray(nodes, np.int32)
        if pd.ndim != 1 or pd.shape != nd.shape:
            raise ValueError("force_add_pods: pods and nodes must be two lists of one length")
        # new_index is worked out here, not asked of the library: the library writes one entry per pending pod IT holds, and
        # this object's shapes (self.enc) are only as current as the caller kept them
        if not self._applied(self.lib.cae_force_add_pods(self.h, len(pd), _vp(pd), _vp(nd), None)):
            return False
        keep = np.ones(self.enc.P, bool)
        keep[pd] = False
        new_index = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
        if enc is not None:
            self.enc = enc
        return new_index

    def feasibility(self, want_bits: bool = True):
        """Dense pods x templates pass. Returns (fit_bits [T][ceil(Pl/32)] uint32 | None,
        reasons [T][Pl] uint8 | None, fit_count [T] int32) for this rank's pod shard."""
        enc = self.enc
        pb, pe = self.pod_shard(enc.P)
        Pl, T = pe - pb, enc.T
        bits = self._pin("bits", (T, (Pl + 31) // 32), np.uint32) if want_bits else None
        reasons = self._pin("reasons", (T, Pl), np.uint8) if self.want_reasons else None
        count = self._pin("count", (T,), np.int32)
        self._check(self.lib.cae_feasibility(self.h, _vp(bits), _vp(reasons), _vp(count)))
        return bits, reasons, count

    def feasibility_groups(self) -> np.ndarray:
        enc = self.enc
        out = np.zeros((enc.T, enc.E), np.uint8)
        self._check(self.lib.cae_feasibility_groups(self.h, _vp(out)))
        return out

    def group_reasons(self, considered=None, exist=None, want_detail: bool = False):
        """cae_group_reasons: every group's rejection reasons counted over the node groups.  considered / exist: [T] flags
        (None = all).  Returns (schedulable [E] uint8, counts [E][CAE_REASON_KEYS] int32, detail [T][E] uint16 | None)."""
        enc = self.enc
        T, E = enc.T, enc.E
        cons, ex = _opt(considered, np.uint8), _opt(exist, np.uint8)
        for m in (cons, ex):
            if m is not None and m.shape != (T,):
                raise ValueError("group_reasons: a mask needs one flag per template")
        sched = np.zeros(E, np.uint8)
        counts = np.zeros((E, capi.CONST["CAE_REASON_KEYS"]), np.int32)
        detail = np.zeros((T, E), np.uint16) if want_detail else None
        self._check(self.lib.cae_group_reasons(self.h, _vp(cons), _vp(ex), _vp(sched), _vp(counts), _vp(detail)))
        return sched, counts, detail

    def estimate_all_li(self, max_nodes, last_index_in):
        """cae_estimate_all_ex: Estimate of every template with the plugin runner's lastIndex carried in per template.
        Returns node_count, pod_count, sched, order, last_index_out."""
        enc = self.enc
        T, E = enc.T, enc.E
        mn = _opt(max_nodes, np.int32)
        li = np.ascontiguousarray(last_index_in, np.int32)
        nc, pc = np.zeros(T, np.int32), np.zeros(T, np.int32)
        sched, order = np.zeros((T, E), np.int32), np.zeros((T, E), np.int32)
        lo = np.zeros(T, np.int32)
        self._check(self.lib.cae_estimate_all_ex(self.h, _vp(mn), _vp(li), _vp(nc), _vp(pc), _vp(sched), _vp(order), _vp(lo)))
        return nc, pc, sched, order, lo

    def estimate_all(self, max_nodes: Optional[Sequence[int]] = None, want_sched: bool = True, copy: bool = True):
        """Returns node_count[T], pod_count[T], sched_count[T][E], order[T][E] (rows outside this
        rank's template shard are zero / -1).  Outputs land in pinned buffers; copy=False returns
        views that the next call overwrites; want_sched=False skips the two [T][E] matrices."""
        enc = self.enc
        T, E = enc.T, enc.E
        mn = _opt(max_nodes, np.int32)
        node_count = self._pin("node_count", (T,), np.int32)
        pod_count = self._pin("pod_count", (T,), np.int32)
        sched = self._pin("sched", (T, E), np.int32) if want_sched else None
        order = self._pin("order", (T, E), np.int32) if want_sched else None
        self._check(self.lib.cae_estimate_all(self.h, _vp(mn), _vp(node_count), _vp(pod_count), _vp(sched), _vp(order)))
        if copy:
            return (node_count.copy(), pod_count.copy(), None if sched is None else sched.copy(),
                    None if order is None else order.copy())
        return node_count, pod_count, sched, order

    def expander_best(self, chain: Sequence[int], node_count, pod_count, sched=None):
        """sched=None scores the device-resident result of the last estimate_all (single shard)."""
        enc = self.enc
        ch = np.asarray(chain, np.int32)
        nc = np.ascontiguousarray(node_count, np.int32)
        pc = np.ascontiguousarray(pod_count, np.int32)
        sc = _opt(sched, np.int32)
        mask = np.zeros(enc.T, np.uint8)
        waste = np.zeros(enc.T, np.float64)
        self._check(self.lib.cae_expander_best(self.h, _vp(ch), len(ch), _vp(nc), _vp(pc), _vp(sc), _vp(mask), _vp(waste)))
        return mask, waste

    def waste_scores(self) -> np.ndarray:
        """Least-waste score of this rank's template shard from the device-resident result of the last estimate_all
        (0.0 for the rows of other ranks: a sum all-reduce of float64[T] assembles the vector)."""
        waste = np.zeros(self.enc.T, np.float64)
        self._check(self.lib.cae_waste_scores(self.h, _vp(waste)))
        return waste

    def price_scores(self, node_price, pod_price, stabilization_price: float, preferred_cpu_milli: int = 0, unfitness=None,
                     has_gpu=None, exists=None, node_count=None, sched=None, order=None) -> np.ndarray:
        """Price expander score per option (expander/price/price.go).  node_count/sched/order None = the device-resident
        result of the last estimate_all."""
        pin = PriceInputs(node_price=node_price, pod_price=pod_price, unfitness=unfitness, has_gpu=has_gpu, exists=exists,
                          price_error=None, stabilization_price=float(stabilization_price),
                          preferred_cpu_milli=int(preferred_cpu_milli))
        score = np.zeros(self.enc.T, np.float64)
        nc, sc, od = _opt(node_count, np.int32), _opt(sched, np.int32), _opt(order, np.int32)
        self._check(self.lib.cae_price_scores(self.h, pin.ptr(), _vp(nc), _vp(sc), _vp(od), _vp(score)))
        return score

    def filter_schedulable(self, pod_order: Sequence[int], hint_node=None, sim_class=None, class_ctrl=None, node_ok=None,
                           last_index: int = 0, break_on_failure: bool = False):
        """HintingSimulator.TrySchedulePods on the cluster snapshot of the last load.  Returns (assigned[P] cluster node
        index or -1, lastIndex afterwards, overflowing controller count)."""
        enc = self.enc
        order = np.ascontiguousarray(pod_order, np.int32)
        hn = _opt(hint_node, np.int32)
        sc = _opt(sim_class, np.int32)
        cc = _opt(class_ctrl, np.int32)
        ok = _opt(node_ok, np.uint8)
        assigned = np.full(max(enc.P, 1), -1, np.int32)
        li, ov = np.zeros(1, np.int32), np.zeros(1, np.int32)
        self._check(self.lib.cae_filter_schedulable(self.h, _vp(order), len(order), _vp(hn), _vp(sc), _vp(cc),
                                                    0 if cc is None else len(cc), _vp(ok), int(last_index), int(break_on_failure),
                                                    _vp(assigned), _vp(li), _vp(ov)))
        return assigned[:enc.P], int(li[0]), int(ov[0])

    def simulate_removals(self, cand_node, move_off, move_pod, dest_ok=None, hint_node=None, sim_class=None, class_ctrl=None,
                          last_index: int = 0, persist: bool = False, log_cap: Optional[int] = None):
        """RemovalSimulator.SimulateNodeRemoval on every candidate in order, on the snapshot of the last load
        (cae_simulate_removals).  Returns (result[n_cand] CAE_REMOVAL_*, lastIndex afterwards, log [n][3] = (candidate,
        pending pod, cluster row or -1) per pod tried).  A log that outgrows `log_cap` (default: one entry per listed pod
        plus room for moved-in pods) is fetched again at the size the engine reports."""
        move_off = np.ascontiguousarray(move_off, np.int32)
        cap = int(log_cap) if log_cap is not None else int(move_off[-1]) + 64 if len(move_off) else 0
        rc, res, li, log = self._simulate_removals_raw(cand_node, move_off, move_pod, dest_ok, hint_node, sim_class, class_ctrl,
                                                        last_index, persist, cap)
        if rc == 1:   # the log needed more room: once more at the size it reported
            rc, res, li, log = self._simulate_removals_raw(cand_node, move_off, move_pod, dest_ok, hint_node, sim_class,
                                                            class_ctrl, last_index, persist, len(log))
        self._check(rc)
        return res, li, log

    def _simulate_removals_raw(self, cand_node, move_off, move_pod, dest_ok, hint_node, sim_class, class_ctrl, last_index,
                               persist, log_cap):
        """One cae_simulate_removals call: (status, result, lastIndex, log); on status 1 the log is zeros of the needed length."""
        cn = np.ascontiguousarray(cand_node, np.int32)
        mo = np.ascontiguousarray(move_off, np.int32)
        mp = np.ascontiguousarray(move_pod, np.int32)
        ok = _opt(dest_ok, np.uint8)
        hn = _opt(hint_node, np.int32)
        sc = _opt(sim_class, np.int32)
        cc = _opt(class_ctrl, np.int32)
        res = np.zeros(max(len(cn), 1), np.int32)
        log = np.zeros((max(log_cap, 1), 3), np.int32)
        li, n = np.zeros(1, np.int32), np.zeros(1, np.int32)
        rc = self.lib.cae_simulate_removals(self.h, len(cn), _vp(cn), _vp(mo), _vp(mp), _vp(ok), _vp(hn), _vp(sc), _vp(cc),
                                            0 if cc is None else len(cc), int(last_index), int(bool(persist)), _vp(res), _vp(li),
                                            _vp(log), int(log_cap), _vp(n))
        if rc == 1:
            return rc, None, None, np.zeros((int(n[0]), 3), np.int32)
        return rc, res[:len(cn)], int(li[0]), log[:int(n[0])]

    def simulate_resident_removals(self, cand_node, move_off, move_slot, dest_ok=None, hint_node=None, sim_class=None,
                                   class_ctrl=None, last_index: int = 0, persist: bool = False, log_cap: Optional[int] = None,
                                   enc: Optional[EncodedObjects] = None):
        """The removal batch of simulate_removals on the resident snapshot (cae_simulate_resident_removals): move_slot
        names each pod to move by its position in its candidate row's resident list; hint_node / sim_class are per listed
        pod.  Returns (result[n_cand], lastIndex afterwards, log [n][3] = (candidate, k, cluster row or -1) with k the
        listing where the pod was first listed).  Afterwards the engine holds the movers as its pending pods; this object's
        shapes follow through EncodedObjects.apply_resident_removals (`enc`: that result, when the caller has it).
        Raises EngineUnsupported on status 1 (a limit judged on the movers) or 2 (a table would overflow)."""
        move_off = np.ascontiguousarray(move_off, np.int32)
        cap = int(log_cap) if log_cap is not None else int(move_off[-1]) + 64 if len(move_off) else 0
        args = (cand_node, move_off, move_slot, dest_ok, hint_node, sim_class, class_ctrl, last_index, persist)
        rc, res, li, log = self._simulate_resident_removals_raw(*args, cap)
        if rc == 1 and len(log) > cap:   # the log needed more room: once more at the size it reported
            rc, res, li, log = self._simulate_resident_removals_raw(*args, len(log))
        self._check(rc)
        self.enc = enc if enc is not None else self.enc.apply_resident_removals(cand_node, move_off, move_slot)[0]
        return res, li, log

    def _simulate_resident_removals_raw(self, cand_node, move_off, move_slot, dest_ok, hint_node, sim_class, class_ctrl,
                                        last_index, persist, log_cap):
        """One cae_simulate_resident_removals call: (status, result, lastIndex, log); on status 1 the log is zeros of the
        needed length (0 for a limit)."""
        cn = np.ascontiguousarray(cand_node, np.int32).reshape(-1)
        cc = _opt(class_ctrl, np.int32)
        rr = ResidentRemovals(cand_node=cn, move_off=np.ascontiguousarray(move_off, np.int32),
                              move_slot=np.ascontiguousarray(move_slot, np.int32), dest_ok=_opt(dest_ok, np.uint8),
                              hint_node=_opt(hint_node, np.int32), sim_class=_opt(sim_class, np.int32), class_ctrl=cc,
                              n_classes=0 if cc is None else len(cc), last_index_in=int(last_index), persist=int(bool(persist)))
        res = np.zeros(max(len(cn), 1), np.int32)
        log = np.zeros((max(log_cap, 1), 3), np.int32)
        li, n = np.zeros(1, np.int32), np.zeros(1, np.int32)
        rc = self.lib.cae_simulate_resident_removals(self.h, rr.ptr(), _vp(res), _vp(li), _vp(log), int(log_cap), _vp(n))
        if rc == 1:
            return rc, None, None, np.zeros((int(n[0]), 3), np.int32)
        return rc, res[:len(cn)], int(li[0]), log[:int(n[0])]

    def plan_removals(self, plan: RemovalPlan, log_cap: Optional[int] = None, enc: Optional[EncodedObjects] = None):
        """The planner's removal loop on the resident snapshot (cae_plan_removals) for the inputs `plan`.  Returns a dict:
        result [n_cand] CAE_REMOVAL_*, block_pos / block_reason / pdb_slack [n_cand], pdb_left [n_pdb], last_index, log
        [n][3] = (candidate, k, cluster row or -1) with k the potential-mover listing where the pod was first listed, and
        move_off / move_slot, that listing (every MOVE or UNDEFINED resident pod of each candidate's row, in slot order).
        A log past `log_cap` (default: one entry per potential mover plus 64) is fetched again at the size the engine
        reports.  Afterwards the engine holds the potential movers as its pending pods (`enc`: the objects after the call,
        when the caller has them).  Raises EngineUnsupported on status 1 or 2."""
        cand = plan.arrays["cand_node"]
        drain = plan.arrays["drain"]
        N = self.enc.struct.num_cluster_nodes
        res_off = self.enc.arrays["node_pod_off"][:N + 1]
        move_off, move_slot = [0], []
        for row in cand.tolist():
            if 0 <= row < N:   # (a row out of range is the engine's to refuse)
                b = drain[res_off[row]:res_off[row + 1]] & 3
                move_slot += np.flatnonzero((b == 0) | (b == 2)).tolist()
            move_off.append(len(move_slot))
        n, B = len(cand), plan.struct.n_pdb
        cap = int(log_cap) if log_cap is not None else len(move_slot) + 64
        out = {nm: np.zeros(max(n, 1), np.int32) for nm in ("result", "block_pos", "block_reason", "pdb_slack")}
        out["pdb_left"] = np.zeros(max(B, 1), np.int32)
        li, m = np.zeros(1, np.int32), np.zeros(1, np.int32)
        for _ in range(2):
            log = np.zeros((max(cap, 1), 3), np.int32)
            rc = self.lib.cae_plan_removals(self.h, plan.ptr(), _vp(out["result"]), _vp(out["block_pos"]), _vp(out["block_reason"]),
                                            _vp(out["pdb_slack"]), _vp(out["pdb_left"]), _vp(li), _vp(log), int(cap), _vp(m))
            if rc != 1 or int(m[0]) <= cap:
                break
            cap = int(m[0])   # the log needed more room: once more at the size it reported
        self._check(rc)
        move_off = np.asarray(move_off, np.int32)
        self.enc = enc if enc is not None else self.enc.apply_resident_removals(cand, move_off, move_slot)[0]
        res = {nm: a[:n] for nm, a in out.items() if nm != "pdb_left"}
        res.update(pdb_left=out["pdb_left"][:B], last_index=int(li[0]), log=log[:int(m[0])], move_off=move_off,
                   move_slot=np.asarray(move_slot, np.int32))
        return res

    def check_capacity(self, req_kind, req_off, req_pod, hint_node=None, sim_class=None, class_ctrl=None, last_index: int = 0):
        """The ProvisioningRequest capacity batch on the snapshot of the last load (cae_check_capacity): BOOK requests keep
        what they place, a CHECK request is committed only when every pod fits, and nothing stays in the snapshot.
        Returns (result [n_req] CAE_CAPACITY_*, assigned [P] cluster row or -1 per pending pod, lastIndex afterwards)."""
        kd = np.ascontiguousarray(req_kind, np.int32)
        ro = np.ascontiguousarray(req_off, np.int32)
        rp = np.ascontiguousarray(req_pod, np.int32)
        hn = _opt(hint_node, np.int32)
        sc = _opt(sim_class, np.int32)
        cc = _opt(class_ctrl, np.int32)
        res = np.zeros(max(len(kd), 1), np.int32)
        assigned = np.full(max(self.enc.P, 1), -1, np.int32)
        li = np.zeros(1, np.int32)
        self._check(self.lib.cae_check_capacity(self.h, len(kd), _vp(kd), _vp(ro), _vp(rp), _vp(hn), _vp(sc), _vp(cc),
                                                0 if cc is None else len(cc), int(last_index), _vp(res), _vp(assigned), _vp(li)))
        return res[:len(kd)], assigned[:self.enc.P], int(li[0])

    def similar_node_groups(self, res_sig, free_dims, eligible, max_size, target_size, ignored_keys=(), safe=None,
                            ratios=(0.05, 0.05, 0.015)):
        """cae_similar_node_groups over the loaded templates.  ratios = (allocatable, free, memory capacity).  Returns
        (bits [T, ceil(T/32)] uint32: bit s of row t = s is similar to t, count [T] int32, sng_limit [T] int64).  Raises
        EngineUnsupported on status 1 (a quantity past INT64_MAX / 1000)."""
        T = self.enc.T
        alloc_ratio, free_ratio, mem_ratio = (float(r) for r in ratios)
        si = SimilarityInputs(ignored_keys=list(ignored_keys), res_sig=res_sig, free_dims=free_dims, eligible=eligible, safe=safe,
                              max_size=max_size, target_size=target_size, max_allocatable_difference_ratio=alloc_ratio,
                              max_free_difference_ratio=free_ratio, max_capacity_memory_difference_ratio=mem_ratio)
        bits = np.zeros((T, (T + 31) // 32), np.uint32)
        count = np.zeros(T, np.int32)
        limit = np.zeros(T, np.int64)
        self._check(self.lib.cae_similar_node_groups(self.h, si.ptr(), _vp(bits), _vp(count), _vp(limit)))
        return bits, count, limit

    def template_daemonsets(self, ds_spec, evaluate=None, running=None, keep=None, enc: Optional[EncodedObjects] = None):
        """cae_template_daemonsets: NodeShouldRunDaemonPod of every loaded template and DaemonSet spec ds_spec [D].
        evaluate [T] flags (None = all); running [T][ceil(D/32)] uint32 bits of the DaemonSets already on the example node
        (None = none); keep [T] (None = report only): each evaluated template keeps its first keep[t] pods and gets the
        pods of its bits after them.  Returns (bits [T][ceil(D/32)] uint32, count [T] int32).  After an apply this object's
        shapes follow daemonset.apply_run_bits (`enc`: the objects after the call, when the caller has them).  Raises
        EngineUnsupported when the apply is refused (status 1 or 2); the engine is unchanged then."""
        T = self.enc.T
        ds = np.ascontiguousarray(ds_spec, np.int32).reshape(-1)
        Dw = (len(ds) + 31) // 32
        di = DaemonSetInputs(ds_spec=ds, evaluate=_opt(evaluate, np.uint8), running=_opt(running, np.uint32), keep=_opt(keep, np.int32))
        for nm, shape in (("evaluate", (T,)), ("keep", (T,)), ("running", (T, Dw))):
            if nm in di.arrays and di.arrays[nm].size != int(np.prod(shape)):
                raise ValueError("template_daemonsets: %s needs %s entries" % (nm, shape))
        bits = np.zeros((T, Dw), np.uint32)
        count = np.zeros(T, np.int32)
        self._check(self.lib.cae_template_daemonsets(self.h, di.ptr(), _vp(bits), _vp(count)))
        if keep is not None:
            if enc is None:
                from .daemonset import apply_run_bits, unpack_rows
                enc = apply_run_bits(self.enc, ds, unpack_rows(bits, len(ds)), di.arrays["keep"], evaluate)[1]
            self.enc = enc
        return bits, count

    def scale_down_eligibility(self, cand_node, gpu_dim, threshold, pod_flags=None, skip_ds=None, skip_mirror: bool = False,
                               pre_reason=None, unready=None):
        """cae_scale_down_eligibility on the resident snapshot: every candidate's utilization and eligibility reason.
        cand_node [n] cluster rows; gpu_dim [n] (-1 no GpuConfig, -2 a resource the load has no dim for); threshold [n];
        pod_flags [resident pods of the cluster rows] bits DaemonSet | mirror << 1 | long-terminating << 2 (None = all 0);
        skip_ds / pre_reason / unready [n] flags (None = all 0).  Returns (util [n][4] float64: cpu, mem, gpu, Utilization;
        reason [n] uint8 CAE_ELIG_*; unneeded: the candidate indices with reason CAE_ELIG_UNNEEDED, in input order).
        Raises EngineUnsupported on status 1 (a quantity that leaves int64)."""
        cn = np.ascontiguousarray(cand_node, np.int32).reshape(-1)
        n = len(cn)
        ei = EligibilityInputs(cand_node=cn, gpu_dim=np.ascontiguousarray(gpu_dim, np.int32), skip_mirror=int(bool(skip_mirror)),
                               threshold=np.ascontiguousarray(threshold, np.float64), pod_flags=_opt(pod_flags, np.uint8),
                               skip_ds=_opt(skip_ds, np.uint8), pre_reason=_opt(pre_reason, np.uint8), unready=_opt(unready, np.uint8))
        for nm in ("gpu_dim", "threshold", "skip_ds", "pre_reason", "unready"):
            if nm in ei.arrays and ei.arrays[nm].shape != (n,):
                raise ValueError("scale_down_eligibility: %s needs one entry per candidate" % nm)
        util = np.zeros((max(n, 1), 4), np.float64)
        reason = np.zeros(max(n, 1), np.uint8)
        unneeded = np.zeros(max(n, 1), np.int32)
        m = np.zeros(1, np.int32)
        self._check(self.lib.cae_scale_down_eligibility(self.h, ei.ptr(), _vp(util), _vp(reason), _vp(unneeded), _vp(m)))
        return util[:n], reason[:n], unneeded[:int(m[0])]

    # ---- fused histogram exchange over peer memory (multi-GPU dense pass) -------------------------
    def peer_handle(self) -> bytes:
        buf = C.create_string_buffer(capi.CONST["CAE_PEER_HANDLE_BYTES"])
        self._check(self.lib.cae_peer_handle(self.h, buf))
        return buf.raw

    def peer_attach(self, handles: Sequence[bytes]) -> None:
        blob = b"".join(handles)
        assert len(blob) == capi.CONST["CAE_PEER_HANDLE_BYTES"] * self.world_size
        self._check(self.lib.cae_peer_attach(self.h, C.create_string_buffer(blob, len(blob)), self.world_size))

    def stats(self) -> capi.cae_stats:
        s = capi.cae_stats()
        self._check(self.lib.cae_get_stats(self.h, C.byref(s)))
        return s

    def stream(self) -> int:
        """cudaStream_t of the engine (e.g. for torch.cuda.ExternalStream)."""
        return int(self.lib.cae_stream(self.h) or 0)

    def device_buffer(self, which: int) -> Tuple[int, int]:
        n = C.c_size_t(0)
        p = self.lib.cae_device_buffer(self.h, which, C.byref(n))
        return int(p or 0), int(n.value)


def _expander_chain(fn: str, chain: Sequence[int], node_count, pod_count, *scores) -> np.ndarray:
    """One call of the host-side filter chain `fn` (cae_expander_chain or cae_expander_chain_ex): the best-option mask."""
    lib = capi.load_engine_lib()
    ch = np.asarray(chain, np.int32)
    nc = np.ascontiguousarray(node_count, np.int32)
    pc = np.ascontiguousarray(pod_count, np.int32)
    mask = np.zeros(len(nc), np.uint8)
    rc = getattr(lib, fn)(_vp(ch), len(ch), len(nc), _vp(nc), _vp(pc), *map(_vp, scores), _vp(mask))
    if rc != 0:
        raise EngineError("%s status %d: %s" % (fn, rc, (lib.cae_last_error() or b"").decode()))
    return mask


def expander_chain(chain: Sequence[int], node_count, pod_count, waste) -> np.ndarray:
    """The expander filter chain on the host (cae_expander_chain): needs the library, not a GPU."""
    return _expander_chain("cae_expander_chain", chain, node_count, pod_count, np.ascontiguousarray(waste, np.float64))


def expander_chain_ex(chain: Sequence[int], node_count, pod_count, waste=None, price=None, price_error=None, priority=None) -> np.ndarray:
    """cae_expander_chain_ex: the chain with the price (price.go:166-173) and priority (priority.go:119-165) filters."""
    return _expander_chain("cae_expander_chain_ex", chain, node_count, pod_count, _opt(waste, np.float64),
                           _opt(price, np.float64), _opt(price_error, np.uint8), _opt(priority, np.int32))


def resolve_priorities(config: dict, group_ids: Sequence[str]) -> np.ndarray:
    """What the Go shim does for the priority expander: highest priority of the ConfigMap (priority -> regexp list) whose
    list matches the node group id (regexp.FindStringIndex = unanchored search), -1 when no entry matches
    (expander/priority/priority.go:137-150, groupIDMatchesList :171-178)."""
    import re
    out = np.full(len(group_ids), -1, np.int32)
    for i, gid in enumerate(group_ids):
        for prio, res in config.items():
            if any(re.search(r, gid) for r in res):
                out[i] = max(out[i], int(prio))
    return out


def unpack_bits(bits: np.ndarray, P: int) -> np.ndarray:
    """fit_bits [T][Pw] uint32 -> bool [T][P]."""
    b = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")
    return b[:, :P].astype(bool)
