"""String world -> interned columnar tables (``cae_objects``).

This is the Python twin of what the Go shim does once per autoscaler tick (INTEGRATION.md): walk
the snapshot's NodeInfos, the template NodeInfos and the pending pod groups, intern every string,
and lay the result out as the CSR tables ``include/caengine.h`` declares.  It evaluates no
predicate.  Two layers:

* :class:`TableBuilder` — integer-level, de-duplicating table construction (used directly by the
  synthetic generator for 10^5..10^6 pods);
* :class:`Encoder`      — interns ``objects.py`` dataclasses on top of it.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import capi
from .objects import (LABEL_HOSTNAME, TAINT_NODE_UNSCHEDULABLE, LabelSelector, Namespace, Node, NodeInfo, Pod,
                      PodEquivalenceGroup, Requirement)

MAX_RES = capi.CONST["CAE_MAX_RES"]

_OPS = {"In": 0, "Equals": 0, "=": 0, "==": 0, "NotIn": 1, "!=": 1, "Exists": 2,
        "DoesNotExist": 3, "Gt": 4, "Lt": 5}
_TOL_OPS = {"": 0, "Equal": 0, "Exists": 1, "Lt": 2, "Gt": 3}
_EFFECTS = {"": 0, "NoSchedule": 1, "PreferNoSchedule": 2, "NoExecute": 3}
_PROTOS = {"": 0, "TCP": 0, "UDP": 1, "SCTP": 2}
_POLICY = {"Ignore": 0, "Honor": 1}


class Unsupported(Exception):
    """Input the engine refuses (SURVEY §7 hard part 7): the caller must use the stock Go path."""


class _Interner:
    def __init__(self) -> None:
        self.ids: Dict[object, int] = {}
        self.items: List[object] = []

    def __call__(self, x) -> int:
        i = self.ids.get(x)
        if i is None:
            i = len(self.items)
            self.ids[x] = i
            self.items.append(x)
        return i

    def __len__(self) -> int:
        return len(self.items)


class _Csr:
    """A de-duplicating list-of-lists table; list 0 is the empty list."""

    def __init__(self, ncols: int) -> None:
        self.ncols = ncols
        self.ids: Dict[tuple, int] = {(): 0}
        self.off: List[int] = [0, 0]
        self.cols: List[List[int]] = [[] for _ in range(ncols)]

    def add(self, rows: Sequence[tuple], dedupe: bool = True) -> int:
        key = tuple(rows)
        if dedupe:
            i = self.ids.get(key)
            if i is not None:
                return i
        for r in rows:
            for c in range(self.ncols):
                self.cols[c].append(int(r[c]))
        self.off.append(self.off[-1] + len(rows))
        i = len(self.off) - 2
        if dedupe:
            self.ids[key] = i
        return i

    @property
    def n(self) -> int:
        return len(self.off) - 1


def _i32(x) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=np.int32)
    return a if a.size else np.zeros(1, np.int32)[:0].copy()


class TableBuilder:
    """Integer-level construction of every table of ``cae_objects``."""

    def __init__(self, num_res: int = 3) -> None:
        self.num_res = num_res
        self.hostname_key = -1
        self.unschedulable_taint_key = -1
        self.value_is_int: List[int] = []
        self.value_int: List[int] = []
        self.ns_labelset: List[int] = []
        self.ns_exists: List[int] = []
        self.labelsets = _Csr(2)
        self.reqs_key: List[int] = []
        self.reqs_op: List[int] = []
        self.reqs_val_off: List[int] = [0]
        self.reqs_vals: List[int] = []
        self.sel_ids: Dict[tuple, int] = {}
        self.sel_kind: List[int] = []
        self.sel_req_off: List[int] = [0]
        self.naff_ids: Dict[tuple, int] = {}
        self.naff_nodesel: List[int] = []
        self.naff_has_required: List[int] = []
        self.naff_term_off: List[int] = [0]
        self.term_expr_sel: List[int] = []
        self.term_field_off: List[int] = [0]
        self.field_op: List[int] = []
        self.field_node_name: List[int] = []
        self.tols = _Csr(4)
        self.taints = _Csr(3)
        self.ports = _Csr(3)
        self.pts = _Csr(6)
        # affinity lists: list of term ids; terms are rows with their own namespace CSR
        self.aff_ids: Dict[tuple, int] = {(): 0}
        self.aff_off: List[int] = [0, 0]
        self.aterm_selector: List[int] = []
        self.aterm_key: List[int] = []
        self.aterm_ns_off: List[int] = [0]
        self.aterm_ns: List[int] = []
        self.aterm_ns_selector: List[int] = []
        self.ps_ids: Dict[tuple, int] = {}
        self.ps_rows: List[tuple] = []
        # nodes
        self.node_rows: List[tuple] = []
        self.node_alloc: List[List[int]] = []
        self.node_pod_off: List[int] = [0]
        self.node_pod_spec: List[int] = []
        self.num_cluster_nodes = 0
        self.num_templates = 0
        # pending
        self.group_off: List[int] = [0]
        self.pend_spec_chunks: List[np.ndarray] = []
        self._nothing_sel = None

    # ---- dictionaries -------------------------------------------------------------------
    def declare_value(self, vid: int, text: Optional[str]) -> None:
        while len(self.value_is_int) <= vid:
            self.value_is_int.append(0)
            self.value_int.append(0)
        if text is not None:
            ok, v = _parse_int64(text)
            self.value_is_int[vid] = int(ok)
            self.value_int[vid] = v

    def declare_namespace(self, nsid: int, labelset: int = 0, exists: bool = False) -> None:
        while len(self.ns_labelset) <= nsid:
            self.ns_labelset.append(0)
            self.ns_exists.append(0)
        self.ns_labelset[nsid] = labelset
        self.ns_exists[nsid] = int(exists)

    # ---- tables ---------------------------------------------------------------------------
    def labelset(self, pairs: Iterable[Tuple[int, int]]) -> int:
        return self.labelsets.add(sorted(pairs))

    def selector(self, reqs: Optional[Sequence[Tuple[int, int, Tuple[int, ...]]]]) -> int:
        """reqs = None -> Nothing; [] -> Everything; else AND of (key, op, values)."""
        key = ("nothing",) if reqs is None else tuple((k, o, tuple(v)) for k, o, v in reqs)
        i = self.sel_ids.get(key)
        if i is not None:
            return i
        i = len(self.sel_kind)
        self.sel_ids[key] = i
        self.sel_kind.append(0 if reqs is None else 1)
        for k, o, vals in (reqs or []):
            self.reqs_key.append(k)
            self.reqs_op.append(o)
            self.reqs_vals.extend(vals)
            self.reqs_val_off.append(len(self.reqs_vals))
        self.sel_req_off.append(len(self.reqs_key))
        return i

    def nothing_selector(self) -> int:
        return self.selector(None)

    def node_affinity(self, nodesel: int, has_required: bool,
                      terms: Sequence[Tuple[int, Sequence[Tuple[int, int]]]]) -> int:
        """terms = [(expr_selector_or_-1, [(field_op, node_name_id), ...]), ...] (empty terms dropped)."""
        key = (nodesel, bool(has_required), tuple((e, tuple(f)) for e, f in terms))
        i = self.naff_ids.get(key)
        if i is not None:
            return i
        i = len(self.naff_nodesel)
        self.naff_ids[key] = i
        self.naff_nodesel.append(nodesel)
        self.naff_has_required.append(int(has_required))
        for e, fields in terms:
            self.term_expr_sel.append(e)
            for op, nm in fields:
                self.field_op.append(op)
                self.field_node_name.append(nm)
            self.term_field_off.append(len(self.field_op))
        self.naff_term_off.append(len(self.term_expr_sel))
        return i

    def toleration_list(self, tols: Sequence[Tuple[int, int, int, int]]) -> int:
        return self.tols.add(list(tols))

    def taint_list(self, taints: Sequence[Tuple[int, int, int]]) -> int:
        return self.taints.add(list(taints))

    def port_list(self, ports: Sequence[Tuple[int, int, int]]) -> int:
        return self.ports.add(list(ports))

    def pts_list(self, cons: Sequence[Tuple[int, int, int, int, int, int]]) -> int:
        """(max_skew, key, selector, min_domains, node_affinity_policy, node_taints_policy)"""
        return self.pts.add(list(cons))

    def affinity_list(self, terms: Sequence[Tuple[int, int, Tuple[int, ...], int]]) -> int:
        """terms = [(selector, topology_key, namespaces, ns_selector)]"""
        key = tuple((s, k, tuple(ns), nss) for s, k, ns, nss in terms)
        i = self.aff_ids.get(key)
        if i is not None:
            return i
        for s, k, ns, nss in terms:
            self.aterm_selector.append(s)
            self.aterm_key.append(k)
            self.aterm_ns.extend(ns)
            self.aterm_ns_off.append(len(self.aterm_ns))
            self.aterm_ns_selector.append(nss)
        self.aff_off.append(len(self.aterm_selector))
        i = len(self.aff_off) - 2
        self.aff_ids[key] = i
        return i

    def podspec(self, namespace: int, labelset: int, req: Sequence[int], tol_list: int = 0,
                naff: int = -1, node_name: int = -1, port_list: int = 0, pts_list: int = 0,
                aff_list: int = 0, anti_list: int = 0, terminating: bool = False,
                hostname_spread: Optional[bool] = None) -> int:
        req = tuple(int(x) for x in req) + (0,) * (MAX_RES - len(req))
        if hostname_spread is None:  # default: derived from the hard constraints
            hostname_spread = any(self.pts.cols[1][i] == self.hostname_key
                                  for i in range(self.pts.off[pts_list], self.pts.off[pts_list + 1]))
        key = (namespace, labelset, req, tol_list, naff, node_name, port_list, pts_list, aff_list,
               anti_list, bool(terminating), bool(hostname_spread))
        i = self.ps_ids.get(key)
        if i is None:
            i = len(self.ps_rows)
            self.ps_ids[key] = i
            self.ps_rows.append(key)
        return i

    def _node(self, name: int, labelset: int, taint_list: int, unschedulable: bool,
              alloc: Sequence[int], allowed_pods: int, cap_cpu: int, cap_mem: int,
              has_alloc_cpu: bool, has_alloc_mem: bool, pod_specs: Sequence[int]) -> int:
        self.node_rows.append((name, labelset, taint_list, int(unschedulable), allowed_pods, cap_cpu,
                               cap_mem, int(has_alloc_cpu), int(has_alloc_mem)))
        self.node_alloc.append(list(alloc) + [0] * (MAX_RES - len(alloc)))
        self.node_pod_spec.extend(pod_specs)
        self.node_pod_off.append(len(self.node_pod_spec))
        return len(self.node_rows) - 1

    def cluster_node(self, *a, **kw) -> int:
        if self.num_templates:
            raise ValueError("cluster nodes must be added before templates")
        self.num_cluster_nodes += 1
        return self._node(*a, **kw)

    def template(self, *a, **kw) -> int:
        self.num_templates += 1
        return self._node(*a, **kw) - self.num_cluster_nodes

    def group(self, spec_ids: Sequence[int]) -> int:
        arr = np.asarray(spec_ids, dtype=np.int32)
        self.pend_spec_chunks.append(arr)
        self.group_off.append(self.group_off[-1] + len(arr))
        return len(self.group_off) - 2

    # ---- finish ---------------------------------------------------------------------------
    def finish(self) -> "EncodedObjects":
        return EncodedObjects(self)


def _parse_int64(s: str) -> Tuple[bool, int]:
    """strconv.ParseInt(s, 10, 64): optional sign, decimal digits only (underscores not allowed with base 10)."""
    t = s
    if t[:1] in "+-":
        t = t[1:]
    if not t or not t.isascii() or not t.isdigit():
        return False, 0
    v = int(s)
    if v < -(1 << 63) or v > (1 << 63) - 1:
        return False, 0
    return True, v


# The dictionary tables of cae_objects that the deltas continue with tails (the engine states the same list in
# csrc/engine.h, CAE_DICT_TABLES): (ABI array, the count that sizes it, the child count an offsets array indexes,
# dtype, the builder storage behind it, the column of a row tuple or None).  An offsets array has count + 1 entries.
_DICT = tuple((nm, cnt, child, dt, get, col) for nm, cnt, child, dt, get, col in (
    ("value_is_int", "values", None, np.uint8, lambda b: b.value_is_int, None),
    ("value_int", "values", None, np.int64, lambda b: b.value_int, None),
    ("ns_labelset", "namespaces", None, np.int32, lambda b: b.ns_labelset, None),
    ("ns_exists", "namespaces", None, np.uint8, lambda b: b.ns_exists, None),
    ("ls_off", "labelsets", "pairs", np.int32, lambda b: b.labelsets.off, None),
    ("ls_key", "pairs", None, np.int32, lambda b: b.labelsets.cols[0], None),
    ("ls_val", "pairs", None, np.int32, lambda b: b.labelsets.cols[1], None),
    ("req_key", "reqs", None, np.int32, lambda b: b.reqs_key, None),
    ("req_op", "reqs", None, np.int32, lambda b: b.reqs_op, None),
    ("req_val_off", "reqs", "req_vals", np.int32, lambda b: b.reqs_val_off, None),
    ("req_vals", "req_vals", None, np.int32, lambda b: b.reqs_vals, None),
    ("sel_kind", "selectors", None, np.int32, lambda b: b.sel_kind, None),
    ("sel_req_off", "selectors", "reqs", np.int32, lambda b: b.sel_req_off, None),
    ("naff_nodesel", "naff", None, np.int32, lambda b: b.naff_nodesel, None),
    ("naff_has_required", "naff", None, np.uint8, lambda b: b.naff_has_required, None),
    ("naff_term_off", "naff", "naff_terms", np.int32, lambda b: b.naff_term_off, None),
    ("term_expr_sel", "naff_terms", None, np.int32, lambda b: b.term_expr_sel, None),
    ("term_field_off", "naff_terms", "fields", np.int32, lambda b: b.term_field_off, None),
    ("field_op", "fields", None, np.int32, lambda b: b.field_op, None),
    ("field_node_name", "fields", None, np.int32, lambda b: b.field_node_name, None),
    ("tol_off", "tol_lists", "tols", np.int32, lambda b: b.tols.off, None),
    ("tol_key", "tols", None, np.int32, lambda b: b.tols.cols[0], None),
    ("tol_op", "tols", None, np.int32, lambda b: b.tols.cols[1], None),
    ("tol_val", "tols", None, np.int32, lambda b: b.tols.cols[2], None),
    ("tol_effect", "tols", None, np.int32, lambda b: b.tols.cols[3], None),
    ("taint_off", "taint_lists", "taints", np.int32, lambda b: b.taints.off, None),
    ("taint_key", "taints", None, np.int32, lambda b: b.taints.cols[0], None),
    ("taint_val", "taints", None, np.int32, lambda b: b.taints.cols[1], None),
    ("taint_effect", "taints", None, np.int32, lambda b: b.taints.cols[2], None),
    ("port_off", "port_lists", "ports", np.int32, lambda b: b.ports.off, None),
    ("port_ip", "ports", None, np.int32, lambda b: b.ports.cols[0], None),
    ("port_proto", "ports", None, np.int32, lambda b: b.ports.cols[1], None),
    ("port_num", "ports", None, np.int32, lambda b: b.ports.cols[2], None),
    ("pts_off", "pts_lists", "pts", np.int32, lambda b: b.pts.off, None),
    ("pts_max_skew", "pts", None, np.int32, lambda b: b.pts.cols[0], None),
    ("pts_key", "pts", None, np.int32, lambda b: b.pts.cols[1], None),
    ("pts_selector", "pts", None, np.int32, lambda b: b.pts.cols[2], None),
    ("pts_min_domains", "pts", None, np.int32, lambda b: b.pts.cols[3], None),
    ("pts_node_affinity_policy", "pts", None, np.int32, lambda b: b.pts.cols[4], None),
    ("pts_node_taints_policy", "pts", None, np.int32, lambda b: b.pts.cols[5], None),
    ("aff_off", "aff_lists", "aterms", np.int32, lambda b: b.aff_off, None),
    ("aterm_selector", "aterms", None, np.int32, lambda b: b.aterm_selector, None),
    ("aterm_key", "aterms", None, np.int32, lambda b: b.aterm_key, None),
    ("aterm_ns_off", "aterms", "aterm_ns", np.int32, lambda b: b.aterm_ns_off, None),
    ("aterm_ns", "aterm_ns", None, np.int32, lambda b: b.aterm_ns, None),
    ("aterm_ns_selector", "aterms", None, np.int32, lambda b: b.aterm_ns_selector, None),
    ("ps_namespace", "specs", None, np.int32, lambda b: b.ps_rows, 0),
    ("ps_labelset", "specs", None, np.int32, lambda b: b.ps_rows, 1),
    ("ps_req", "specs", None, np.int64, lambda b: b.ps_rows, 2),
    ("ps_tol_list", "specs", None, np.int32, lambda b: b.ps_rows, 3),
    ("ps_naff", "specs", None, np.int32, lambda b: b.ps_rows, 4),
    ("ps_node_name", "specs", None, np.int32, lambda b: b.ps_rows, 5),
    ("ps_port_list", "specs", None, np.int32, lambda b: b.ps_rows, 6),
    ("ps_pts_list", "specs", None, np.int32, lambda b: b.ps_rows, 7),
    ("ps_aff_list", "specs", None, np.int32, lambda b: b.ps_rows, 8),
    ("ps_anti_list", "specs", None, np.int32, lambda b: b.ps_rows, 9),
    ("ps_terminating", "specs", None, np.uint8, lambda b: b.ps_rows, 10),
    ("ps_hostname_spread", "specs", None, np.uint8, lambda b: b.ps_rows, 11),
))
# cae_objects' field for each count it states; the other counts are the last offset of the offsets array that indexes them
_COUNT_FIELD = {"values": "num_values", "namespaces": "num_namespaces", "labelsets": "num_labelsets", "reqs": "num_reqs",
                "selectors": "num_selectors", "naff": "num_naff", "naff_terms": "num_naff_terms", "tol_lists": "num_tol_lists",
                "taint_lists": "num_taint_lists", "port_lists": "num_port_lists", "pts_lists": "num_pts_lists",
                "aff_lists": "num_aff_lists", "aterms": "num_aterms", "specs": "num_podspecs"}


def _dict_array(nm: str, dt, x) -> np.ndarray:
    if nm == "ps_req":
        return np.ascontiguousarray(np.asarray(x, np.int64).reshape(len(x), MAX_RES))
    return _i32(x) if dt is np.int32 else np.ascontiguousarray(x, dt)


def _cut(b: "TableBuilder", start: Dict[str, int], tables) -> Dict[str, np.ndarray]:
    """The dictionary tables `tables` of builder b from the entries `start` of each count on (offsets relative to the
    start of their child), as ABI arrays.  Costs what the cut holds, not the table."""
    out = {}
    for nm, cnt, child, dt, get, col in _DICT:
        if nm in tables:
            x = get(b)[start.get(cnt, 0):]
            if col is not None:
                x = [r[col] for r in x]
            if child is not None and start.get(child, 0):
                x = [o - start[child] for o in x]
            out[nm] = _dict_array(nm, dt, x)
    return out


def _dict_sizes(b: "TableBuilder", counts) -> Dict[str, int]:
    """The entries of each of `counts` in builder b."""
    return {cnt: len(get(b)) - (child is not None) for nm, cnt, child, dt, get, col in _DICT if cnt in counts}


def _dict_counts(s, a: Dict[str, np.ndarray]) -> Dict[str, int]:
    """The entries of every count in the tables of cae_objects `s` with arrays `a`."""
    n = {cnt: getattr(s, f) for cnt, f in _COUNT_FIELD.items()}
    for nm, cnt, child, *_ in _DICT:
        if child is not None and child not in _COUNT_FIELD:
            n[child] = int(a[nm][n[cnt]])
    return n


def _root_counts(a: Dict[str, np.ndarray]) -> Dict[str, int]:
    """cae_objects' count fields, from the lengths of the dictionary arrays `a`."""
    out = {}
    for nm, cnt, child, *_ in _DICT:
        if cnt in _COUNT_FIELD and _COUNT_FIELD[cnt] not in out:
            out[_COUNT_FIELD[cnt]] = len(a[nm]) - (child is not None)
    return out


def _table_names(struct_cls) -> set:
    """The dictionary tables a delta struct carries."""
    fields = {f for f, _ in struct_cls._fields_}
    return {nm for nm, *_ in _DICT if nm in fields}


def _families(tables) -> set:
    """The counts that size `tables`."""
    return {cnt for nm, cnt, *_ in _DICT if nm in tables}


_ALL_TABLES = {nm for nm, *_ in _DICT}
_NODE_TABLES = _table_names(capi.cae_node_delta)   # values, label sets, taint lists
_POD_TABLES = _table_names(capi.cae_pod_delta)     # every family but the taint lists


class EncodedObjects:
    """Owns the numpy arrays behind one ``cae_objects`` struct."""

    def __init__(self, b: TableBuilder) -> None:
        a: Dict[str, np.ndarray] = _cut(b, {}, _ALL_TABLES)
        for nm in ("value_is_int", "value_int", "ns_labelset", "ns_exists"):   # the value and namespace tables hold one entry at least
            if not len(a[nm]):
                a[nm] = np.zeros(1, a[nm].dtype)
        nn = len(b.node_rows)
        ncols = list(zip(*b.node_rows)) if nn else [[] for _ in range(9)]
        a["node_name"] = _i32(ncols[0])
        a["node_labelset"] = _i32(ncols[1])
        a["node_taint_list"] = _i32(ncols[2])
        a["node_unschedulable"] = np.asarray(ncols[3], dtype=np.uint8)
        a["node_allowed_pods"] = _i32(ncols[4])
        a["node_cap_cpu"] = np.asarray(ncols[5], dtype=np.int64)
        a["node_cap_mem"] = np.asarray(ncols[6], dtype=np.int64)
        a["node_has_alloc_cpu"] = np.asarray(ncols[7], dtype=np.uint8)
        a["node_has_alloc_mem"] = np.asarray(ncols[8], dtype=np.uint8)
        a["node_alloc"] = np.ascontiguousarray(np.asarray(b.node_alloc, dtype=np.int64).reshape(nn, MAX_RES))
        a["node_pod_off"] = _i32(b.node_pod_off)
        a["node_pod_spec"] = _i32(b.node_pod_spec)
        a["group_off"] = _i32(b.group_off)
        a["pend_spec"] = (np.ascontiguousarray(np.concatenate(b.pend_spec_chunks).astype(np.int32))
                          if b.pend_spec_chunks else np.zeros(0, np.int32))
        self.arrays = a
        s = capi.cae_objects()
        s.abi_version = capi.CONST["CAE_ABI_VERSION"]
        s.num_res = b.num_res
        s.hostname_key = b.hostname_key
        s.unschedulable_taint_key = b.unschedulable_taint_key
        for f, v in _root_counts(a).items():
            setattr(s, f, v)
        s.num_cluster_nodes = b.num_cluster_nodes
        s.num_templates = b.num_templates
        s.num_groups = len(b.group_off) - 1
        s.num_pending = int(b.group_off[-1])
        for name, ctype in capi.cae_objects._fields_:
            if name in a:
                arr = a[name]
                setattr(s, name, arr.ctypes.data_as(ctype))
        missing = [n for n, t in capi.cae_objects._fields_
                   if n not in a and hasattr(t, "contents")]
        if missing:
            raise RuntimeError("encoder does not fill ABI fields: %s" % missing)
        self.struct = s

    def slice_pods(self, p_begin: int, p_end: int) -> "EncodedObjects":
        """The same snapshot with only the pending pods [p_begin, p_end) (groups clipped to the range; every other table is
        shared): what rank r of a pod-sharded dense pass uploads (CAE_CFG_PODS_PRESHARDED)."""
        import copy
        out = copy.copy(self)
        out.arrays = dict(self.arrays)
        go = np.clip(self.arrays["group_off"], p_begin, p_end) - p_begin
        out.arrays["group_off"] = np.ascontiguousarray(go.astype(np.int32))
        out.arrays["pend_spec"] = np.ascontiguousarray(self.arrays["pend_spec"][p_begin:p_end])
        s = capi.cae_objects()
        C.memmove(C.byref(s), C.byref(self.struct), C.sizeof(s))
        s.num_pending = p_end - p_begin
        for name, ctype in capi.cae_objects._fields_:
            if name in ("group_off", "pend_spec"):
                setattr(s, name, out.arrays[name].ctypes.data_as(ctype))
        out.struct = s
        return out

    def with_pending(self, pend_spec, group_off) -> "EncodedObjects":
        """The same snapshot with other pending-pod rows (every other table is shared): what cae_load_pending uploads."""
        import copy
        out = copy.copy(self)
        out.arrays = dict(self.arrays)
        out.arrays["pend_spec"] = np.ascontiguousarray(pend_spec, np.int32)
        out.arrays["group_off"] = np.ascontiguousarray(group_off, np.int32)
        out.struct = self._restruct(out.arrays, num_pending=int(out.arrays["group_off"][-1]),
                                    num_groups=len(out.arrays["group_off"]) - 1)
        return out

    def apply_node_delta(self, delta: "NodeDelta") -> "EncodedObjects":
        """The objects after cae_load_nodes(delta), stated on the host: the dictionary tails appended, the dirty cluster
        rows rewritten and the resident-pod CSR rebuilt.  A cae_load of the result must answer like the engine after the
        delta."""
        import copy
        a, d = self._with_tails(delta.arrays, _NODE_TABLES), delta.arrays
        rows = d["row"]
        for nm, src in (("node_labelset", "labelset"), ("node_taint_list", "taint_list"),
                        ("node_unschedulable", "unschedulable"), ("node_allowed_pods", "allowed_pods")):
            a[nm] = a[nm].copy()
            a[nm][rows] = d[src]
        a["node_alloc"] = a["node_alloc"].copy()
        a["node_alloc"][rows] = d["alloc"]
        off, spec, po = a["node_pod_off"], a["node_pod_spec"], d["pod_off"]
        dirty = {int(r): i for i, r in enumerate(rows)}
        pieces, new_off = [], [0]
        for r in range(len(off) - 1):
            i = dirty.get(r)
            pieces.append(spec[off[r]:off[r + 1]] if i is None else d["pod_spec"][po[i]:po[i + 1]])
            new_off.append(new_off[-1] + len(pieces[-1]))
        a["node_pod_off"] = _i32(new_off)
        a["node_pod_spec"] = _i32(np.concatenate(pieces) if pieces else [])
        out = copy.copy(self)
        out.arrays = a
        out.struct = self._restruct(a, **_root_counts(a))
        return out

    def apply_node_churn(self, churn: "NodeChurn") -> "EncodedObjects":
        """The objects after cae_load_node_churn(churn), stated on the host: the tails and dirty rows of ``churn.changed``
        applied (row numbers before the call), then the removed rows dropped and the added rows appended after the
        surviving cluster rows, before the templates.  An added node has no capacity and no has_alloc_* (read for
        templates only).  A cae_load of the result must answer like the engine after the churn."""
        import copy
        out = self.apply_node_delta(churn.changed) if churn.changed is not None else self
        a, c = dict(out.arrays), churn.arrays
        N = out.struct.num_cluster_nodes
        na = len(c["name"])
        keep = np.setdiff1d(np.arange(N), c["removed"])
        zeros = {"node_cap_cpu": np.int64, "node_cap_mem": np.int64, "node_has_alloc_cpu": np.uint8, "node_has_alloc_mem": np.uint8}
        added = {"node_name": c["name"], "node_labelset": c["labelset"], "node_taint_list": c["taint_list"],
                 "node_unschedulable": c["unschedulable"], "node_allowed_pods": c["allowed_pods"], "node_alloc": c["alloc"]}
        for nm in list(added) + list(zeros):
            col = a[nm]
            new = added[nm] if nm in added else np.zeros(na, zeros[nm])
            a[nm] = np.ascontiguousarray(np.concatenate([col[keep], np.asarray(new, col.dtype).reshape((na,) + col.shape[1:]), col[N:]]))
        off, spec, po = a["node_pod_off"], a["node_pod_spec"], c["pod_off"]
        pieces = [spec[off[r]:off[r + 1]] for r in keep] + [c["pod_spec"][po[j]:po[j + 1]] for j in range(na)] + \
                 [spec[off[r]:off[r + 1]] for r in range(N, len(off) - 1)]
        a["node_pod_off"] = _i32(np.concatenate([[0], np.cumsum([len(p) for p in pieces], dtype=np.int64)]))
        a["node_pod_spec"] = _i32(np.concatenate(pieces) if pieces else [])
        res = copy.copy(out)
        res.arrays = a
        res.struct = out._restruct(a, num_cluster_nodes=len(keep) + na)
        return res

    def apply_pod_delta(self, delta: "PodDelta") -> "EncodedObjects":
        """The objects after cae_load_pods(delta), stated on the host: every dictionary tail and the new specs appended
        (tail offsets made absolute) and the pending list replaced.  A cae_load of the result must answer like the engine
        after the delta."""
        import copy
        a, d = self._with_tails(delta.arrays, _POD_TABLES), delta.arrays
        a["pend_spec"] = np.ascontiguousarray(d["pend_spec"], np.int32)
        a["group_off"] = np.ascontiguousarray(d["group_off"], np.int32)
        out = copy.copy(self)
        out.arrays = a
        out.struct = self._restruct(a, num_pending=len(a["pend_spec"]), num_groups=len(a["group_off"]) - 1, **_root_counts(a))
        return out

    def _with_tails(self, d: Dict[str, np.ndarray], tables) -> Dict[str, np.ndarray]:
        """A copy of the arrays with the tails `d` of the dictionary tables `tables` appended (tail offsets made absolute)."""
        a, n = dict(self.arrays), _dict_counts(self.struct, self.arrays)
        for nm, cnt, child, dt, *_ in _DICT:
            if nm in tables:
                tail = np.asarray(d[nm] if child is None else n[child] + d[nm][1:], dt)
                a[nm] = np.ascontiguousarray(np.concatenate([a[nm][:n[cnt] + (child is not None)], tail]).astype(dt))
        return a

    def _restruct(self, arrays, **counts) -> "capi.cae_objects":
        s = capi.cae_objects()
        C.memmove(C.byref(s), C.byref(self.struct), C.sizeof(s))
        for k, v in counts.items():
            setattr(s, k, v)
        for name, ctype in capi.cae_objects._fields_:
            if name in arrays:
                setattr(s, name, arrays[name].ctypes.data_as(ctype))
        return s

    # convenience
    @property
    def P(self) -> int:
        return self.struct.num_pending

    @property
    def T(self) -> int:
        return self.struct.num_templates

    @property
    def E(self) -> int:
        return self.struct.num_groups

    def ptr(self):
        return C.byref(self.struct)


class NodeDelta:
    """Owns the numpy arrays behind one ``cae_node_delta`` struct: the dictionary tails (values, label sets, taint lists
    that continue the resident tables; offsets relative to the tail) and the complete new state of the dirty cluster
    rows.  Field names are the header's."""

    _I32 = ("ls_off", "ls_key", "ls_val", "taint_off", "taint_key", "taint_val", "taint_effect", "row", "labelset",
            "taint_list", "allowed_pods", "pod_off", "pod_spec")

    def __init__(self, **arrays) -> None:
        a: Dict[str, np.ndarray] = {}
        for nm in self._I32:
            a[nm] = _i32(arrays.get(nm, [0] if nm in ("ls_off", "taint_off", "pod_off") else []))
        a["value_is_int"] = np.ascontiguousarray(arrays.get("value_is_int", []), np.uint8)
        a["value_int"] = np.ascontiguousarray(arrays.get("value_int", []), np.int64)
        a["unschedulable"] = np.ascontiguousarray(arrays.get("unschedulable", []), np.uint8)
        nd = len(a["row"])
        a["alloc"] = np.ascontiguousarray(np.asarray(arrays.get("alloc", np.zeros((nd, MAX_RES))), np.int64).reshape(nd, MAX_RES))
        self.arrays = a
        s = capi.cae_node_delta()
        s.abi_version = capi.CONST["CAE_ABI_VERSION"]
        s.num_new_values = len(a["value_is_int"])
        s.num_new_labelsets = len(a["ls_off"]) - 1
        s.num_new_taint_lists = len(a["taint_off"]) - 1
        s.num_dirty = nd
        for name, ctype in capi.cae_node_delta._fields_:
            if name in a:
                setattr(s, name, a[name].ctypes.data_as(ctype))
        self.struct = s

    def replace(self, **arrays) -> "NodeDelta":
        """A copy with some arrays replaced (the counts follow the arrays)."""
        return NodeDelta(**{**self.arrays, **arrays})

    @property
    def num_dirty(self) -> int:
        return self.struct.num_dirty

    def ptr(self):
        return C.byref(self.struct)


class NodeChurn:
    """Owns the numpy arrays behind one ``cae_node_churn`` struct: ``changed`` (a NodeDelta with the dirty rows and the
    dictionary tails the dirty and the added rows use, or None), the removed rows and the added nodes.  Field names are
    the header's."""

    _I32 = ("removed", "name", "labelset", "taint_list", "allowed_pods", "pod_off", "pod_spec")

    def __init__(self, changed: Optional[NodeDelta] = None, **arrays) -> None:
        a: Dict[str, np.ndarray] = {}
        for nm in self._I32:
            a[nm] = _i32(arrays.get(nm, [0] if nm == "pod_off" else []))
        a["unschedulable"] = np.ascontiguousarray(arrays.get("unschedulable", np.zeros(len(a["name"]))), np.uint8)
        na = len(a["name"])
        a["alloc"] = np.ascontiguousarray(np.asarray(arrays.get("alloc", np.zeros((na, MAX_RES))), np.int64).reshape(na, MAX_RES))
        self.arrays = a
        self.changed = changed
        s = capi.cae_node_churn()
        s.abi_version = capi.CONST["CAE_ABI_VERSION"]
        s.changed = C.pointer(changed.struct) if changed is not None else None
        s.num_removed = len(a["removed"])
        s.num_added = na
        for name, ctype in capi.cae_node_churn._fields_:
            if name in a:
                setattr(s, name, a[name].ctypes.data_as(ctype))
        self.struct = s

    def replace(self, **arrays) -> "NodeChurn":
        """A copy with some arrays (or ``changed``) replaced (the counts follow the arrays)."""
        changed = arrays.pop("changed", self.changed)
        return NodeChurn(changed, **{**self.arrays, **arrays})

    @property
    def num_removed(self) -> int:
        return self.struct.num_removed

    @property
    def num_added(self) -> int:
        return self.struct.num_added

    def ptr(self):
        return C.byref(self.struct)


class PodDelta:
    """Owns the numpy arrays behind one ``cae_pod_delta`` struct: the dictionary tails and new pod specs (continuing the
    resident tables; offsets relative to the tail) and the complete new pending list.  Field names are the header's."""

    # count field -> the array whose length gives it (minus one for an offsets array)
    _COUNTS = {"num_new_values": "value_is_int", "num_new_namespaces": "ns_labelset", "num_new_labelsets": "ls_off",
               "num_new_reqs": "req_key", "num_new_selectors": "sel_kind", "num_new_naff": "naff_nodesel",
               "num_new_naff_terms": "term_expr_sel", "num_new_tol_lists": "tol_off", "num_new_port_lists": "port_off",
               "num_new_pts_lists": "pts_off", "num_new_aff_lists": "aff_off", "num_new_aterms": "aterm_selector",
               "num_new_specs": "ps_namespace", "num_groups": "group_off", "num_pending": "pend_spec"}
    _OFFSETS = ("ls_off", "req_val_off", "sel_req_off", "naff_term_off", "term_field_off", "tol_off", "port_off", "pts_off",
                "aff_off", "aterm_ns_off", "group_off")

    def __init__(self, **arrays) -> None:
        a: Dict[str, np.ndarray] = {}
        for name, ctype in capi.cae_pod_delta._fields_:
            if not hasattr(ctype, "contents"):
                continue
            dt = {C.c_uint8: np.uint8, C.c_int64: np.int64}.get(ctype._type_, np.int32)
            a[name] = np.ascontiguousarray(arrays.get(name, [0] if name in self._OFFSETS else []), dt)
        a["ps_req"] = np.ascontiguousarray(a["ps_req"].reshape(len(a["ps_namespace"]), MAX_RES))
        self.arrays = a
        s = capi.cae_pod_delta()
        s.abi_version = capi.CONST["CAE_ABI_VERSION"]
        for cnt, nm in self._COUNTS.items():
            setattr(s, cnt, len(a[nm]) - (nm in self._OFFSETS))
        for name, ctype in capi.cae_pod_delta._fields_:
            if name in a:
                setattr(s, name, a[name].ctypes.data_as(ctype))
        self.struct = s

    def replace(self, **arrays) -> "PodDelta":
        """A copy with some arrays replaced (the counts follow the arrays)."""
        return PodDelta(**{**self.arrays, **arrays})

    @property
    def num_new_specs(self) -> int:
        return self.struct.num_new_specs

    def ptr(self):
        return C.byref(self.struct)


# ----------------------------------------------------------------------------------------------
class Encoder:
    """Interns objects.py dataclasses into a TableBuilder (the Go shim's job in production)."""

    FIXED_RES = {"cpu": 0, "memory": 1, "ephemeral-storage": 2}

    def __init__(self) -> None:
        self.keys = _Interner()
        self.values = _Interner()
        self.namespaces = _Interner()
        self.node_names = _Interner()
        self.ips = _Interner()
        self.ips("0.0.0.0")
        self.resources = _Interner()
        for r in ("cpu", "memory", "ephemeral-storage"):
            self.resources(r)
        self.b = TableBuilder()
        self._podspec_cache: Dict[int, int] = {}
        self._ns_objects: Dict[str, Namespace] = {}

    # ---- interning helpers --------------------------------------------------------------
    def _val(self, v: str) -> int:
        n = len(self.values)
        i = self.values(v)
        if i == n:
            self.b.declare_value(i, v)
        return i

    def _key(self, k: str) -> int:
        i = self.keys(k)
        if k == LABEL_HOSTNAME:
            self.b.hostname_key = i
        elif k == TAINT_NODE_UNSCHEDULABLE:
            self.b.unschedulable_taint_key = i
        return i

    def _ns(self, ns: str) -> int:
        n = len(self.namespaces)
        i = self.namespaces(ns)
        if i == n:
            obj = self._ns_objects.get(ns)
            if obj is not None:
                self.b.declare_namespace(i, self._labelset(obj.labels), True)
            else:
                self.b.declare_namespace(i, 0, False)
        return i

    def _labelset(self, labels: Dict[str, str]) -> int:
        return self.b.labelset((self._key(k), self._val(v)) for k, v in labels.items())

    def _selector(self, sel: Optional[LabelSelector], extra: Optional[Dict[str, str]] = None) -> int:
        """metav1.LabelSelectorAsSelector; `extra` = matchLabelKeys merge (common.go:96-106,131-143)."""
        if sel is None:
            # mergeLabelSetWithSelector on Nothing: Requirements() of Nothing is not ok -> returns s
            return self.b.nothing_selector()
        reqs: List[Tuple[int, int, Tuple[int, ...]]] = []
        for k, v in sorted((extra or {}).items()):
            reqs.append((self._key(k), 0, (self._val(v),)))
        for k, v in sorted(sel.match_labels.items()):
            reqs.append((self._key(k), 0, (self._val(v),)))
        for r in sel.match_expressions:
            reqs.append(self._req(r))
        return self.b.selector(reqs)

    def _req(self, r: Requirement) -> Tuple[int, int, Tuple[int, ...]]:
        if r.operator not in _OPS:
            raise Unsupported("selector operator %r" % r.operator)
        return (self._key(r.key), _OPS[r.operator], tuple(self._val(v) for v in r.values))

    def _resource_vec(self, rl: Dict[str, int]) -> List[int]:
        vec = [0] * MAX_RES
        for name, amt in rl.items():
            if name == "pods":
                continue
            i = self.resources(name)
            if i >= MAX_RES:
                raise Unsupported("more than %d resource dimensions" % MAX_RES)
            vec[i] = int(amt)
        self.b.num_res = max(self.b.num_res, len(self.resources))
        return vec

    # ---- objects --------------------------------------------------------------------------
    def add_namespace(self, ns: Namespace) -> None:
        self._ns_objects[ns.name] = ns
        if ns.name in self.namespaces.ids:
            self.b.declare_namespace(self.namespaces.ids[ns.name], self._labelset(ns.labels), True)

    def podspec(self, pod: Pod, resident: bool = False) -> int:
        """resident: a pod already running on a cluster node.  The volume / DRA filters (VolumeRestrictions, VolumeBinding,
        VolumeZone, NodeVolumeLimits, DynamicResources) only ever reject an INCOMING pod that carries volumes or claims, so
        residents with volumes are harmless as long as no pending (or template DaemonSet) pod has any — those are refused."""
        if pod.has_volumes_or_claims and not resident:
            raise Unsupported("pod %s/%s uses volumes or resource claims" % (pod.namespace, pod.name))
        cached = self._podspec_cache.get(id(pod))
        if cached is not None:
            return cached
        b = self.b
        ns = self._ns(pod.namespace)
        tols = b.toleration_list([
            (self._key(t.key) if t.key else -1, _TOL_OPS.get(t.operator, 4),
             self._val(t.value) if t.value else -1, _EFFECTS[t.effect]) for t in pod.tolerations])
        naff = -1
        if pod.node_selector or pod.node_affinity_terms is not None:
            nodesel = -1
            if pod.node_selector:
                nodesel = b.selector([(self._key(k), 0, (self._val(v),))
                                      for k, v in sorted(pod.node_selector.items())])
            terms = []
            for t in (pod.node_affinity_terms or []):
                # empty terms are kept: they select nothing in Filter (nodeaffinity.go:60-66) but make
                # NodeAffinity.PreFilter return "all nodes" (node_affinity.go:176-196)
                expr = -1
                if t.match_expressions:
                    expr = b.selector([self._req(r) for r in t.match_expressions])
                flds = []
                for f in t.match_fields:
                    if f.key != "metadata.name" or f.operator not in ("In", "NotIn") or len(f.values) != 1:
                        raise Unsupported("matchFields other than metadata.name In/NotIn [one value]")
                    flds.append((_OPS[f.operator], self.node_names(f.values[0])))
                terms.append((expr, flds))
            naff = b.node_affinity(nodesel, pod.node_affinity_terms is not None, terms)
        ports = b.port_list([(self.ips(p.host_ip or "0.0.0.0"), _PROTOS[p.protocol], p.host_port)
                             for p in pod.host_ports if p.host_port > 0])
        cons = []
        for c in pod.topology_spread:
            if c.when_unsatisfiable != "DoNotSchedule":
                continue  # plugin.go:273-296 keeps only the hard constraints
            extra = {k: pod.labels[k] for k in c.match_label_keys if k in pod.labels}
            cons.append((c.max_skew, self._key(c.topology_key), self._selector(c.label_selector, extra),
                         1 if c.min_domains is None else c.min_domains,
                         _POLICY[c.node_affinity_policy or "Honor"],
                         _POLICY[c.node_taints_policy or "Ignore"]))
        pts = b.pts_list(cons)

        def aff(terms) -> int:
            rows = []
            for t in terms:
                nss = list(t.namespaces)
                if not nss and t.namespace_selector is None:
                    nss = [pod.namespace]  # types.go:436-444
                rows.append((self._selector(t.label_selector), self._key(t.topology_key),
                             tuple(sorted(self._ns(n) for n in nss)),
                             self._selector(t.namespace_selector)))
            return b.affinity_list(rows)

        sid = b.podspec(ns, self._labelset(pod.labels), self._resource_vec(pod.requests), tols, naff,
                        self.node_names(pod.node_name) if pod.node_name else -1, ports, pts,
                        aff(pod.pod_affinity), aff(pod.pod_anti_affinity), pod.terminating,
                        any(c.topology_key == LABEL_HOSTNAME for c in pod.topology_spread))
        self._podspec_cache[id(pod)] = sid
        return sid

    def _node_args(self, ni: NodeInfo, resident: bool = False):
        n = ni.node
        taints = self.b.taint_list([(self._key(t.key), self._val(t.value) if t.value else -1,
                                     _EFFECTS[t.effect]) for t in n.taints])
        return dict(name=self.node_names(n.name), labelset=self._labelset(n.labels), taint_list=taints,
                    unschedulable=n.unschedulable, alloc=self._resource_vec(n.allocatable),
                    allowed_pods=int(n.allocatable.get("pods", 0)),
                    cap_cpu=int(n.capacity.get("cpu", 0)), cap_mem=int(n.capacity.get("memory", 0)),
                    has_alloc_cpu="cpu" in n.allocatable, has_alloc_mem="memory" in n.allocatable,
                    pod_specs=[self.podspec(p, resident) for p in ni.pods])

    def add_cluster_node(self, ni: NodeInfo) -> int:
        return self.b.cluster_node(**self._node_args(ni, resident=True))

    def add_template(self, ni: NodeInfo) -> int:
        return self.b.template(**self._node_args(ni))

    def add_group(self, g: PodEquivalenceGroup) -> int:
        return self.b.group([self.podspec(p) for p in g.pods])

    # ---- inputs of cae_similar_node_groups ------------------------------------------------------
    def similarity_signatures(self, templates: Sequence[NodeInfo]) -> Tuple[np.ndarray, np.ndarray]:
        """(res_sig [T] int32, free_dims [T] uint32) of the encoded templates, in their order.  res_sig interns what the
        comparator (compare_nodegroups.go:104-163) compares exactly: the Allocatable key set, the key set of
        ResourceToResourceList(Requested) (cpu, memory, pods, ephemeral-storage always, plus every resource a pod of the
        template requests) and the Capacity map with memory's value left out.  free_dims: bit r = dim r is such a key."""
        sigs: Dict[tuple, int] = {}
        res_sig = np.zeros(len(templates), np.int32)
        free_dims = np.zeros(len(templates), np.uint32)
        for t, ni in enumerate(templates):
            requested = {"cpu", "memory", "pods", "ephemeral-storage"}
            for p in ni.pods:
                requested.update(p.requests)
            cap = tuple(sorted((k, None if k == "memory" else int(v)) for k, v in ni.node.capacity.items()))
            key = (frozenset(ni.node.allocatable), frozenset(requested), cap)
            res_sig[t] = sigs.setdefault(key, len(sigs))
            free_dims[t] = sum(1 << self.resources.ids[r] for r in requested if r != "pods")
        return res_sig, free_dims

    def label_key_ids(self, keys: Iterable[str]) -> np.ndarray:
        """Key ids of label keys; a key the interner never saw is on no template and is left out."""
        return np.asarray(sorted({self.keys.ids[k] for k in keys if k in self.keys.ids}), np.int32)

    def finish(self) -> EncodedObjects:
        self._key(LABEL_HOSTNAME)
        self._key(TAINT_NODE_UNSCHEDULABLE)
        self.b.num_res = max(3, len(self.resources))
        enc = self.b.finish()
        # what the engine holds after a load of `enc`, per count: node_delta() / pod_delta() emit what the interner adds
        # beyond it as tails (the value and namespace tables of a load may be padded)
        self._emitted = _dict_counts(enc.struct, enc.arrays)
        self._num_res = enc.struct.num_res
        self._delta_ok = True
        self._spec_wo_name: Optional[Dict[tuple, int]] = None
        # the cluster rows the engine holds: (node-name id, row state) per row, kept current by node_delta / node_churn
        b, off = self.b, self.b.node_pod_off
        self._cluster = [(b.node_rows[r][0], (b.node_rows[r][1], b.node_rows[r][2], b.node_rows[r][3], tuple(b.node_alloc[r]),
                                              b.node_rows[r][4], tuple(b.node_pod_spec[off[r]:off[r + 1]])))
                         for r in range(b.num_cluster_nodes)]
        return enc

    def _resident_spec(self, pod: Pod, allow_new: bool = False) -> int:
        """Spec id of a resident pod of a changed node, among the specs of the last load.  No filter reads a resident pod's
        spec.nodeName (only the incoming pod's), so the lookup ignores it: a pod bound since the last tick finds its
        pending spec.  No match: Unsupported (the tick needs a full load), or with `allow_new` (pod_delta) a new spec."""
        b = self.b
        n = len(b.ps_rows)
        saved, self._podspec_cache = self._podspec_cache, {}
        try:
            sid = self.podspec(pod, resident=True)
        finally:
            self._podspec_cache = saved
        if sid < n:
            return sid
        key = b.ps_rows.pop()           # the interner added a row: take it back and look for the same spec without nodeName
        del b.ps_ids[key]
        hit = b.ps_ids.get(key[:5] + (-1,) + key[6:])
        if hit is None and allow_new:   # the first pod of a new spec: keep the row
            b.ps_ids[key] = sid
            b.ps_rows.append(key)
            self._spec_wo_name = None
            return sid
        if hit is None:
            if self._spec_wo_name is None:
                self._spec_wo_name = {}
                for i, k in enumerate(b.ps_rows):
                    self._spec_wo_name.setdefault(k[:5] + k[6:], i)
            hit = self._spec_wo_name.get(key[:5] + key[6:])
        if hit is None:
            self._delta_ok = False
            raise Unsupported("resident pod %s/%s has a spec the last load did not have" % (pod.namespace, pod.name))
        return hit

    def node_delta(self, changed: Sequence[Tuple[int, NodeInfo]]) -> NodeDelta:
        """The shim's side of cae_load_nodes: the new state of changed cluster nodes (row of the last load, NodeInfo) as a
        NodeDelta against what the engine holds.  The interner stays append-only; the values, label sets and taint lists
        the changed rows add since the last load or delta become the delta's tails.  Unsupported = use a full load (and
        a fresh Encoder: this one no longer matches the engine)."""
        self._check_resident()
        items = sorted(changed, key=lambda x: x[0])
        rows: List[int] = []
        states = []
        for row, ni in items:
            if not 0 <= row < len(self._cluster) or (rows and row == rows[-1]):
                raise ValueError("node delta row %d: not a cluster node of the last load, or given twice" % row)
            if self.node_names.ids.get(ni.node.name) != self._cluster[row][0]:
                self._delta_ok = False
                raise Unsupported("row %d is no longer node %s" % (row, ni.node.name))
            rows.append(row)
            states.append(self._row_state(ni))
        delta = self._tails_and_rows(rows, states)
        for row, st in zip(rows, states):
            self._cluster[row] = (self._cluster[row][0], st)
        return delta

    def _check_resident(self) -> None:
        """Unsupported unless the interner still matches what the engine holds."""
        if not getattr(self, "_delta_ok", False):
            raise Unsupported("no load to apply a node delta to, or an earlier delta was refused")
        if len(self.b.value_is_int) < self._emitted["values"]:
            self._delta_ok = False
            raise Unsupported("the value table of the last load was padded")

    def _row_state(self, ni: NodeInfo) -> tuple:
        """(label set, taint list, unschedulable, allocatable, allowed pods, resident specs) of a cluster node, interned
        append-only against the last load."""
        n, b = ni.node, self.b
        nres = len(self.resources)
        tl = b.taint_list([(self._key(t.key), self._val(t.value) if t.value else -1, _EFFECTS[t.effect]) for t in n.taints])
        ls = self._labelset(n.labels)
        vec = self._resource_vec(n.allocatable)
        if len(self.resources) > nres:
            self._delta_ok = False
            raise Unsupported("node %s has a resource the last load did not have" % n.name)
        specs = tuple(self._resident_spec(p) for p in ni.pods)
        return (ls, tl, int(n.unschedulable), tuple(vec), int(n.allocatable.get("pods", 0)), specs)

    def _tails_and_rows(self, rows: Sequence[int], states: Sequence[tuple]) -> NodeDelta:
        """The NodeDelta of dirty rows `rows` with row states `states`, carrying as tails what the interner added since the
        last load or delta."""
        pod_off, pod_spec = [0], []
        for st in states:
            pod_spec.extend(st[5])
            pod_off.append(len(pod_spec))
        delta = NodeDelta(
            **self._tails(_NODE_TABLES), row=rows, labelset=[st[0] for st in states], taint_list=[st[1] for st in states],
            unschedulable=[st[2] for st in states], alloc=np.asarray([st[3] for st in states], np.int64).reshape(len(rows), MAX_RES),
            allowed_pods=[st[4] for st in states], pod_off=pod_off, pod_spec=pod_spec)
        return delta

    def _tails(self, tables) -> Dict[str, np.ndarray]:
        """The tails of the dictionary tables `tables`: what the interner added since they were last emitted.  Their
        families are emitted and advance."""
        counts = _families(tables)
        out = _cut(self.b, self._emitted, tables)
        self._emitted.update(_dict_sizes(self.b, counts))
        return out

    def node_churn(self, new_cluster: Sequence[NodeInfo]) -> "NodeChurn":
        """The shim's side of cae_load_node_churn: the complete new cluster-node list as a NodeChurn against what the engine
        holds.  Nodes are matched by name: names that are gone are removed, new names are added, survivors whose state
        changed become dirty rows.  The survivors must keep their relative order and the new nodes must all come after
        them (Unsupported otherwise: a full load).  Resident specs are found as for node_delta."""
        self._check_resident()
        old = {nid: r for r, (nid, _) in enumerate(self._cluster)}
        names = [ni.node.name for ni in new_cluster]
        if len(set(names)) != len(names):
            raise ValueError("node churn: a node name is given twice")
        last, seen_new = -1, False
        for nm in names:
            r = old.get(self.node_names.ids.get(nm, -1))
            if r is None:
                seen_new = True
            elif seen_new or r < last:
                raise Unsupported("node churn: the surviving nodes are reordered or a new node comes before one of them")
            else:
                last = r
        kept = {old[self.node_names.ids[nm]] for nm in names if self.node_names.ids.get(nm, -1) in old}
        removed = [r for r in range(len(self._cluster)) if r not in kept]
        rows, dirty_states, new_list, added = [], [], [], []
        for ni in new_cluster:
            st = self._row_state(ni)
            r = old.get(self.node_names.ids.get(ni.node.name, -1))
            if r is None:
                nid = self.node_names(ni.node.name)
                added.append((nid, st))
                continue
            if st != self._cluster[r][1]:
                rows.append(r)
                dirty_states.append(st)
            new_list.append((self._cluster[r][0], st))
        changed = self._tails_and_rows(rows, dirty_states)
        po = [0]
        for _, st in added:
            po.append(po[-1] + len(st[5]))
        churn = NodeChurn(changed, removed=removed, name=[nid for nid, _ in added], labelset=[st[0] for _, st in added],
                          taint_list=[st[1] for _, st in added], unschedulable=[st[2] for _, st in added],
                          alloc=np.asarray([st[3] for _, st in added], np.int64).reshape(len(added), MAX_RES),
                          allowed_pods=[st[4] for _, st in added], pod_off=po, pod_spec=[x for _, st in added for x in st[5]])
        self._cluster = new_list + added
        return churn

    def pod_delta(self, groups: Sequence[PodEquivalenceGroup], residents: Sequence[NodeInfo] = ()) -> "PodDelta":
        """The shim's side of cae_load_pods: `groups` become the complete new pending list, and every spec and dictionary
        entry interned since the last load or delta becomes a tail.  The pods of `residents` (the changed or added nodes
        of this tick) are interned first, so that the node_delta / node_churn that follows finds their specs; the tick
        is load_pods, then the node call.  Unsupported: a resource dimension the last load did not have (a full load)."""
        self._check_resident()
        for ni in residents:
            for p in ni.pods:
                self._resident_spec(p, allow_new=True)
        pend, off = [], [0]
        for g in groups:
            pend.extend(self.podspec(p) for p in g.pods)
            off.append(len(pend))
        if len(self.resources) > self._num_res:
            self._delta_ok = False
            raise Unsupported("a pod requests a resource the last load did not have")
        if len(self.b.ns_labelset) < self._emitted["namespaces"]:
            self._delta_ok = False
            raise Unsupported("the namespace table of the last load was padded")
        return PodDelta(**self._tails(_POD_TABLES), group_off=off, pend_spec=pend)


def encode(cluster: Sequence[NodeInfo], templates: Sequence[NodeInfo],
           groups: Sequence[PodEquivalenceGroup],
           namespaces: Sequence[Namespace] = (), encoder: Optional[Encoder] = None) -> EncodedObjects:
    """encoder: the Encoder to intern with (a fresh one by default), for a caller that needs its dictionaries afterwards."""
    enc = encoder or Encoder()
    for ns in namespaces:
        enc.add_namespace(ns)
    for ni in cluster:
        enc.add_cluster_node(ni)
    for ni in templates:
        enc.add_template(ni)
    for g in groups:
        enc.add_group(g)
    return enc.finish()
