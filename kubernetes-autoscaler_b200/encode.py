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
        _fill_pointers(s, a)
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
        out.struct = self._restruct(out.arrays, num_pending=p_end - p_begin)
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

    def apply_upcoming(self, up: "UpcomingNodes") -> "EncodedObjects":
        """The objects after cae_add_upcoming_nodes(up), stated on the host: ``up.churn`` applied as apply_node_churn does,
        then the copies appended after the cluster rows, before the templates.  A copy has its template's columns and
        resident pods, its own node name and label set, and no capacity or has_alloc_*.  A cae_load of the result must
        answer like the engine after the call."""
        import copy
        out = self.apply_node_churn(up.churn) if up.churn is not None else self
        a, u = dict(out.arrays), up.arrays
        N = out.struct.num_cluster_nodes
        tr = N + np.asarray(u["template_idx"], np.int64)    # the template rows the copies are made from
        nu = len(tr)
        cols = {"node_name": u["name"], "node_labelset": u["labelset"], "node_cap_cpu": np.zeros(nu), "node_cap_mem": np.zeros(nu),
                "node_has_alloc_cpu": np.zeros(nu), "node_has_alloc_mem": np.zeros(nu)}
        for nm in ("node_name", "node_labelset", "node_taint_list", "node_unschedulable", "node_allowed_pods", "node_alloc",
                   "node_cap_cpu", "node_cap_mem", "node_has_alloc_cpu", "node_has_alloc_mem"):
            col = a[nm]
            new = np.asarray(cols[nm], col.dtype) if nm in cols else col[tr]
            a[nm] = np.ascontiguousarray(np.concatenate([col[:N], new.reshape((nu,) + col.shape[1:]), col[N:]]))
        off, spec = a["node_pod_off"], a["node_pod_spec"]
        rows = list(range(N)) + tr.tolist() + list(range(N, len(off) - 1))
        pieces = [spec[off[r]:off[r + 1]] for r in rows]
        a["node_pod_off"] = _i32(np.concatenate([[0], np.cumsum([len(p) for p in pieces], dtype=np.int64)]))
        a["node_pod_spec"] = _i32(np.concatenate(pieces) if pieces else [])
        res = copy.copy(out)
        res.arrays = a
        res.struct = out._restruct(a, num_cluster_nodes=N + nu)
        return res

    def apply_template_delta(self, delta: "TemplateDelta") -> "EncodedObjects":
        """The objects after cae_load_templates(delta), stated on the host: the tails of ``delta.tails`` appended, then the
        template rows rebuilt: the surviving templates in their old order (a changed one replaced by its staged row in
        place), then the added ones.  A cae_load of the result must answer like the engine after the delta."""
        import copy
        out = self.apply_node_delta(delta.tails) if delta.tails is not None else self
        a, d = dict(out.arrays), delta.arrays
        N, T = out.struct.num_cluster_nodes, out.struct.num_templates
        removed = set(d["removed"].tolist())
        changed = {int(t): i for i, t in enumerate(d["changed"])}
        src = []                                      # per new template: ("old", row) or ("new", staged row)
        for t in range(T):
            if t in removed:
                continue
            src.append(("new", changed[t]) if t in changed else ("old", N + t))
        src += [("new", len(changed) + j) for j in range(delta.num_added)]
        staged = {"node_name": d["name"], "node_labelset": d["labelset"], "node_taint_list": d["taint_list"],
                  "node_unschedulable": d["unschedulable"], "node_allowed_pods": d["allowed_pods"], "node_alloc": d["alloc"],
                  "node_cap_cpu": d["cap_cpu"], "node_cap_mem": d["cap_mem"], "node_has_alloc_cpu": d["has_alloc_cpu"],
                  "node_has_alloc_mem": d["has_alloc_mem"]}
        for nm, new in staged.items():
            col = a[nm]
            rows = [col[r] if kind == "old" else np.asarray(new[r], col.dtype) for kind, r in src]
            tail = np.asarray(rows, col.dtype).reshape((len(src),) + col.shape[1:])
            a[nm] = np.ascontiguousarray(np.concatenate([col[:N], tail]))
        off, spec, po = a["node_pod_off"], a["node_pod_spec"], d["pod_off"]
        pieces = [spec[off[r]:off[r + 1]] for r in range(N)] + \
                 [spec[off[r]:off[r + 1]] if kind == "old" else d["pod_spec"][po[r]:po[r + 1]] for kind, r in src]
        a["node_pod_off"] = _i32(np.concatenate([[0], np.cumsum([len(p) for p in pieces], dtype=np.int64)]))
        a["node_pod_spec"] = _i32(np.concatenate(pieces) if pieces else [])
        res = copy.copy(out)
        res.arrays = a
        res.struct = out._restruct(a, num_templates=len(src))
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

    def apply_force_add(self, pods, nodes) -> Tuple["EncodedObjects", np.ndarray]:
        """The objects after cae_force_add_pods(pods, nodes), stated on the host, and the new_index map: pending pod
        pods[i] is appended to the resident pods of cluster row nodes[i] in list order (its spec id unchanged) and leaves
        the pending list; the other pods keep their order and groups, so a group may become empty.  new_index [P] is
        each pod's index afterwards, -1 for a moved one.  A cae_load of the result must answer like the engine after
        the call.  ValueError: what the engine answers with status -2."""
        import copy
        pods, nodes = np.asarray(pods, np.int64).reshape(-1), np.asarray(nodes, np.int64).reshape(-1)
        P, N = self.P, self.struct.num_cluster_nodes
        if len(pods) != len(nodes):
            raise ValueError("force add: pods and nodes differ in length")
        if len(pods) and (pods.min() < 0 or pods.max() >= P or len(np.unique(pods)) != len(pods)):
            raise ValueError("force add: a pod index is out of range or listed twice")
        if len(nodes) and (nodes.min() < 0 or nodes.max() >= N):
            raise ValueError("force add: a node is not a cluster row")
        a = dict(self.arrays)
        keep = np.ones(P, bool)
        keep[pods] = False
        new_index = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
        kept_before = np.concatenate([[0], np.cumsum(keep)])
        a["pend_spec"] = np.ascontiguousarray(a["pend_spec"][keep])
        a["group_off"] = _i32(kept_before[a["group_off"]])
        off, spec = a["node_pod_off"], a["node_pod_spec"]
        by_row = np.argsort(nodes, kind="stable")                     # arrivals grouped by row, list order kept
        arrivals = np.bincount(nodes, minlength=len(off) - 1)
        new_off = np.concatenate([[0], np.cumsum((off[1:] - off[:-1]) + arrivals)])
        out_spec = np.empty(int(new_off[-1]), np.int32)
        is_old = np.ones(len(out_spec), bool)
        first_new = new_off[1:] - arrivals                            # where each row's arrivals start
        rows_sorted = nodes[by_row]
        rank = np.arange(len(pods)) - np.searchsorted(rows_sorted, rows_sorted, side="left")
        dst = first_new[rows_sorted] + rank
        is_old[dst] = False
        out_spec[is_old] = spec[:off[-1]]
        out_spec[dst] = self.arrays["pend_spec"][pods[by_row]]
        a["node_pod_off"] = _i32(new_off)
        a["node_pod_spec"] = out_spec
        out = copy.copy(self)
        out.arrays = a
        out.struct = self._restruct(a, num_pending=int(keep.sum()))
        return out, new_index

    def apply_resident_removals(self, cand_node, move_off, move_slot) -> Tuple["EncodedObjects", np.ndarray, np.ndarray]:
        """The objects after cae_simulate_resident_removals(cand_node, move_off, move_slot), stated on the host, and where
        each pod sits: listing k names resident slot move_slot[k] of cluster row cand_node[c]; the distinct (row, slot)
        pairs in first-listing order become the pending list, each with its spec or, when that spec names a node, its
        nodeName-cleared twin (the lowest spec id equal in every other column, else a spec appended in first-need order);
        one group per run of consecutive pending pods with the same spec.  Returns (objects, pend [M] = pending index of
        every listing, first [P] = the listing where each pending pod first appears).  A cae_load of the objects must
        answer like the engine after the call.  ValueError: what the engine answers with status -2 for the slot lists."""
        import copy
        cand = np.asarray(cand_node, np.int64).reshape(-1)
        off = np.asarray(move_off, np.int64).reshape(-1)
        slot = np.asarray(move_slot, np.int64).reshape(-1)
        N, a = self.struct.num_cluster_nodes, dict(self.arrays)
        if len(cand) and (len(off) != len(cand) + 1 or off[0] != 0 or (np.diff(off) < 0).any() or off[-1] != len(slot)):
            raise ValueError("resident removals: move_off must start at 0, not decrease and cover move_slot")
        if len(cand) and (cand.min() < -1 or cand.max() >= N):
            raise ValueError("resident removals: a candidate row outside [-1, N)")
        pod_off, pod_spec = a["node_pod_off"], a["node_pod_spec"]
        index_of: Dict[Tuple[int, int], int] = {}
        pend = np.zeros(len(slot), np.int32)
        first, spec = [], []
        for c in range(len(cand)):
            row, listed = int(cand[c]), set()
            for k in range(int(off[c]), int(off[c + 1])):
                s = int(slot[k])
                if row < 0 or s < 0 or s >= pod_off[row + 1] - pod_off[row]:
                    raise ValueError("resident removals: slot %d outside the resident pods of row %d" % (s, row))
                if (row, s) in listed:
                    raise ValueError("resident removals: slot %d of row %d listed twice for candidate %d" % (s, row, c))
                listed.add((row, s))
                p = index_of.setdefault((row, s), len(first))
                if p == len(first):
                    first.append(k)
                    spec.append(int(pod_spec[pod_off[row] + s]))
                pend[k] = p
        cols = [nm for nm in self.arrays if nm.startswith("ps_")]
        S = self.struct.num_podspecs
        twins: Dict[tuple, int] = {}
        new_rows: List[int] = []

        def key(s: int) -> tuple:
            return tuple(a[nm][s].tobytes() for nm in cols if nm != "ps_node_name")

        for i, s in enumerate(spec):
            if a["ps_node_name"][s] < 0:
                continue
            if not twins:
                for x in range(S - 1, -1, -1):
                    if a["ps_node_name"][x] < 0:
                        twins[key(x)] = x
            t = twins.setdefault(key(s), S + len(new_rows))
            if t == S + len(new_rows):
                new_rows.append(s)
            spec[i] = t
        for nm in cols:
            tail = a[nm][:S][new_rows].copy()
            if nm == "ps_node_name":
                tail[:] = -1
            a[nm] = np.ascontiguousarray(np.concatenate([a[nm][:S], tail]))
        ps = np.asarray(spec, np.int32)
        starts = [p for p in range(len(ps)) if p == 0 or ps[p] != ps[p - 1]]
        a["pend_spec"] = np.ascontiguousarray(ps)
        a["group_off"] = _i32(starts + [len(ps)])
        out = copy.copy(self)
        out.arrays = a
        out.struct = self._restruct(a, num_podspecs=S + len(new_rows), num_pending=len(ps), num_groups=len(starts))
        return out, pend, np.asarray(first, np.int32)

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
        _fill_pointers(s, arrays)
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


def _fill_pointers(s, arrays: Dict[str, np.ndarray]) -> None:
    """Point every field of the ctypes struct `s` that names one of `arrays` at that array."""
    for name, ctype in s._fields_:
        if name in arrays:
            setattr(s, name, arrays[name].ctypes.data_as(ctype))


def _count(field: str) -> property:
    return property(lambda self: getattr(self.struct, field))


class AbiArrays:
    """Owns the numpy arrays behind one ABI struct and the struct that points at them.  A subclass states its struct as a
    table; the fields, their dtypes and pointer types are the header's.  The constructor takes fields by name: an array
    left out is empty (an offsets array, which the header names ``*_off``, is ``[0]``; a per-row array is zeros of the
    row count), None is a NULL pointer and a scalar is set as given.  Every count follows its array."""

    STRUCT: type
    COUNTS: Dict[str, str] = {}       # count field -> the array whose length gives it (an offsets array's length - 1)
    ROWS: Optional[str] = None        # the array whose length is the row count
    PER_ROW: Tuple[str, ...] = ()     # the arrays of one entry per row
    PER_ROW_RES: Tuple[str, ...] = ()  # the per-row arrays of [rows][MAX_RES]
    NESTED: Optional[str] = None      # the field that points to an optional nested NodeDelta

    def __init__(self, **fields) -> None:
        nested = fields.pop(self.NESTED, None) if self.NESTED else None
        rows = len(fields.get(self.ROWS, ())) if self.ROWS else 0
        s, a = self.STRUCT(), {}
        fields.setdefault("abi_version", capi.CONST["CAE_ABI_VERSION"])
        for name, ctype in self.STRUCT._fields_:
            if name == self.NESTED:
                continue
            if not hasattr(ctype, "contents"):
                if name in fields:
                    setattr(s, name, fields[name])
                continue
            shape = (rows, MAX_RES) if name in self.PER_ROW_RES else (rows,)
            x = fields.get(name, np.zeros(shape) if name in self.PER_ROW else [0] if name.endswith("_off") else [])
            if x is not None:
                x = np.ascontiguousarray(x, np.dtype(ctype._type_))
                a[name] = np.ascontiguousarray(x.reshape(shape)) if name in self.PER_ROW_RES else x
        for cnt, nm in self.COUNTS.items():
            setattr(s, cnt, len(a[nm]) - nm.endswith("_off"))
        if self.NESTED:
            setattr(self, self.NESTED, nested)
            setattr(s, self.NESTED, C.pointer(nested.struct) if nested is not None else None)
        _fill_pointers(s, a)
        self.arrays, self.struct = a, s

    def replace(self, **arrays):
        """A copy with some arrays (or the nested struct) replaced (the counts follow the arrays)."""
        if self.NESTED:
            arrays.setdefault(self.NESTED, getattr(self, self.NESTED))
        return type(self)(**{**self.arrays, **arrays})

    def ptr(self):
        return C.byref(self.struct)


class NodeDelta(AbiArrays):
    """``cae_node_delta``: the dictionary tails (values, label sets, taint lists that continue the resident tables; offsets
    relative to the tail) and the complete new state of the dirty cluster rows."""

    STRUCT = capi.cae_node_delta
    COUNTS = {"num_new_values": "value_is_int", "num_new_labelsets": "ls_off", "num_new_taint_lists": "taint_off",
              "num_dirty": "row"}
    ROWS, PER_ROW, PER_ROW_RES = "row", ("labelset", "taint_list", "unschedulable", "alloc", "allowed_pods"), ("alloc",)
    num_dirty = _count("num_dirty")


class NodeChurn(AbiArrays):
    """``cae_node_churn``: ``changed`` (a NodeDelta with the dirty rows and the dictionary tails the dirty and the added
    rows use, or None), the removed rows and the added nodes."""

    STRUCT, NESTED = capi.cae_node_churn, "changed"
    COUNTS = {"num_removed": "removed", "num_added": "name"}
    ROWS, PER_ROW, PER_ROW_RES = "name", ("labelset", "taint_list", "unschedulable", "alloc", "allowed_pods"), ("alloc",)
    num_removed, num_added = _count("num_removed"), _count("num_added")

    def __init__(self, changed: Optional[NodeDelta] = None, **arrays) -> None:
        super().__init__(changed=changed, **arrays)


class UpcomingNodes(AbiArrays):
    """``cae_upcoming_nodes``: ``churn`` (a NodeChurn with the loop's real-node changes and the dictionary tails the copies
    use, or None) and the upcoming copies: template index, node-name id and label set of each."""

    STRUCT, NESTED = capi.cae_upcoming_nodes, "churn"
    COUNTS = {"num_upcoming": "template_idx"}
    num_upcoming = _count("num_upcoming")

    def __init__(self, churn: Optional[NodeChurn] = None, **arrays) -> None:
        super().__init__(churn=churn, **arrays)


class TemplateDelta(AbiArrays):
    """``cae_template_delta``: ``tails`` (a NodeDelta without dirty rows that carries the dictionary tails the new rows
    use, or None), the removed and changed template indices and the rows of the changed templates followed by the added
    ones."""

    STRUCT, NESTED = capi.cae_template_delta, "tails"
    COUNTS = {"num_removed": "removed", "num_changed": "changed"}
    ROWS, PER_ROW_RES = "name", ("alloc",)
    PER_ROW = ("labelset", "taint_list", "unschedulable", "alloc", "allowed_pods", "cap_cpu", "cap_mem", "has_alloc_cpu",
               "has_alloc_mem")
    num_removed, num_changed, num_added = _count("num_removed"), _count("num_changed"), _count("num_added")

    def __init__(self, tails: Optional[NodeDelta] = None, **arrays) -> None:
        super().__init__(tails=tails, **arrays)
        self.struct.num_added = len(self.arrays["name"]) - self.struct.num_changed


class PodDelta(AbiArrays):
    """``cae_pod_delta``: the dictionary tails and new pod specs (continuing the resident tables; offsets relative to the
    tail) and the complete new pending list."""

    STRUCT = capi.cae_pod_delta
    COUNTS = {"num_new_values": "value_is_int", "num_new_namespaces": "ns_labelset", "num_new_labelsets": "ls_off",
              "num_new_reqs": "req_key", "num_new_selectors": "sel_kind", "num_new_naff": "naff_nodesel",
              "num_new_naff_terms": "term_expr_sel", "num_new_tol_lists": "tol_off", "num_new_port_lists": "port_off",
              "num_new_pts_lists": "pts_off", "num_new_aff_lists": "aff_off", "num_new_aterms": "aterm_selector",
              "num_new_specs": "ps_namespace", "num_groups": "group_off", "num_pending": "pend_spec"}
    ROWS, PER_ROW_RES = "ps_namespace", ("ps_req",)
    PER_ROW = tuple(f for f, _ in capi.cae_pod_delta._fields_ if f.startswith("ps_"))
    num_new_specs = _count("num_new_specs")


class PriceInputs(AbiArrays):
    """``cae_price_inputs`` of cae_price_scores."""

    STRUCT = capi.cae_price_inputs


class SimilarityInputs(AbiArrays):
    """``cae_similarity_inputs`` of cae_similar_node_groups."""

    STRUCT = capi.cae_similarity_inputs
    COUNTS = {"num_ignored_keys": "ignored_keys"}


class DaemonSetInputs(AbiArrays):
    """``cae_daemonset_inputs`` of cae_template_daemonsets.  The optional arrays left out are NULL; num_ds follows ds_spec."""

    STRUCT = capi.cae_daemonset_inputs
    COUNTS = {"num_ds": "ds_spec"}

    def __init__(self, **fields) -> None:
        for nm in ("evaluate", "running", "keep"):
            fields.setdefault(nm, None)
        super().__init__(**fields)


class EligibilityInputs(AbiArrays):
    """``cae_eligibility_inputs`` of cae_scale_down_eligibility.  The optional arrays left out are NULL; n_pod_flags follows
    pod_flags unless given."""

    STRUCT = capi.cae_eligibility_inputs
    COUNTS = {"n_cand": "cand_node"}

    def __init__(self, **fields) -> None:
        for nm in ("pod_flags", "skip_ds", "pre_reason", "unready"):
            fields.setdefault(nm, None)
        super().__init__(**fields)
        if "n_pod_flags" not in fields:
            self.struct.n_pod_flags = len(self.arrays["pod_flags"]) if "pod_flags" in self.arrays else 0


class ResidentRemovals(AbiArrays):
    """``cae_resident_removals`` of cae_simulate_resident_removals.  The optional arrays left out are NULL."""

    STRUCT = capi.cae_resident_removals
    COUNTS = {"n_cand": "cand_node"}

    def __init__(self, **fields) -> None:
        for nm in ("dest_ok", "hint_node", "sim_class", "class_ctrl"):
            fields.setdefault(nm, None)
        super().__init__(**fields)


class RemovalPlan(AbiArrays):
    """``cae_removal_plan`` of cae_plan_removals.  The optional arrays left out are NULL; n_res follows drain and n_pdb
    pdb_namespace."""

    STRUCT = capi.cae_removal_plan
    COUNTS = {"n_cand": "cand_node", "n_res": "drain", "n_pdb": "pdb_namespace", "num_new_values": "value_is_int"}

    def __init__(self, **fields) -> None:
        for nm in ("dest_ok", "atomic", "hint_node", "sim_class", "class_ctrl"):
            fields.setdefault(nm, None)
        fields.setdefault("pdb_req_off", [0])
        fields.setdefault("req_val_off", [0])
        super().__init__(**fields)


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
        self.template_keys: Optional[List] = None   # the caller's key of each template (node-group id); None = position

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
        # the template rows the engine holds: (caller key, row state) per template, kept current by template_delta
        N, T = b.num_cluster_nodes, b.num_templates
        keys = list(range(T)) if self.template_keys is None else list(self.template_keys)
        if len(keys) != T or len(set(keys)) != T:
            raise ValueError("template_keys: one distinct key per template")
        self._templates = [(keys[t], (b.node_rows[r][0], b.node_rows[r][1], b.node_rows[r][2], b.node_rows[r][3],
                                      tuple(b.node_alloc[r]), b.node_rows[r][4], b.node_rows[r][5], b.node_rows[r][6],
                                      b.node_rows[r][7], b.node_rows[r][8], tuple(b.node_pod_spec[off[r]:off[r + 1]])))
                           for t, r in enumerate(range(N, N + T))]
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

    def upcoming_nodes(self, copies: Sequence[Tuple[int, NodeInfo]],
                       new_cluster: Optional[Sequence[NodeInfo]] = None) -> "UpcomingNodes":
        """The shim's side of cae_add_upcoming_nodes: `copies` = [(template index, sanitized copy)]
        (upcoming.upcoming_node_infos) appended after the cluster nodes, with the loop's real cluster list `new_cluster` as
        the churn of the same call (node_churn's rules; None = the real rows stay as they are).  Only each copy's node name
        and label set are interned; its other columns and its pods are its template's as the engine holds them.  The
        previous loop's copies are cluster rows like any other, so a `new_cluster` without them removes them.  The tails
        the copies' label sets add travel in the churn's ``changed``."""
        self._check_resident()
        T = len(self._templates)
        for t, _ in copies:
            if not 0 <= t < T:
                raise ValueError("upcoming nodes: template index %d out of range" % t)
        names = [self.node_names(ni.node.name) for _, ni in copies]
        ls = [self._labelset(ni.node.labels) for _, ni in copies]
        if new_cluster is None:
            churn = NodeChurn(self._tails_and_rows([], []))
        else:
            churn = self.node_churn(new_cluster)
        for (t, _), nid, l in zip(copies, names, ls):
            st = self._templates[t][1]
            self._cluster.append((nid, (l, st[2], st[3], st[4], st[5], st[10])))
        return UpcomingNodes(churn, template_idx=[t for t, _ in copies], name=names, labelset=ls)

    def _template_state(self, ni: NodeInfo) -> tuple:
        """(name, label set, taint list, unschedulable, allocatable, allowed pods, capacity cpu / memory, has_alloc cpu /
        memory, pod specs) of a template, interned append-only against the last load.  Its pods are incoming pods as far
        as the volume filters go (podspec's non-resident rule), and their specs are looked up among the specs the engine
        holds with nodeName ignored, as for a resident pod."""
        n, b = ni.node, self.b
        a = self._node_args(NodeInfo(n, []))
        if len(self.resources) > self._num_res:
            self._delta_ok = False
            raise Unsupported("template %s has a resource the last load did not have" % n.name)
        specs = []
        for p in ni.pods:
            if p.has_volumes_or_claims:
                raise Unsupported("template pod %s/%s uses volumes or resource claims" % (p.namespace, p.name))
            specs.append(self._resident_spec(p))
        return (a["name"], a["labelset"], a["taint_list"], int(a["unschedulable"]), tuple(a["alloc"]), a["allowed_pods"],
                a["cap_cpu"], a["cap_mem"], int(a["has_alloc_cpu"]), int(a["has_alloc_mem"]), tuple(specs))

    def template_delta(self, new_templates: Sequence[NodeInfo], keys: Optional[Sequence] = None) -> "TemplateDelta":
        """The shim's side of cae_load_templates: the complete new template list (what TemplateNodeInfoProvider returns,
        keyed by node-group id; `keys` None = the position) as a TemplateDelta against what the engine holds.  Vanished
        keys are removed, new keys are added, survivors whose state changed become changed rows.  The survivors must keep
        their relative order and the new templates must all come after them; a template pod's spec must be one the engine
        holds (run pod_delta(..., residents=templates) first for new ones); no new resource dimension.  Unsupported
        otherwise: a full load."""
        self._check_resident()
        keys = list(range(len(new_templates))) if keys is None else list(keys)
        if len(keys) != len(new_templates) or len(set(keys)) != len(keys):
            raise ValueError("template delta: one distinct key per template")
        old = {k: t for t, (k, _) in enumerate(self._templates)}
        last, seen_new = -1, False
        for k in keys:
            t = old.get(k)
            if t is None:
                seen_new = True
            elif seen_new or t < last:
                raise Unsupported("template delta: the surviving templates are reordered or a new one comes before one of them")
            else:
                last = t
        states = [self._template_state(ni) for ni in new_templates]
        kept = {old[k] for k in keys if k in old}
        removed = [t for t in range(len(self._templates)) if t not in kept]
        changed, rows, added = [], [], []
        for k, st in zip(keys, states):
            t = old.get(k)
            if t is None:
                added.append(st)
            elif st != self._templates[t][1]:
                changed.append(t)
                rows.append(st)
        rows += added
        po = [0]
        for st in rows:
            po.append(po[-1] + len(st[10]))
        col = lambda i: [st[i] for st in rows]
        delta = TemplateDelta(NodeDelta(**self._tails(_NODE_TABLES)), removed=removed, changed=changed, name=col(0),
                              labelset=col(1), taint_list=col(2), unschedulable=col(3),
                              alloc=np.asarray(col(4), np.int64).reshape(len(rows), MAX_RES), allowed_pods=col(5),
                              cap_cpu=col(6), cap_mem=col(7), has_alloc_cpu=col(8), has_alloc_mem=col(9), pod_off=po,
                              pod_spec=[x for st in rows for x in st[10]])
        self._templates = list(zip(keys, states))
        return delta

    def note_template_pods(self, enc: EncodedObjects) -> None:
        """Take the template pod lists of `enc` as what the engine holds, after a call that changed them on the device
        (cae_template_daemonsets with keep), so that the next template_delta compares against them."""
        a, N = enc.arrays, enc.struct.num_cluster_nodes
        off, spec = a["node_pod_off"], a["node_pod_spec"]
        self._templates = [(k, st[:10] + (tuple(int(x) for x in spec[off[N + t]:off[N + t + 1]]),))
                           for t, (k, st) in enumerate(self._templates)]

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
           namespaces: Sequence[Namespace] = (), encoder: Optional[Encoder] = None,
           template_keys: Optional[Sequence] = None) -> EncodedObjects:
    """encoder: the Encoder to intern with (a fresh one by default), for a caller that needs its dictionaries afterwards.
    template_keys: the caller's key of each template (node-group id) that Encoder.template_delta matches by."""
    enc = encoder or Encoder()
    if template_keys is not None:
        enc.template_keys = list(template_keys)
    for ns in namespaces:
        enc.add_namespace(ns)
    for ni in cluster:
        enc.add_cluster_node(ni)
    for ni in templates:
        enc.add_template(ni)
    for g in groups:
        enc.add_group(g)
    return enc.finish()
