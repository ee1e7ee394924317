"""ctypes view of ``include/caengine.h``.

The struct layouts and the function signatures are parsed from the header so that the header stays
the single source of truth for the ABI (a field or parameter added there is picked up here; a
mismatch cannot happen silently).  Only ``int32_t`` / ``int64_t`` / ``double`` scalars, arrays of
them and ``const T*`` pointers appear in the ABI structs.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Dict, List, Optional, Tuple

REPO_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO_ROOT, "include", "caengine.h")
PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ENGINE_LIB = os.path.join(PKG_DIR, "libcaengine.so")

_SCALARS = {"int32_t": C.c_int32, "int64_t": C.c_int64, "uint8_t": C.c_uint8, "uint16_t": C.c_uint16,
            "uint32_t": C.c_uint32, "double": C.c_double, "size_t": C.c_size_t}


def _strip_comments(src: str) -> str:
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def _parse_struct(src: str, name: str, structs: Optional[Dict[str, type]] = None) -> List[Tuple[str, object]]:
    """``structs``: ABI structs a field may point to, by their C name."""
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, flags=re.S)
    if not m:
        raise RuntimeError("struct %s not found in %s" % (name, HEADER))
    fields: List[Tuple[str, object]] = []
    for decl in m.group(1).split(";"):
        decl = decl.strip()
        if not decl:
            continue
        mm = re.match(r"(const\s+)?(\w+)\s*(\*?)\s*([\w, ]+?)(\[(\d+)\])?$", decl)
        if not mm:
            raise RuntimeError("cannot parse field %r of %s" % (decl, name))
        ctype = _SCALARS[mm.group(2)] if mm.group(2) in _SCALARS else (structs or {})[mm.group(2)]
        for fname in [f.strip() for f in mm.group(4).split(",")]:
            if mm.group(3):
                fields.append((fname, C.POINTER(ctype)))
            elif mm.group(6):
                fields.append((fname, ctype * int(mm.group(6))))
            else:
                fields.append((fname, ctype))
    return fields


def _parse_enums(src: str) -> Dict[str, int]:
    out: Dict[str, int] = {}
    for m in re.finditer(r"enum \w+ \{(.*?)\};", src, flags=re.S):
        nxt = 0
        for item in m.group(1).split(","):
            item = item.strip()
            if not item:
                continue
            if "=" in item:
                k, v = [s.strip() for s in item.split("=")]
                nxt = int(v, 0)
            else:
                k = item
            out[k] = nxt
            nxt += 1
    for m in re.finditer(r"#define (CAE_\w+) (\d+)", src):
        out[m.group(1)] = int(m.group(2))
    return out


with open(HEADER) as _f:
    _SRC = _strip_comments(_f.read())

CONST = _parse_enums(_SRC)
globals().update(CONST)


class cae_objects(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_objects")


class cae_config(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_config")


class cae_stats(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_stats")


class cae_price_inputs(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_price_inputs")


class cae_node_delta(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_node_delta")


class cae_node_churn(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_node_churn", {"cae_node_delta": cae_node_delta})


class cae_upcoming_nodes(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_upcoming_nodes", {"cae_node_churn": cae_node_churn})


class cae_template_delta(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_template_delta", {"cae_node_delta": cae_node_delta})


class cae_pod_delta(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_pod_delta")


class cae_similarity_inputs(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_similarity_inputs")


class cae_daemonset_inputs(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_daemonset_inputs")


class cae_eligibility_inputs(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_eligibility_inputs")


class cae_resident_removals(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_resident_removals")


class cae_removal_plan(C.Structure):
    _fields_ = _parse_struct(_SRC, "cae_removal_plan")


_STRUCTS = {s.__name__: s for s in (cae_objects, cae_config, cae_stats, cae_price_inputs, cae_node_delta, cae_node_churn,
                                     cae_upcoming_nodes, cae_template_delta, cae_pod_delta, cae_similarity_inputs, cae_daemonset_inputs,
                                     cae_eligibility_inputs,
                                     cae_resident_removals, cae_removal_plan)}


def _ctype(decl: str, opaque, where: str):
    """ctypes type of one C declaration (a return type or a parameter, its name optional); None for ``void``."""
    m = re.fullmatch(r"(?:const\s+)?(\w+)\s*(\**)\s*(?:\w+)?", decl.strip())
    base, stars = (m.group(1), len(m.group(2))) if m else (None, 0)
    if stars and (base in _SCALARS or base in _STRUCTS or base in opaque or base in ("void", "char")):
        if stars > 1:
            return C.POINTER(C.c_void_p)
        if base == "char":
            return C.c_char_p
        if base == "size_t":
            return C.POINTER(C.c_size_t)
        return C.POINTER(_STRUCTS[base]) if base in _STRUCTS else C.c_void_p
    if not stars and (base in _SCALARS or base == "void"):
        return _SCALARS.get(base)
    raise RuntimeError("cannot map the C type %r of %s" % (decl.strip(), where))


def signatures(src: str) -> Dict[str, Tuple[object, List[object]]]:
    """{function: (restype, argtypes)} of every prototype in the comment-stripped header source `src`."""
    opaque = set(re.findall(r"typedef struct (\w+) \1;", src))
    out: Dict[str, Tuple[object, List[object]]] = {}
    for m in re.finditer(r"^((?:const\s+)?\w+\s*\**)\s*(cae_\w+)\s*\(([^()]*)\)\s*;", src, flags=re.M):
        name, params = m.group(2), [p for p in m.group(3).split(",") if p.strip()]
        if [p.strip() for p in params] == ["void"]:
            params = []
        args = [_ctype(p, opaque, name) for p in params]
        if None in args:
            raise RuntimeError("%s has a void parameter" % name)
        out[name] = (_ctype(m.group(1), opaque, name), args)
    missed = set(re.findall(r"\b(cae_\w+)\s*\(", src)) - set(out)
    if missed:
        raise RuntimeError("cannot parse the prototypes of %s" % sorted(missed))
    return out


def declared_functions() -> List[str]:
    """Names of every function the header declares (used by the symbol-export test)."""
    return sorted(signatures(_SRC))


REASON_NAMES = {v: k for k, v in CONST.items() if k.startswith("CAE_R_")}

# reason -> (plugin name, reason string) as the reference reports them
REASON_PLUGIN = {
    CONST["CAE_R_OK"]: ("", ""),
    CONST["CAE_R_PREFILTER_NODEAFFINITY"]: ("NodeAffinity", "PreFilter filtered the Node out"),
    CONST["CAE_R_NODE_UNSCHEDULABLE"]: ("NodeUnschedulable", "node(s) were unschedulable"),
    CONST["CAE_R_NODE_NAME"]: ("NodeName", "node(s) didn't match the requested node name"),
    CONST["CAE_R_TAINT"]: ("TaintToleration", "node(s) had untolerated taint(s)"),
    CONST["CAE_R_NODE_AFFINITY"]: ("NodeAffinity", "node(s) didn't match Pod's node affinity/selector"),
    CONST["CAE_R_NODE_PORTS"]: ("NodePorts", "node(s) didn't have free ports for the requested pod ports"),
    CONST["CAE_R_FIT"]: ("NodeResourcesFit", "Insufficient resources / Too many pods"),
    CONST["CAE_R_PTS_MISSING_LABEL"]: ("PodTopologySpread", "node(s) didn't match pod topology spread constraints (missing required label)"),
    CONST["CAE_R_PTS_SKEW"]: ("PodTopologySpread", "node(s) didn't match pod topology spread constraints"),
    CONST["CAE_R_IPA_AFFINITY"]: ("InterPodAffinity", "node(s) didn't match pod affinity rules"),
    CONST["CAE_R_IPA_ANTI_AFFINITY"]: ("InterPodAffinity", "node(s) didn't match pod anti-affinity rules"),
    CONST["CAE_R_IPA_EXISTING_ANTI_AFFINITY"]: ("InterPodAffinity", "node(s) didn't satisfy existing pods anti-affinity rules"),
}

_engine_lib = None


def load_engine_lib() -> C.CDLL:
    """dlopen the product library.  Fails loudly: there is NO CPU fallback in the product path."""
    global _engine_lib
    if _engine_lib is not None:
        return _engine_lib
    path = os.environ.get("CAE_ENGINE_LIB", ENGINE_LIB)     # experiments: another build of the same library
    if not os.path.exists(path):
        raise RuntimeError(
            "libcaengine.so is missing (%s): build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'`. The engine has no CPU fallback." % path)
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    for name, (restype, argtypes) in signatures(_SRC).items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _engine_lib = lib
    return lib
