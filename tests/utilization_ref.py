"""CPU restatement of the scale-down eligibility from the utilization on (utilization.Calculate, simulator/utilization/
info.go; the end of eligibility.Checker.FilterOutUnremovable, core/scaledown/eligibility/eligibility.go) over NodeInfo
objects, independent of the encoder and the engine: resources by name, exact Python integers, Go's float64 division and
math.Max stated explicitly (Python raises on x / 0.0 and its max() does not propagate NaN)."""
import math
import struct

import numpy as np

UNNEEDED, PRE, UNEXPECTED_ERROR, UNREADY_DISABLED, NOT_UNDERUTILIZED = range(5)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
_ERROR, _BIG = "error", "big"


def go_div(a: float, b: float) -> float:
    """IEEE float64 division as Go evaluates it: 0/0 = NaN, x/0 = +-Inf with the sign of a times that of b."""
    if b == 0.0:
        if a == 0.0 or math.isnan(a):
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def go_max(x: float, y: float) -> float:
    """math.Max: +Inf first, then NaN, then +0 over -0."""
    if x == math.inf or y == math.inf:
        return math.inf
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if x == 0.0 and y == 0.0:
        return y if math.copysign(1.0, x) < 0 else x
    return x if x > y else y


def _wrap64(v: int) -> int:
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


def _fits(v: int) -> bool:
    return INT64_MIN <= v <= INT64_MAX


def _is_daemonset(p) -> bool:
    return p.owner_kind == "DaemonSet" or p.annotations.get("cluster-autoscaler.kubernetes.io/daemonset-pod") == "true"


def _is_mirror(p) -> bool:
    return "kubernetes.io/config.mirror" in p.annotations


def _long_terminating(p, now: float) -> bool:
    if p.deletion_timestamp is None:
        return False
    grace = 30 if p.termination_grace_period_seconds is None else p.termination_grace_period_seconds
    return p.deletion_timestamp + grace + 30 < now


def _milli(resource: str, v: int):
    m = v if resource == "cpu" else v * 1000
    return m if _fits(m) else _BIG


def utilization_of(ni, resource: str, skip_ds: bool, skip_mirror: bool, now: float):
    """CalculateUtilizationOfResource: a float, _ERROR or _BIG (a value Go's Quantity holds past int64)."""
    alloc = ni.node.allocatable.get(resource)
    if alloc is None:
        return _ERROR
    am = _milli(resource, alloc)
    if am is _BIG:
        return _BIG
    if am == 0:
        return _ERROR
    counted = excluded = 0
    for p in ni.pods:
        v = p.requests.get(resource, 0)
        if (skip_ds and _is_daemonset(p)) or (skip_mirror and _is_mirror(p)):
            excluded += v
            continue
        if _long_terminating(p, now):
            continue
        counted += v
    if not (_fits(counted) and _fits(excluded)):
        return _BIG
    cm, em = _milli(resource, counted), _milli(resource, excluded)
    if cm is _BIG or em is _BIG:
        return _BIG
    return go_div(float(cm), float(_wrap64(am - em)))


def eligibility(cluster, cand_rows, gpu_resource, threshold, now, skip_ds=None, skip_mirror=False, pre=None, unready=None):
    """Per candidate i (cluster row cand_rows[i]; gpu_resource[i] None = no GpuConfig): (status, util [n][4], reason [n],
    unneeded).  status 1: some value the utilization reads leaves int64 (util / reason then undefined)."""
    n = len(cand_rows)
    util = np.zeros((n, 4), np.float64)
    reason = np.zeros(n, np.uint8)
    status = 0
    for i in range(n):
        if pre is not None and pre[i]:
            reason[i] = PRE
            continue
        ni = cluster[cand_rows[i]]
        ds = bool(skip_ds[i]) if skip_ds is not None else False
        if gpu_resource[i] is not None:
            g = utilization_of(ni, gpu_resource[i], ds, skip_mirror, now)
            vals = None if g in (_ERROR, _BIG) else (0.0, 0.0, g, g)
            bad = g
        else:
            c = utilization_of(ni, "cpu", ds, skip_mirror, now)
            m = utilization_of(ni, "memory", ds, skip_mirror, now) if c not in (_ERROR, _BIG) else None
            bad = c if c in (_ERROR, _BIG) else m
            vals = None if bad in (_ERROR, _BIG) else (c, m, 0.0, go_max(c, m))
        if vals is None:
            status |= bad is _BIG
            reason[i] = UNEXPECTED_ERROR
            continue
        util[i] = vals
        if unready is not None and unready[i]:
            reason[i] = UNREADY_DISABLED
        else:
            reason[i] = UNNEEDED if not (vals[3] >= threshold[i]) else NOT_UNDERUTILIZED
    return status, util, reason, np.flatnonzero(reason == UNNEEDED).astype(np.int32)


def same_bits(a, b) -> bool:
    """float64 arrays equal bit for bit, every NaN equal to every NaN"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (a.view(np.int64) == b.view(np.int64))))


def bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]
