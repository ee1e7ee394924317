#!/usr/bin/env python
"""Where does the dense pass's step time go?  Event-to-event time of cae_feasibility on C2 with a cold L2
(512 MiB memset before every step, as bench.py does), a warm L2, and of an empty torch kernel for the
launch + event floor of this box.

With a library built with -DCAE_K1_PROF (CAE_NVCC_EXTRA=-DCAE_K1_PROF for build(), or another build through
CAE_ENGINE_LIB) it also prints the kernel's phase timeline on C2 and on the C3-sized launch, cold L2: from
%globaltimer stamps of every thread block (entry, loads done, compute done, bit-matrix stores issued, exit) and one
taken when the stream reached the launch.  The prof build's event time includes the stamp kernel and the clearing
of the stamp buffer; compare step times with a product build."""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

STAMPS = 5
PROF_WORDS = 1 + STAMPS * 8192
PHASES = ("loads", "compute", "stores", "finish")   # stamp i -> i + 1 of one block


def _timeline(prof):
    """Per-step figures (ns) from one read of the stamp buffer."""
    mark = int(prof[0])
    st = prof[1:].reshape(-1, STAMPS).astype(np.int64)
    st = st[st[:, 0] != 0]
    out = {"blocks": int(len(st)), "launch_to_first_block_start": int(st[:, 0].min() - mark),
           "last_block_end": int(st[:, STAMPS - 1].max() - mark),
           "first_block_end": int(st[:, STAMPS - 1].min() - mark)}
    for i, name in enumerate(PHASES):
        d = st[:, i + 1] - st[:, i]
        out[name + "_median"] = float(np.median(d))
        out[name + "_max"] = int(d.max())
    return out


def _measure(eng, flush, cold, steps=25, warm=5, prof_read=None):
    ms, tl = [], []
    buf = (ctypes.c_ulonglong * PROF_WORDS)()
    for i in range(steps):
        if cold:
            flush.zero_()
        torch.cuda.synchronize()
        eng.lib.cae_feasibility(eng.h, None, None, None)
        if i >= warm:
            ms.append(eng.stats().feasibility_ms)
            if prof_read is not None:
                n = prof_read(buf, PROF_WORDS)
                tl.append(_timeline(np.frombuffer(buf, dtype=np.uint64, count=n)))
    return ms, tl


def main():
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine
    eng = Engine()
    prof_read = getattr(eng.lib, "cae_k1_prof_read", None)
    if prof_read is not None:
        prof_read.argtypes = [ctypes.c_void_p, ctypes.c_int]
        prof_read.restype = ctypes.c_int
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    out = {"device": torch.cuda.get_device_name(0), "lib": os.environ.get("CAE_ENGINE_LIB", "tree"),
           "prof_build": prof_read is not None}
    eng.load(synth.generate(2))
    for name, cold in (("cold", True), ("warm", False)):
        ms, _ = _measure(eng, flush, cold)
        out[name + "_us"] = 1e3 * float(np.mean(ms))
        out[name + "_median_us"] = 1e3 * float(np.median(ms))
        out[name + "_min_us"] = 1e3 * float(np.min(ms))
    if prof_read is not None:
        for cfg in (2, 3):
            eng.load(synth.generate(cfg))
            ms, tl = _measure(eng, flush, True, prof_read=prof_read)
            row = {"event_step_us_median": 1e3 * float(np.median(ms))}
            for k in tl[0]:
                row[k if k == "blocks" else k + "_us"] = float(np.median([t[k] for t in tl])) / (1 if k == "blocks" else 1e3)
            out["timeline_C%d" % cfg] = row
    x = torch.zeros(1, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for i in range(25):
        flush.zero_()
        torch.cuda.synchronize()
        e0.record()
        x.add_(1)
        e1.record()
        torch.cuda.synchronize()
        if i >= 5:
            ms.append(e0.elapsed_time(e1))
    out["tiny_kernel_event_to_event_us"] = 1e3 * float(np.mean(ms))
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
