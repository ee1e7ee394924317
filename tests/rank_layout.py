"""Which kernel instantiations a load runs, computed on the host from the encoded tables alone.

``layout_of`` restates what ``cae_load`` derives before any launch (csrc/api.cu, active dims through the threshold rows):
the active resource dims, the rank fields packed into 32-bit words, the bit slices and the threshold rows of the dense
pass, and so whether the dense pass takes the LUT kernel or the bit-sliced one.  ``uses_window`` restates how the
estimator sizes its node store (csrc/binpack.cu, launch_binpack).  The parametrizations of the GPU tests are checked
against these without a GPU, so a change of generator that silently drops a cell fails on any machine."""
import numpy as np

MAX_RES = 8
MAX_W = 4                 # FEAS_MAX_W
LUT_MAX_ROWS = 1024       # FEAS_LUT_MAX_ROWS
MAX_SLICES = 32
SMEM_OPTIN = 227 * 1024   # opt-in shared memory per thread block of an H100 (sharedMemPerBlockOptin)

# one active-dim set per dim count A, most of them not a prefix of (cpu, memory, ephemeral-storage, ...)
DIM_SETS = {0: (), 1: (1,), 2: (0, 4), 3: (1, 2, 6), 4: (0, 3, 5, 7), 5: (1, 2, 3, 4, 6), 6: (0, 1, 2, 5, 6, 7),
            7: (1, 2, 3, 4, 5, 6, 7), 8: (0, 1, 2, 3, 4, 5, 6, 7)}


def layout_of(enc, force_bitslice=False):
    """A, act_dims, lut_rows, slices, W, and path: "lut", "bitslice", or None when the load is refused."""
    req = enc.arrays["ps_req"][np.unique(enc.arrays["pend_spec"])]
    act = [d for d in range(req.shape[1]) if (req[:, d] > 0).any()]
    card = [len(np.unique(req[req[:, d] > 0, d])) for d in act]
    W = word = shift = 0
    ok = True
    for d in card:
        bits = max(1, d.bit_length()) + 1            # ranks 0..d, + the guard bit
        if shift + bits > 32:
            word, shift = word + 1, 0
        ok = ok and word < MAX_W and bits <= 32
        shift += bits
        W = word + 1
    slices = sum(max(1, d.bit_length()) for d in card)
    rows = sum(d + 1 for d in card)
    ok = ok and slices <= MAX_SLICES
    path = None if not ok else ("bitslice" if force_bitslice or rows > LUT_MAX_ROWS else "lut")
    return dict(A=len(act), act_dims=tuple(act), lut_rows=rows, slices=slices, W=W, path=path)


def window_nodes(A, smem_optin=SMEM_OPTIN):
    """The most added nodes the estimator keeps in shared memory (WIN = true) at A active dims."""
    node_bytes = 8 * max(A, 1) + 8 + 4 + 4 + 4 + 1
    limit = smem_optin - 9216
    n = limit // node_bytes
    while (n * node_bytes + 15) & ~15 > limit:
        n -= 1
    return n


def uses_window(A, P, caps, smem_optin=SMEM_OPTIN):
    """Whether Estimate() of a load with P pending pods and these limiter caps runs on the shared window (else the slab)."""
    cap = 1
    for m in caps:
        cap = max(cap, m if m > 0 else (P + 1 if m == 0 else 1))
    return max(1, min(P + 1, cap)) <= window_nodes(A, smem_optin)
