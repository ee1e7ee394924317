"""Dense pass (K1) at the edges of its decomposition over pod words and template words: a single pod, fewer pod words
than thread blocks, fewer templates than one word, ragged P and T, many template words.  Bit matrix, histogram and
(with reasons) the first failing plugin must equal the oracle bit for bit, also on a second pass over the same load.

Every instantiation of the pass: A = 0..8 active resource dims (not a prefix of the dims for most A) on the LUT kernel,
also with several pod words per thread block, and on the bit-sliced kernel, and the boundaries of the rank layout (a second rank word, the largest
threshold table, the 32-slice limit).  The non-GPU test at the end checks that these inputs really have those layouts."""
import functools

import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import synth

SHAPES = [
    pytest.param(1, 50, id="one_pod"),                              # Pl = 1: one pod word
    pytest.param(100, 20, id="few_pod_words_T_lt_32"),              # 4 pod words, one partial template word
    pytest.param(3001, 1181, id="ragged_P_prime_Tw"),               # P % 32 != 0, Tw = 37 (prime)
    pytest.param(1500, 5000, id="many_template_words"),             # Tw = 157
]

# the shape of the instantiation sweep: ragged P and T, 3 template chunks of 512, G > 1 pod blocks per chunk
SWEEP_P, SWEEP_T = 3001, 1181
# one template chunk and more pod words than an H100 holds LUT blocks at once: every block takes several pod words, and the
# words do not split evenly over the blocks
MULTIWORD_P, MULTIWORD_T = 20011, 500
# variant -> (environment, shape)
VARIANTS = {"lut16": ({}, (SWEEP_P, SWEEP_T)), "lut16_multiword": ({}, (MULTIWORD_P, MULTIWORD_T)),
            "bitslice": ({"CAE_K1_BITSLICE": "1"}, (SWEEP_P, SWEEP_T))}

# rank-layout boundaries: dim -> distinct request values, and the layout that must result
_SMALL6 = {0: 3, 1: 2, 2: 3, 4: 2, 5: 3}                            # 18 threshold rows, 10 slices
BOUNDARIES = {
    "W2_lut_32_slices": ({d: 15 for d in range(8)}, dict(A=8, W=2, slices=32, lut_rows=128, path="lut")),
    "W2_bitslice_fallback": ({0: 1000, 1: 15, 2: 15, 3: 15, 5: 15, 7: 1}, dict(A=6, W=2, slices=27, lut_rows=1067, path="bitslice")),
    "lut_rows_1024": ({**_SMALL6, 7: 1005}, dict(A=6, W=1, slices=20, lut_rows=1024, path="lut")),
    "lut_rows_1025": ({**_SMALL6, 7: 1006}, dict(A=6, W=1, slices=20, lut_rows=1025, path="bitslice")),
    "33_slices": ({**{d: 15 for d in range(7)}, 7: 16}, dict(A=8, W=2, slices=33, lut_rows=129, path=None)),
}


@functools.lru_cache(maxsize=None)
def _sweep_enc(A, shape=(SWEEP_P, SWEEP_T)):
    return synth.generate(2, pods=shape[0], templates=shape[1], dims=rank_layout.DIM_SETS[A])


@functools.lru_cache(maxsize=None)
def _boundary_enc(name):
    return synth.generate(2, pods=SWEEP_P, templates=300, dims=BOUNDARIES[name][0])


_want = {}


def _oracle_dense(oracle, key, enc):
    if key not in _want:
        _want[key] = oracle.feasibility_dense(enc)[0]
    return _want[key]


def _check_passes(e, enc, want, want_reasons):
    from kubernetes_autoscaler_b200.engine import unpack_bits
    e.load(enc)
    for _ in range(2):   # a second pass must not see state of the first
        bits, reasons, count = e.feasibility()
        if want_reasons:
            assert np.array_equal(reasons, want)
        assert np.array_equal(unpack_bits(bits, enc.P), want == 0)
        assert np.array_equal(count, (want == 0).sum(axis=1))


@pytest.mark.gpu
@pytest.mark.parametrize("want_reasons", [True, False])
@pytest.mark.parametrize("pods,templates", SHAPES)
def test_dense_decomposition_edges(oracle, pods, templates, want_reasons):
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    enc = synth.generate(2, pods=pods, templates=templates)
    want, _ = oracle.feasibility_dense(enc)
    e = Engine(device=0, want_reasons=want_reasons)
    try:
        _check_passes(e, enc, want, want_reasons)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("want_reasons", [True, False])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("A", range(9))
def test_dense_every_dim_count(oracle, monkeypatch, A, variant, want_reasons):
    """feasibility_lut_kernel<A, REASONS, 16> for A = 0..8 (at one and at several pod words per block), and the bit-sliced
    kernel at the slice counts these give."""
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    env, shape = VARIANTS[variant]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    enc = _sweep_enc(A, shape)
    want = _oracle_dense(oracle, ("sweep", A, shape), enc)
    e = Engine(device=0, want_reasons=want_reasons)
    try:
        _check_passes(e, enc, want, want_reasons)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("want_reasons", [True, False])
@pytest.mark.parametrize("name", [n for n in BOUNDARIES if BOUNDARIES[n][1]["path"]] + ["W2_lut_32_slices/bitslice"])
def test_dense_rank_layout_boundaries(oracle, monkeypatch, name, want_reasons):
    """A second rank word on both kernels, 32 slices (the most the bit-sliced encoding holds), 1024 threshold rows at A = 6
    on the LUT kernel (104 KB of shared memory per block) and 1025 on the automatic fallback."""
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    base, _, forced = name.partition("/")
    if forced:
        monkeypatch.setenv("CAE_K1_BITSLICE", "1")
    enc = _boundary_enc(base)
    want = _oracle_dense(oracle, ("boundary", base), enc)
    e = Engine(device=0, want_reasons=want_reasons)
    try:
        _check_passes(e, enc, want, want_reasons)
    finally:
        e.close()


@pytest.mark.gpu
def test_dense_33_slices_is_refused(oracle):
    """One slice more than the bit-sliced encoding holds: the load answers "unsupported", whichever kernel would run, and
    the engine still takes the next load."""
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine, EngineUnsupported
    e = Engine(device=0, want_reasons=True)
    try:
        with pytest.raises(EngineUnsupported, match="bit-sliced"):
            e.load(_boundary_enc("33_slices"))
        enc = _boundary_enc("W2_lut_32_slices")
        _check_passes(e, enc, _oracle_dense(oracle, ("boundary", "W2_lut_32_slices"), enc), True)
    finally:
        e.close()


def test_dense_parametrization_covers_every_cell():
    """Without a GPU: the inputs above have the layouts the GPU tests claim to cover."""
    Tw, Plw = -(-SWEEP_T // 32), -(-SWEEP_P // 32)
    assert SWEEP_P % 32 and SWEEP_T % 32
    assert -(-Tw // 16) == 3           # template chunks of FEAS_TW = 16 words
    assert -(-Plw // 16) > 1           # even a 16-warp block takes a part of the pod words: G > 1 blocks per chunk
    Tw_m, Plw_m = -(-MULTIWORD_T // 32), -(-MULTIWORD_P // 32)
    assert -(-Tw_m // 16) == 1         # one template chunk
    assert Plw_m > 3 * 132 and all(Plw_m % g for g in (132, 264, 396))   # 132 SMs x 1..3 LUT blocks: >= 2 words for some blocks, uneven
    bitsliced = set()                  # instantiations feasibility_kernel<B> run, B = slices rounded up to 4
    for A in range(9):
        enc = _sweep_enc(A)
        lay = rank_layout.layout_of(enc)
        assert (lay["A"], lay["act_dims"], lay["W"], lay["path"]) == (A, rank_layout.DIM_SETS[A], 1 if A else 0, "lut"), lay
        assert rank_layout.layout_of(enc, force_bitslice=True)["path"] == "bitslice"
        bitsliced.add(-(-lay["slices"] // 4) * 4)
        lay_m = rank_layout.layout_of(_sweep_enc(A, (MULTIWORD_P, MULTIWORD_T)))
        assert (lay_m["A"], lay_m["act_dims"], lay_m["path"]) == (A, rank_layout.DIM_SETS[A], "lut"), lay_m
    assert sum(s != tuple(range(len(s))) for s in rank_layout.DIM_SETS.values()) >= 6   # mostly non-prefix active sets
    for name, (_, want) in BOUNDARIES.items():
        lay = rank_layout.layout_of(_boundary_enc(name))
        assert {k: lay[k] for k in want} == want, name
        if lay["path"] == "bitslice" or name == "W2_lut_32_slices":   # the latter also runs with CAE_K1_BITSLICE=1
            bitsliced.add(-(-lay["slices"] // 4) * 4)
    assert bitsliced == {0, 4, 8, 12, 16, 20, 28, 32}, bitsliced
