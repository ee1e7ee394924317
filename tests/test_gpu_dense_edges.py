"""Dense pass (K1) at the edges of its decomposition over pod words and template words: a single pod, fewer pod words
than thread blocks, fewer templates than one word, ragged P and T, many template words.  Bit matrix, histogram and
(with reasons) the first failing plugin must equal the oracle bit for bit, also on a second pass over the same load."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import synth

pytestmark = pytest.mark.gpu

SHAPES = [
    pytest.param(1, 50, id="one_pod"),                              # Pl = 1: one pod word
    pytest.param(100, 20, id="few_pod_words_T_lt_32"),              # 4 pod words, one partial template word
    pytest.param(3001, 1181, id="ragged_P_prime_Tw"),               # P % 32 != 0, Tw = 37 (prime)
    pytest.param(1500, 5000, id="many_template_words"),             # Tw = 157
]


@pytest.mark.parametrize("want_reasons", [True, False])
@pytest.mark.parametrize("pods,templates", SHAPES)
def test_dense_decomposition_edges(oracle, pods, templates, want_reasons):
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine, unpack_bits
    enc = synth.generate(2, pods=pods, templates=templates)
    want, _ = oracle.feasibility_dense(enc)
    e = Engine(device=0, want_reasons=want_reasons)
    try:
        e.load(enc)
        for _ in range(2):   # a second pass must not see state of the first
            bits, reasons, count = e.feasibility()
            if want_reasons:
                assert np.array_equal(reasons, want)
            assert np.array_equal(unpack_bits(bits, enc.P), want == 0)
            assert np.array_equal(count, (want == 0).sum(axis=1))
    finally:
        e.close()
