"""K1q's lookup tables under changing weights (-m gpu).  The host-streaming Form Q / P calls keep tables of their own, which
the next such call rebuilds when its codebook or the weights changed; the resident Form Q tensor (or the Form Q / W copy of a
Form D one) keeps its tables, which apo_set_weights rebuilds, across streamed calls with another codebook.  Every result must
equal the oracle's integers under the weights set last."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W2 = np.array([0.3, 0.05, 0.1, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])


@pytest.fixture
def bare(apo, orc):
    """an engine with no resident Form Q tensor and no copy: nothing but streamed calls build K1q's tables"""
    e = apo.Engine(0)
    try:
        yield e
    finally:
        e.set_weights(orc.weights())
        e.close()


@pytest.mark.parametrize("wire", ["compact", "packed"])
def test_streamed_calls_follow_set_weights(bare, orc, apo, wire):
    """a weight sweep over one streamed tensor: the second call, with the same codebook, must use the new weights"""
    seed, C, T = 0x5EEDC0DE, 4, 30_003
    dims = orc.gen_dims(seed, 2, C, 100, T, 400, 8)
    if wire == "compact":
        q8, d2, li, book = apo.compact_encode_host(dims, nthreads=4)
        call = lambda: bare.score_host_compact(q8, d2, li, book, 2)
    else:
        pc, pd, book, d2book = apo.packed_encode_host(dims, nthreads=4)
        call = lambda: bare.score_host_packed(pc, pd, book, d2book, 2)
    call()
    assert bare.debug_partials(C) == orc.score_dims_fx(dims)
    for w in (W2, orc.weights(), W2):
        bare.set_weights(w)
        call()
        assert bare.debug_partials(C) == orc.score_dims_fx(dims, w=w)


@pytest.mark.parametrize("resident", ["compact", "copy"])
def test_resident_tables_survive_a_streamed_codebook(engine, orc, apo, resident):
    """a resident Form Q tensor, or the Form W copy of a Form D one, scored after a streamed call with another codebook and
    a weight change"""
    seed, C, T = 0x5EEDC0DF, 3, 20_001
    dims = orc.gen_dims(seed, 2, C, 100, T, 400, 8)
    other = dims.copy()
    other[:, :, 0] *= 0.5                                                   # same shape, other values: another codebook
    q8, d2, li, book = apo.compact_encode_host(other, nthreads=4)
    try:
        engine.set_tuning(0)
        engine.dims_upload(dims)
        if resident == "compact":
            engine.dims_compact()
            assert engine.dims_layout() == 2
            assert not np.array_equal(engine.dims_codebook(), book)
        for w in (orc.weights(), W2):
            engine.set_weights(w)
            engine.score(C, 1)
            assert engine.debug_partials(C) == orc.score_dims_fx(dims, w=w)
            engine.score_host_compact(q8, d2, li, book, 1)
            assert engine.debug_partials(C) == orc.score_dims_fx(other, w=w)
            engine.score(C, 1)
            assert engine.debug_partials(C) == orc.score_dims_fx(dims, w=w)
    finally:
        engine.set_weights(orc.weights())
