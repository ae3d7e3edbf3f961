"""GPU: K2 DNN-HMM forward (wgmma bf16x3 GEMM stack) through the C-ABI vs the reference's golden scores."""
import numpy as np
import pytest

from julius_b200 import capi
from julius_b200 import desc, synth
from util import DNN_CASES, Golden, atoms_equal, full_dnn_blob, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", DNN_CASES)
def test_dnn_scores_within_1e4_relative_of_reference(case):
    g = Golden(case)
    dnn = capi.DnnScorer(g.ds)
    for u, x in zip(g.utts, g.feats):
        out = dnn.score(x)
        assert out.shape == u.outprob.shape
        # tolerance: BASELINE.json north_star, 1e-4 relative with an absolute floor of 1 because DNN
        # pseudo-likelihoods cross zero (SURVEY 7, hard parts)
        err = rel_err(out, u.outprob, floor=1.0)
        assert err.max() <= 1e-4, f"max rel err {err.max():.3e}, max abs {np.abs(out - u.outprob).max():.3e}"


def test_dnn_ragged_batches():
    g = Golden("small_dnn")
    dnn = capi.DnnScorer(g.ds)
    x = g.feats[0]
    full = dnn.score(x)
    for T in (1, 5, 127, 129):
        part = dnn.score(x[:T])
        assert np.abs(part - full[:T]).max() <= 1e-5


@pytest.mark.parametrize("case", DNN_CASES)
def test_decode_with_dnn_scores_matches_reference_words(case):
    """DNN scoring -> GPU beam.  Scores differ from the reference by <=1e-4 so the trellis is compared
    through the beam run on the reference's own score matrix (bit-exact) and, end to end, by the
    pass-1 best word sequence.  small_dnn_iwsp = BASELINE configs[4] flavour (multipath tree, -iwsp, wide beam)."""
    g = Golden(case)
    am = capi.GmmScorer(g.ds, gmm_desc=g.ds.cd_only_gmm())
    dec = capi.Decoder(g.ds, am, max_utts=4, max_frames=2048)
    res = dec.decode_scores([u.outprob for u in g.utts])
    for r, u in zip(res, g.utts):
        ok, why = atoms_equal(r["atoms"], u.atoms)
        assert ok, why
        assert r["words"] == u.words
    dnn = capi.DnnScorer(g.ds)
    dec.attach_dnn(dnn)
    res = dec.decode(g.feats)
    for r, u in zip(res, g.utts):
        assert r["overflow"] == 0 and r["status"] == u.status
        assert r["words"] == u.words
        assert abs(r["score"] - u.score) <= 1e-4 * abs(u.score) + 0.05


@pytest.fixture(scope="module")
def full_dnn():
    return desc.Descriptors(full_dnn_blob())


@pytest.mark.parametrize("T", [1, 127, 129, 300, 1100, 2200])
def test_dnn_full_shape_within_1e4_of_the_oracle(full_dnn, T, oracle_lib):
    """K2 at the BASELINE configs[3] shape, 528 -> 7 x 2048 -> 3000: 32 k-blocks per hidden layer, a partial last
    column block (3000 = 23 x 128 + 56), ragged frame counts around the 128-row tile.  The GEMM runs one persistent CTA per
    SM at most: T = 1100 gives 9 x 16 hidden-layer and 9 x 24 last-layer tiles, T = 2200 18 x 16 and 18 x 24, more than the
    132 SMs of an H100 in both, so CTAs take a second (and third) tile -- the operand ring carried across tiles, the next
    tile's loads issued during an epilogue, the accumulator restarted at each tile's first k-step.
    The checker is the CPU restatement of dnn_calc_outprob (calc_dnn.c:774-868), itself pinned bit-exact to the
    compiled reference on the golden DNN cases."""
    x = synth.sample_dnn_input(np.random.default_rng(100 + T), T, 528)
    want = oracle_lib.dnn_score(full_dnn, x)
    dnn = capi.DnnScorer(full_dnn)
    got = dnn.score(x)
    assert got.shape == want.shape == (T, 3000)
    err = rel_err(got, want, floor=1.0)
    assert err.max() <= 1e-4, f"max rel err {err.max():.3e}, max abs {np.abs(got - want).max():.3e}"
