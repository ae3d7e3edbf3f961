"""GPU: K1 GMM state scoring through the C-ABI vs the oracle / the reference's golden scores."""
import numpy as np
import pytest

from julius_b200 import capi, desc
from util import CASES, GMM_DIMS, Golden, random_frames, random_gmm, random_gmm_counts, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES)
def test_gmm_exact_mode_is_bit_identical_to_reference(case):
    g = Golden(case)
    sc = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    for u, x in zip(g.utts, g.feats):
        out = sc.score(x)
        assert np.array_equal(out.view(np.uint32), u.outprob.view(np.uint32)), \
            f"max abs diff {np.abs(out - u.outprob).max()}"


@pytest.mark.parametrize("case", CASES)
def test_gmm_fast_mode_within_1e4_relative(case):
    g = Golden(case)
    sc = capi.GmmScorer(g.ds, mode=capi.GMM_FAST)
    for u, x in zip(g.utts, g.feats):
        out = sc.score(x)
        # tolerance from BASELINE.json north_star: 1e-4 relative on float log-likelihoods
        assert rel_err(out, u.outprob).max() <= 1e-4


def test_cdset_columns_match_oracle(oracle_lib):
    g = Golden("small_b100")
    sc = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    rows = sc.score_rows(g.feats[0])
    S, Cn = sc.n_states, sc.n_cdsets
    want = oracle_lib.cdset_score(g.ds, g.utts[0].outprob)
    assert np.array_equal(rows[:, :S].view(np.uint32), g.utts[0].outprob.view(np.uint32))
    assert np.array_equal(rows[:, S:S + Cn].view(np.uint32), want.view(np.uint32))


def test_ragged_and_tiny_batches(oracle_lib):
    g = Golden("tiny")
    sc = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    x = g.feats[0]
    for T in (1, 2, 127, 129):
        out = sc.score(x[:T])
        assert np.array_equal(out, g.utts[0].outprob[:T])


def _check_gauss_hook(b, ds, x):
    """the device's per-Gaussian scores of frame x against a float32 loop in the reference's statement order; a NULL
    density scores LOG_ZERO"""
    sc = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
    got = sc.gauss(x)
    D = b["gmm.dim"][0]
    mean = b["gmm.mean"].reshape(-1, D); iv = b["gmm.ivar"].reshape(-1, D)
    want = np.empty(len(mean), np.float32)
    for k in range(len(mean)):
        tmp = np.float32(b["gmm.gconst"][k])
        for d in range(D):
            xx = np.float32(x[d] - mean[k, d])
            tmp = np.float32(tmp + np.float32(np.float32(xx * xx) * iv[k, d]))
        want[k] = np.float32(tmp * np.float32(-0.5)) if b["gmm.valid"][k] else np.float32(-1e6)
    assert np.array_equal(got, want)


def test_gauss_hook_contract(oracle_lib):
    """calcmix contract: per-Gaussian ln scores without mixture weight (plugin/calcmix.c:226-323)."""
    g = Golden("tiny")
    _check_gauss_hook(g.blob, g.ds, g.feats[0][7])


@pytest.mark.parametrize("dim", GMM_DIMS)
def test_gauss_hook_contract_at_each_dimension(dim):
    """the same contract on a ragged random model with NULL densities at each dimension K1 is built for"""
    blob = random_gmm(random_gmm_counts(dim), dim, seed=dim)
    assert (blob["gmm.valid"] == 0).any()
    _check_gauss_hook(blob, desc.Descriptors(blob), random_frames(dim, 1, seed=dim, n_far=0)[0])


def test_large_batch_linearity_property():
    """Full-size property check (3000 states x 16 mix is covered in test_gpu_full): scoring a
    concatenation equals concatenating the scores (frames are independent)."""
    g = Golden("small_b100")
    sc = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    cat = np.concatenate(g.feats, 0)
    big = np.tile(cat, (8, 1))
    out = sc.score(big)
    ref = np.concatenate([u.outprob for u in g.utts], 0)
    assert np.array_equal(out, np.tile(ref, (8, 1)))
