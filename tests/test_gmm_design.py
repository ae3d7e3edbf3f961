"""CPU: the designed GMMs of tests/test_gpu_gmm_shapes.py are what they claim to be.  Each addlog design hits its edge
(the LOG_ADDMIN cut by one ulp, table indices just below and just above an integer), and the restatement of calc_mix
gives, bit for bit, what numpy gives from the designed terms through addlog_array and the finish rule of calc_mix.c.
Where the two disagreed the design or the restatement would be wrong, so this is settled before any GPU comparison."""
import numpy as np
import pytest

from julius_b200 import desc
from util import ADDMIN_DROPPED, ADDMIN_KEPT, EMPTY_STATE_PATTERNS, GMM_DIMS, LOG_ADDMIN, TILE_GAUSS, TILE_STATES, \
    TILING_PATTERN, addlog_array_np, addlog_designs, addlog_table_np, design_gmm, finish_np, gmm_tiles, \
    index_rounding_diffs, prune_designs, random_frames, random_gmm, random_gmm_counts

TMIX = [1, 2, 3, 4, 8, 16]


@pytest.fixture(scope="module")
def tbl(oracle_lib):
    t = addlog_table_np()
    assert np.array_equal(t, oracle_lib.addlog_table())
    return t


def test_addmin_pairs_straddle_the_cut_by_one_ulp():
    assert float(ADDMIN_KEPT) >= LOG_ADDMIN > float(ADDMIN_DROPPED)
    assert np.nextafter(ADDMIN_DROPPED, np.float32(0)) == ADDMIN_KEPT
    d = addlog_designs()
    for name, want in (("addmin_kept", ADDMIN_KEPT), ("addmin_dropped", ADDMIN_DROPPED)):
        a, b = d[name]
        assert np.float32(b - a) == want, name                  # the walk's difference is the designed float


def test_index_designs_land_on_both_sides_of_an_integer():
    d = index_rounding_diffs()
    r = (-d).astype(np.float64) * 33333.3333 + 0.5
    frac = r - np.rint(r)
    ulp = np.spacing(r.astype(np.float32)).astype(np.float64)
    assert (np.abs(frac) < 4 * ulp).all()
    assert (frac < 0).sum() >= 2 and (frac > 0).sum() >= 2
    # the same index taken in float arithmetic lands on the other side of the integer
    i_f = (np.float32(-d) * np.float32(33333.3333) + np.float32(0.5)).astype(np.int64)
    assert (i_f != r.astype(np.int64)).all()
    assert (d > LOG_ADDMIN).all()


def test_tiling_pattern_covers_its_edges():
    """every state is in exactly one tile; the pattern has a tile ending at exactly 64 Gaussians, a 64-mixture state,
    a split at 65, empty states after a full 4-state tile, and more than 4 one-mixture states in a row"""
    for counts in [TILING_PATTERN, random_gmm_counts(1)] + list(EMPTY_STATE_PATTERNS.values()):
        tiles = gmm_tiles(counts)
        assert sum(ns for _, ns, _ in tiles) == len(counts) and tiles[0][0] == 0
        assert all(t[0] + t[1] == u[0] for t, u in zip(tiles, tiles[1:]))
        assert all(0 < ng <= TILE_GAUSS for _, _, ng in tiles)
        assert all(sum(c > 0 for c in counts[s:s + n]) <= TILE_STATES for s, n, _ in tiles)
    tiles = gmm_tiles(TILING_PATTERN)
    assert sum(ng == TILE_GAUSS and ns > 1 for _, ns, ng in tiles) >= 2
    assert 64 in TILING_PATTERN and "40, 25" in str(TILING_PATTERN)
    assert any(counts[-1] == 0 and sum(c > 0 for c in counts) == 4 for counts in EMPTY_STATE_PATTERNS.values())


@pytest.mark.parametrize("dim", GMM_DIMS)
def test_addlog_designs_replay_bit_for_bit(dim, tbl, oracle_lib):
    blob, names = design_gmm(dim, seed=dim)
    x = random_frames(dim, 5, seed=dim, n_far=0)
    got = oracle_lib.gmm_score(desc.Descriptors(blob), x)
    designs = addlog_designs()
    for s, name in enumerate(names):
        want = np.full(len(x), -1e6, np.float32) if name is None else \
            np.repeat(finish_np(addlog_array_np(designs[name][None], tbl)), len(x))
        assert np.array_equal(got[:, s].view(np.uint32), want.view(np.uint32)), name


@pytest.mark.parametrize("tmix", TMIX)
def test_prune_designs_keep_the_designed_list(tmix, tbl, oracle_lib):
    """-tmix: the restatement's sum is that of the designed top-N list (ids, order and weights)"""
    blob, names = design_gmm(39, seed=tmix, tmix=tmix)
    ds = desc.Descriptors(blob)
    ds.gmm.gprune_method, ds.gmm.gprune_num = 1, tmix
    got = oracle_lib.gmm_score(ds, random_frames(39, 3, seed=tmix, n_far=0))
    for name, (sc, lnw, kept) in prune_designs(tmix).items():
        terms = (sc[kept] + lnw[kept]).astype(np.float32)
        want = finish_np(addlog_array_np(terms[None], tbl))[0]
        s = names.index(name)
        assert (got[:, s].view(np.uint32) == want.view(np.uint32)).all(), name


def test_random_models_reach_their_edges(oracle_lib):
    """NULL densities, an all-NULL state, empty states, and far frames on both sides of LOG_ZERO"""
    counts = random_gmm_counts(1)
    blob = random_gmm(counts, 39, seed=1)
    v = blob["gmm.valid"]
    assert 0.05 < 1 - v.mean() < 0.2
    got = oracle_lib.gmm_score(desc.Descriptors(blob), random_frames(39, 64, seed=2))
    empty = np.asarray(counts) == 0
    assert (got[:, empty] == np.float32(-1e6)).all()
    far = got[-32:, ~empty]
    assert (far == np.float32(-1e6)).any() and (far > np.float32(-1e6)).any()
