"""GPU: K1 (GMM state scoring) and the cd-set kernels on designed models, against the CPU restatement.

The models (tests/util.py, checked on the CPU in tests/test_gmm_design.py) cover every instantiated feature dimension,
ragged and empty states, tiles ending at exactly 64 Gaussians, NULL densities, far frames whose sums cross LOG_ZERO,
addlog designs at the LOG_ADDMIN cut and at table-index rounding edges, and the ties of the pruned top-N list."""
import numpy as np
import pytest
import torch

from julius_b200 import capi, desc
from util import EMPTY_STATE_PATTERNS, EXACT_ZERO_DESIGNS, GMM_DIMS, Golden, atoms_equal, design_gmm, gmm_tiles, \
    random_frames, random_gmm, random_gmm_counts, rel_err, tiles_per_cta

pytestmark = pytest.mark.gpu

PRUNE = [(0, 0)] + [(m, n) for m in (1, 2, 3) for n in (1, 2, 3, 4, 8, 16)]    # (gprune method, -tmix)
SENTINEL = 0x7FC0DEAD                       # the bits of a NaN no kernel writes (a positive int32)


def _model(kind, dim, prune):
    """-> (Descriptors, frames, names of the exact-zero design states or [])"""
    method, tmix = prune
    if kind == "random":
        blob = random_gmm(random_gmm_counts(dim), dim, seed=dim)
        x, zero = random_frames(dim, 300, seed=dim + 1), []
    else:
        blob, names = design_gmm(dim, seed=dim, tmix=tmix if method else None)
        x = random_frames(dim, 40, seed=dim + 1, n_far=0)
        # under -tmix 1 the index designs keep only their term 0, so they sum to exactly 0 as well
        zero = [s for s, n in enumerate(names) if n in EXACT_ZERO_DESIGNS or (tmix == 1 and str(n).startswith("index_"))]
    ds = desc.Descriptors(blob)
    ds.gmm.gprune_method, ds.gmm.gprune_num = method, tmix
    return ds, x, zero


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _first_diff(got, want):
    t, s = np.argwhere(_bits(got) != _bits(want))[0]
    return f"first difference at frame {t} state {s}: {got[t, s]!r} vs {want[t, s]!r}"


@pytest.mark.parametrize("prune", PRUNE, ids=lambda p: f"gprune{p[0]}_tmix{p[1]}")
@pytest.mark.parametrize("dim", GMM_DIMS)
@pytest.mark.parametrize("kind", ["random", "design"])
def test_exact_mode_is_bit_identical_to_restatement(kind, dim, prune, oracle_lib):
    ds, x, _ = _model(kind, dim, prune)
    got = capi.GmmScorer(ds, mode=capi.GMM_EXACT).score(x)
    want = oracle_lib.gmm_score(ds, x)
    assert np.array_equal(_bits(got), _bits(want)), _first_diff(got, want)


@pytest.mark.parametrize("prune", PRUNE, ids=lambda p: f"gprune{p[0]}_tmix{p[1]}")
@pytest.mark.parametrize("dim", GMM_DIMS)
@pytest.mark.parametrize("kind", ["random", "design"])
def test_fast_mode_within_1e4_relative(kind, dim, prune, oracle_lib):
    ds, x, zero = _model(kind, dim, prune)
    got = capi.GmmScorer(ds, mode=capi.GMM_FAST).score(x)
    want = oracle_lib.gmm_score(ds, x)
    # The exact-zero designs are left out: the reference turns a log-sum of exactly 0 into LOG_ZERO, and a log-sum a
    # rounding away from 0 into about 0, so no tolerance mode can follow it there.  The same holds at the floor: a
    # log-sum within rounding of LOG_ZERO becomes LOG_ZERO or LOG_ZERO * INV_LOG_TEN, so there both sides need only be
    # one of the two.
    keep = np.setdiff1d(np.arange(want.shape[1]), zero)
    got, want = got[:, keep], want[:, keep]
    floor = lambda a: (a == np.float32(-1e6)) | (rel_err(a, np.float32(-1e6 * 0.434294482)) <= 1e-4)
    err = np.where(floor(got) & floor(want), 0, rel_err(got, want))
    t, s = np.unravel_index(np.argmax(err), err.shape)
    assert err.max() <= 1e-4, f"max rel err {err.max():.3e} at frame {t} state {keep[s]}: {got[t, s]!r} vs {want[t, s]!r}"


def test_tile_walk_depth(oracle_lib):
    """T chosen so that each CTA walks 1, 2, 3, about 10 and all tiles of a ragged model with 60+ tiles; the frames are
    copies of one block of distinct frames, and every copy must equal the restatement's scores of the block"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    counts = random_gmm_counts(39)
    n_tiles = len(gmm_tiles(counts))
    assert n_tiles >= 60
    block_n = 509
    for prune in ((0, 0), (2, 3)):
        ds = desc.Descriptors(random_gmm(counts, 39, seed=39))
        ds.gmm.gprune_method, ds.gmm.gprune_num = prune
        block = random_frames(39, block_n, seed=7)
        ref = torch.from_numpy(_bits(oracle_lib.gmm_score(ds, block)).view(np.int32)).cuda()
        sc = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
        S = sc.n_states
        depths = {}
        for T in list(range(77, 60000, 256)) + [8 * sms * 256 + 77]:
            d = tiles_per_cta(T, n_tiles, sms)
            if d not in depths and (d <= 3 or 9 <= d <= 11 or d == n_tiles):
                depths[d] = T
        assert {1, 2, 3, n_tiles} <= set(depths) and any(9 <= d <= 11 for d in depths), depths
        xb = torch.from_numpy(block).cuda()
        for d, T in sorted(depths.items()):
            feats = xb.repeat(-(-T // block_n), 1)[:T].contiguous()
            rows = torch.full((T, sc.stride), SENTINEL, dtype=torch.int32, device="cuda")
            sc.score_device(feats.data_ptr(), T, rows.data_ptr())
            torch.cuda.synchronize()
            want = ref.repeat(-(-T // block_n), 1)[:T]
            bad = (rows[:, :S] != want).nonzero()
            assert len(bad) == 0, f"{prune} depth {d} T {T}: first difference at frame/state {bad[0].tolist()}"


def _write_models():
    for dim in GMM_DIMS:
        yield f"random_d{dim}", random_gmm(random_gmm_counts(dim), dim, seed=dim)
    for name, counts in EMPTY_STATE_PATTERNS.items():
        yield name, random_gmm(counts + [16, 12, 12], 39, seed=1)


@pytest.mark.parametrize("prune", [(0, 0), (1, 2)], ids=["none", "safe2"])
def test_every_state_and_cd_column_is_written(prune):
    """score_device into a buffer filled with a NaN sentinel: every state and cd column of every frame is written,
    including those of states without mixtures (a fresh scratch buffer could hide a missing write)"""
    for name, blob in _write_models():
        ds = desc.Descriptors(blob)
        ds.gmm.gprune_method, ds.gmm.gprune_num = prune
        sc = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
        dim, S, C = sc.dim, sc.n_states, sc.n_cdsets
        T = 300
        feats = torch.from_numpy(random_frames(dim, T, seed=3)).cuda()
        rows = torch.full((T, sc.stride), SENTINEL, dtype=torch.int32, device="cuda")
        sc.score_device(feats.data_ptr(), T, rows.data_ptr())
        torch.cuda.synchronize()
        miss = (rows[:, :S + C] == SENTINEL).any(0).nonzero().flatten().tolist()
        assert not miss, f"{name}: columns never written: {miss} (S = {S})"


CD_METHODS = [(0, 3), (1, 3)] + [(2, n) for n in (1, 2, 3, 4, 5, 8, 16)]    # (iwcd method, N)


def _cd_compare(got, want):
    """An all-LOG_ZERO set gives 0/0 under AVG and best N on both sides; the x86 and CUDA NaN bit patterns differ, so
    there NaN-ness is compared, elsewhere the bits."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(_bits(got)[~nan], _bits(want)[~nan]), \
        f"first difference at {np.argwhere((_bits(got) != _bits(want)) & ~nan)[0]}"


@pytest.mark.parametrize("method", CD_METHODS, ids=lambda m: f"iwcd{m[0]}_n{m[1]}")
def test_cdset_columns_match_restatement(method, oracle_lib):
    """cd sets of 1 member, fewer than, exactly and more than N members (up to 40), with ties and LOG_ZERO members;
    then T = 65 537 frames, across the kernel's 65 535-frame launch split"""
    for dim in (39, 26):
        ds = desc.Descriptors(random_gmm(random_gmm_counts(dim), dim, seed=dim))
        ds.gmm.iwcd_method, ds.gmm.iwcd_nbest = method
        sc = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
        S, C = sc.n_states, sc.n_cdsets
        x = random_frames(dim, 200, seed=11)
        rows = sc.score_rows(x)
        st = oracle_lib.gmm_score(ds, x)
        assert np.array_equal(_bits(rows[:, :S]), _bits(st))
        _cd_compare(rows[:, S:S + C], oracle_lib.cdset_score(ds, st))
    T = 65537
    block = x[:137]
    want = oracle_lib.cdset_score(ds, st[:137])
    feats = torch.from_numpy(block).cuda().repeat(-(-T // 137), 1)[:T].contiguous()
    out = torch.empty((T, sc.stride), dtype=torch.float32, device="cuda")
    sc.score_device(feats.data_ptr(), T, out.data_ptr())
    torch.cuda.synchronize()
    idx = np.r_[0:300, 65400:T]
    got = out[idx][:, S:S + C].cpu().numpy()
    _cd_compare(got, want[idx % 137])


@pytest.mark.parametrize("method", CD_METHODS, ids=lambda m: f"iwcd{m[0]}_n{m[1]}")
def test_beam_cdset_scores_on_designed_rows(method, oracle_lib):
    """the beam's own cd-set code (evaluated on demand) against the restatement: real scores on a 0.25 grid (ties),
    about 5 % of them LOG_ZERO, decoded on the small_b100 tree; frames where a set would be all LOG_ZERO are left out"""
    g = Golden("small_b100")
    ds = g.ds
    ds.gmm.iwcd_method, ds.gmm.iwcd_nbest = method
    cd_off, cd_states = g.blob["am.cd_off"], g.blob["am.cd_states"]
    rng = np.random.default_rng(method[0] * 100 + method[1])
    rows = []
    for u in g.utts:
        r = (np.round(u.outprob * 4) / 4).astype(np.float32)
        r[rng.random(r.shape) < 0.05] = np.float32(-1e6)
        dead = np.zeros(len(r), bool)
        for c in range(len(cd_off) - 1):
            dead |= (r[:, cd_states[cd_off[c]:cd_off[c + 1]]] <= np.float32(-1e6)).all(1)
        rows.append(np.ascontiguousarray(r[~dead]))
    am = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(ds, am, max_utts=8, max_frames=4096)
    for r, st in zip(dec.decode_scores(rows), rows):
        o = oracle_lib.beam_decode(ds, st, gmm=ds.gmm)
        ok, why = atoms_equal(r["atoms"], o["atoms"])
        assert ok, why
        assert r["words"] == o["words"]
