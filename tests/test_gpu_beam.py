"""GPU: K3 pass-1 beam through the C-ABI.  Bit-exact word trellis vs the compiled reference's
golden outputs (same score matrix on both sides) and end to end (GPU scores -> GPU beam)."""
import numpy as np
import pytest

from julius_b200 import capi
from util import CASES, Golden, atoms_equal

pytestmark = pytest.mark.gpu


def _check(r, u):
    assert r["overflow"] == 0
    ok, why = atoms_equal(r["atoms"], u.atoms)
    assert ok, why
    assert r["status"] == u.status
    assert r["words"] == u.words
    assert np.float32(r["score"]) == np.float32(u.score)


@pytest.mark.parametrize("case", CASES)
def test_beam_on_reference_scores_is_bit_exact(case):
    """Feed the reference's own [T x S] score matrix to the GPU beam: trellis must be identical."""
    g = Golden(case)
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
    res = dec.decode_scores([u.outprob for u in g.utts])
    for r, u in zip(res, g.utts):
        _check(r, u)


@pytest.mark.parametrize("case", CASES)
def test_end_to_end_exact_mode_matches_reference(case):
    """Host features -> GPU GMM (exact mode) -> GPU beam -> host trellis == reference run."""
    g = Golden(case)
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
    res = dec.decode(g.feats)
    for r, u in zip(res, g.utts):
        _check(r, u)


def test_batch_order_and_repeat_are_deterministic():
    g = Golden("small_b100")
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=16, max_frames=8192)
    feats = g.feats + g.feats[::-1] + g.feats
    utts = g.utts + g.utts[::-1] + g.utts
    for _ in range(2):                      # second pass reuses the node-slot work areas
        res = dec.decode(feats)
        for r, u in zip(res, utts):
            _check(r, u)


def test_multipath_work_areas_are_clean_after_each_batch():
    """the multipath kernel leaves node slots set in its unfinished last frame and must reset them"""
    g = Golden("small_mp")
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
    for feats, utts in ((g.feats, g.utts), (g.feats[::-1], g.utts[::-1]), (g.feats, g.utts)):
        for r, u in zip(dec.decode(feats), utts):
            _check(r, u)


@pytest.mark.parametrize("case", ["tiny", "small_mp"])
def test_ragged_lengths_and_single_frame(case):
    g = Golden(case)
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=2048)
    from oracle import ffi
    x = g.feats[0]
    lens = [1, 2, 3, 17, 100]
    res = dec.decode([x[:n] for n in lens])
    for r, n in zip(res, lens):
        o = ffi.beam_decode(g.ds, g.utts[0].outprob[:n])
        ok, why = atoms_equal(r["atoms"], o["atoms"])
        assert ok, f"T={n}: {why}"
        assert r["status"] == o["status"] and r["words"] == o["words"]


@pytest.mark.parametrize("case", ["small_b100", "small_mp"])
def test_frame_counts_match_oracle_trace(case):
    g = Golden(case)
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=4, max_frames=4096)
    from oracle import ffi
    dec.decode_scores([g.utts[0].outprob])
    T = g.utts[0].n_frames
    c = dec.frame_counts(0, T)
    o = ffi.beam_decode(g.ds, g.utts[0].outprob, trace=True)["trace"]
    assert np.array_equal(c, o[:T])


def test_capacity_errors_are_loud():
    g = Golden("tiny")
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=1, max_frames=64)
    with pytest.raises(capi.Jb200Error):
        dec.decode([g.feats[0], g.feats[0]])
    with pytest.raises(capi.Jb200Error):
        dec.decode([g.feats[0]])          # 150 frames > 64


def test_fast_heap_replay_agrees_with_sequential_replay(monkeypatch):
    """JB200_CHECK_HEAP=1 makes the kernel run BOTH heap replays every frame (the sentinel/speculative-load
    one with the loser cut, and the plain in-place one) and flag any difference in the survivor order
    (overflow code 4)."""
    monkeypatch.setenv("JB200_CHECK_HEAP", "1")
    for case in ("small_b100", "small_safe"):
        g = Golden(case)
        am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
        dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
        res = dec.decode(g.feats)
        for r, u in zip(res, g.utts):
            _check(r, u)


def test_grammar_mode_trellis_matches_reference():
    g = Golden("small_dfa")
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
    for r, u in zip(dec.decode_scores([u.outprob for u in g.utts]), g.utts):
        _check(r, u)
    for r, u in zip(dec.decode(g.feats), g.utts):
        _check(r, u)


@pytest.mark.parametrize("case", ["small_tr", "small_tm"])
def test_cpu_pinned_cases_end_to_end_on_the_device(case):
    """transparent (filler) words and the flattened tied-mixture model: host features -> GPU scores -> GPU beam."""
    g = Golden(case)
    am = capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    for u, x in zip(g.utts, g.feats):
        sc = am.score(x)
        assert np.array_equal(sc.view(np.uint32), u.outprob.view(np.uint32))
    dec = capi.Decoder(g.ds, am, max_utts=8, max_frames=4096)
    for r, u in zip(dec.decode(g.feats), g.utts):
        _check(r, u)
