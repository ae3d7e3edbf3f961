"""GPU: the CUDA path against the compiled reference across jconf options beyond the committed golden cases --
the device-side twin of tests/test_oracle_sweep.py.  Each case's utterances (decoded by the compiled reference, stored
under tests/golden/sweep/) go through K1 + K3, which must reproduce the reference's state scores bit for bit and its
word trellis exactly.  Covers -iwcd1 avg / best N, -lmp, score-envelope pruning (-bs), -gprune heuristic, -iwsp,
transparent words, flattened tied-mixture codebooks and DFA grammars on the device."""
import numpy as np
import pytest

from julius_b200 import capi
from util import atoms_equal, load_sweep_case, scores_sha
from test_oracle_sweep import SWEEP, GRAMMAR_SWEEP

pytestmark = pytest.mark.gpu


def _room_for_atoms(monkeypatch, feats, utts):
    """the decoder keeps room for 64 trellis words a frame on average; the widest sweep cases (-b 2500) store more"""
    need = max(-(-len(u.atoms) // len(x)) + 1 for u, x in zip(utts, feats))
    if need > 64:
        monkeypatch.setenv("JB200_ATOMS_PER_FRAME", str(need))


def _check(r, u):
    ok, why = atoms_equal(r["atoms"], u.atoms)
    assert ok, why
    assert r["words"] == u.words and r["status"] == u.status and r["overflow"] == 0
    assert np.float32(r["score"]) == np.float32(u.score)


@pytest.mark.parametrize("preset,extra", SWEEP, ids=[" ".join([p] + e) for p, e in SWEEP])
def test_gpu_path_equals_compiled_reference(preset, extra, monkeypatch):
    ds, feats, utts = load_sweep_case(preset, extra)
    _room_for_atoms(monkeypatch, feats, utts)
    am = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
    for u, x in zip(utts, feats):
        assert scores_sha(am.score(x)) == u.outprob_sha256, "state scores differ from the reference"
    dec = capi.Decoder(ds, am, max_utts=4, max_frames=2048)
    for r, u in zip(dec.decode(feats), utts):
        _check(r, u)


# the GPU beam takes grammars on normal trees only (creation refuses -multipath loudly, tested in test_gpu_beam.py)
@pytest.mark.parametrize("extra", [e for e in GRAMMAR_SWEEP if "-multipath" not in e], ids=lambda e: " ".join(e))
def test_gpu_grammar_mode_equals_compiled_reference(extra, monkeypatch):
    ds, feats, utts = load_sweep_case("small", extra, grammar=True)
    _room_for_atoms(monkeypatch, feats, utts)
    am = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
    dec = capi.Decoder(ds, am, max_utts=4, max_frames=2048)
    for r, u in zip(dec.decode(feats), utts):
        _check(r, u)
