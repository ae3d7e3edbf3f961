"""CPU: the restatement against the compiled reference itself, across jconf options beyond the committed golden
cases.  Each case's utterances were decoded by the compiled reference (tests/golden/make_golden.py sweep, stored under
tests/golden/sweep/); the restatement must reproduce its state scores bit for bit and its word trellis exactly."""
import os

import numpy as np
import pytest

from util import ROOT, atoms_equal, load_sweep_case, scores_sha

JREF = os.path.join(ROOT, "oracle", "_ref", "jref")

SWEEP = [
    ("small", ["-b", "80", "-iwcd1", "avg"]),
    ("small", ["-b", "80", "-iwcd1", "best", "5"]),
    ("small", ["-b", "120", "-lmp", "12.0", "-3.0"]),
    ("small", ["-b", "200", "-bs", "60"]),                       # score-envelope pruning (SCORE_PRUNING, beam.c:2718-2730)
    ("small", ["-multipath", "-b", "150", "-bs", "80"]),
    ("small_sp", ["-iwsp", "-b", "100", "-bs", "50", "-iwcd1", "avg"]),
    ("small", ["-gprune", "heuristic", "-tmix", "2", "-b", "90"]),
    ("small_tr", ["-multipath", "-b", "90"]),                    # transparent words on the multipath tree
    ("small_tm", ["-gprune", "none", "-b", "100"]),              # tied-mixture codebooks, calc_tied_mix.c:161-248
    ("small_tm", ["-gprune", "safe", "-tmix", "2", "-b", "80", "-multipath"]),
]
# beam widths at the edges of the beam cut (tests/test_gpu_beam_widths.py decodes the golden cases at the same widths
# against the restatement): a search that finds no sentence end (-b 2), fewer than 16 extractions in flight and a small histogram
# (-b 17), upward and downward cuts mixed (-b 300), only downward cuts and, on the device, the heap in global memory (-b 2500)
WIDTHS = ["2", "17", "300", "2500"]
SWEEP += [("small", ["-b", b]) for b in WIDTHS] + [("small", ["-multipath", "-b", b]) for b in WIDTHS]


GRAMMAR_SWEEP = [["-b", "100"], ["-b", "60", "-penalty1", "-2.5", "-iwcd1", "max"], ["-b", "150", "-multipath", "-penalty1", "1.5"]]
GRAMMAR_SWEEP += [["-b", b] for b in WIDTHS]


@pytest.mark.parametrize("extra", GRAMMAR_SWEEP, ids=[" ".join(e) for e in GRAMMAR_SWEEP])
def test_grammar_mode_restatement_equals_compiled_reference(extra, oracle_lib):
    """Grammar (DFA) recognition: category tree, category-pair constraint, insertion penalty, all sentence-initial
    words alive at frame 0, best atom of the last frame as the pass-1 result (beam.c:1669-1760, :2404-2455, :435-458)."""
    ds, feats, utts = load_sweep_case("small", extra, grammar=True)
    assert ds.tree.lm_type == 1 and ds.tree.n_shared == 0 and ds.tree.n_init >= 1
    for x, u in zip(feats, utts):
        sc = oracle_lib.gmm_score(ds, x)
        assert scores_sha(sc) == u.outprob_sha256, "state scores differ from the reference"
        r = oracle_lib.beam_decode(ds, sc)
        ok, why = atoms_equal(r["atoms"], u.atoms)
        assert ok, why
        assert r["words"] == u.words and r["status"] == u.status
        assert np.float32(r["score"]) == np.float32(u.score)


@pytest.mark.skipif(not os.path.exists(JREF), reason="compiled reference (oracle/_ref/jref) not present")
def test_tied_mixture_with_history_dependent_pruning_is_refused(tmp_path):
    """-gprune beam (the default) on a tied-mixture AM seeds each codebook's pruning with the previous frame's best
    ids, so its scores depend on which frames the search evaluated; the exporter must refuse rather than approximate."""
    from oracle import fixtures
    with pytest.raises(RuntimeError):
        fixtures.make_fixture("small_tm", str(tmp_path), n_utts=1, n_frames=50, extra_args=["-b", "60"])
    assert not (tmp_path / "model.jb2m").exists()


@pytest.mark.parametrize("preset,extra", SWEEP, ids=[" ".join([p] + e) for p, e in SWEEP])
def test_restatement_equals_compiled_reference(preset, extra, oracle_lib):
    ds, feats, utts = load_sweep_case(preset, extra)
    for u, x in zip(utts, feats):
        sc = oracle_lib.gmm_score(ds, x)
        assert scores_sha(sc) == u.outprob_sha256, "state scores differ from the reference"
        r = oracle_lib.beam_decode(ds, sc)
        ok, why = atoms_equal(r["atoms"], u.atoms)
        assert ok, why
        assert r["words"] == u.words and r["status"] == u.status
        assert np.float32(r["score"]) == np.float32(u.score)
