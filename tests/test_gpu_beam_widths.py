"""GPU: the beam cut (beam_cut / select_exact, the replay of sort_token_no_order) at every kind of beam width, in all
three beam kernels and both placements of the heap-select array, with the kernels' own self-check on
(JB200_CHECK_HEAP=1: every cut is compared with the plain sequential heap select, overflow code 4 on a difference).

Each golden case is decoded on the reference's score matrix at widths that reach the cut's edges: searches that find no
sentence end (1-3), fewer extractions than the replay keeps in flight and a histogram of a few bins (16, 17, 33), the golden width,
upward and downward cuts mixed (300), and only downward cuts with the heap in global memory (2500), plus the two widths
on either side of the shared/global placement.  The word trellis must be the CPU restatement's at the same width, and
so must the token count of every frame (the cut's output order is the next frame's visiting order, so a slip shows up
there first).  The CPU restatement itself is pinned to the compiled reference at these widths by the -b 2 / 17 / 300 /
2500 cases of tests/test_oracle_sweep.py."""
import functools
import os

import numpy as np
import pytest

from julius_b200 import capi
from util import Golden, atoms_equal

pytestmark = pytest.mark.gpu

GMM_CASES = ["tiny", "small_b100", "small_mp", "small_iwsp", "small_dfa", "small_tr", "small_userlm"]
CASES = GMM_CASES + ["small_dnn_iwsp"]
# one case per kernel also runs end to end from its features (GPU GMM -> GPU beam)
END_TO_END = {"small_b100", "small_mp", "small_dfa"}
FIXED_WIDTHS = [1, 2, 3, 16, 17, 33, 300, 2500]


def _kernel(ds):
    return "grammar" if ds.tree.lm_type == 1 else "multipath" if ds.tree.multipath else "normal"


def _heap_global(beam, n_start, smem_optin):
    """size_cut's placement rule (csrc/beam.cu): the heap-select array goes to global memory when it and the per-survivor
    offsets would take more than half of a block's shared memory"""
    maxt = (max(4 * beam + n_start, 5 * beam) + 64 + 3) & ~3
    return (maxt + 4) * 8 + (beam + 2) * 8 > (smem_optin - 2048) // 2


def _placement_edge(n_start):
    """(largest width whose heap stays in shared memory, smallest width that moves it to global memory)"""
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    lo, hi = 1, 1 << 16                    # shared at lo, global at hi
    assert not _heap_global(lo, n_start, optin) and _heap_global(hi, n_start, optin)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _heap_global(mid, n_start, optin):
            hi = mid
        else:
            lo = mid
    return lo, hi


@functools.lru_cache(maxsize=None)
def _golden(case):
    return Golden(case)


@functools.lru_cache(maxsize=None)
def _widths(case):
    t = _golden(case).ds.tree
    return sorted(set(FIXED_WIDTHS + [t.beam_width, *_placement_edge(t.n_start)]))


@functools.lru_cache(maxsize=None)
def _oracle(case, beam):
    from oracle import ffi
    g = _golden(case)
    g.ds.tree.beam_width = beam
    return [ffi.beam_decode(g.ds, u.outprob, trace=True) for u in g.utts]


def _decoder(g, beam, env):
    g.ds.tree.beam_width = beam
    am = (capi.GmmScorer(g.ds, gmm_desc=g.ds.cd_only_gmm()) if g.ds.gmm is None
          else capi.GmmScorer(g.ds, mode=capi.GMM_EXACT))
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return capi.Decoder(g.ds, am, max_utts=len(g.utts), max_frames=sum(len(u.outprob) for u in g.utts) + 64)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


# Near -b 2500 almost every word end of the small models survives: up to 250 trellis words a frame, more than the
# default room of 64 a frame on average, which the decoder reports as overflow 1 (test below).  The width tests give it room.
CHECK_ENV = {"JB200_CHECK_HEAP": "1", "JB200_ATOMS_PER_FRAME": "512"}


def _same(r, o, what):
    assert r["overflow"] == 0, f"{what}: overflow {r['overflow']} (4 = the self-check found a different cut)"
    ok, why = atoms_equal(r["atoms"], o["atoms"])
    assert ok, f"{what}: {why}"
    assert r["words"] == o["words"] and r["status"] == o["status"], what
    assert np.float32(r["score"]) == np.float32(o["score"]), what


def _compare_counts(c, tr, what):
    """frame_counts against the oracle trace, up to and including the frame where the search died (no tokens left)"""
    dead = np.nonzero(tr[:, 0] == 0)[0]
    n = int(dead[0]) + 1 if len(dead) else len(tr)
    assert np.array_equal(c[:n], tr[:n]), f"{what}: per-frame token counts differ first at frame " \
                                          f"{int(np.nonzero((c[:n] != tr[:n]).any(1))[0][0])}"
    return c[:n]


@functools.lru_cache(maxsize=None)
def _run(case, beam):
    """decode the reference's scores at this width (self-check on); returns what the cut did"""
    g = _golden(case)
    want = _oracle(case, beam)
    dec = _decoder(g, beam, CHECK_ENV)
    try:
        res = dec.decode_scores([u.outprob for u in g.utts])
    except capi.Jb200Error as e:
        raise AssertionError(f"{case} -b {beam}: {e}") from e
    cells = dict(up=0, down=0, none=0)
    for i, (r, o, u) in enumerate(zip(res, want, g.utts)):
        what = f"{case} -b {beam} utterance {i}"
        _same(r, o, what)
        c = _compare_counts(dec.frame_counts(i, len(u.outprob)), o["trace"], what)
        n = c[:, 0].astype(np.int64)
        up = beam < n - beam
        cells["up"] += int(up.sum())
        cells["down"] += int(((n > beam) & ~up).sum())
        cells["none"] += int((n <= beam).sum())
    hs, pl = dec.heap_stats(), dec.cut_placement()
    if case in END_TO_END:
        for i, (r, o) in enumerate(zip(dec.decode(g.feats), want)):
            _same(r, o, f"{case} -b {beam} utterance {i} from features")
    return dict(kernel=_kernel(g.ds), cells=cells, heap=hs, placement=pl)


@pytest.mark.parametrize("case", CASES)
def test_every_width_matches_restatement_with_self_check(case):
    for beam in _widths(case):
        _run(case, beam)


@pytest.mark.parametrize("case", ["tiny", "small_mp", "small_dfa"])
def test_heap_placement_follows_the_sizing_rule(case):
    """the two widths around the shared/global edge land on the side the rule predicts"""
    lo, hi = _placement_edge(_golden(case).ds.tree.n_start)
    assert not _run(case, lo)["placement"]["heap_global"]
    assert _run(case, hi)["placement"]["heap_global"]
    assert _run(case, 2500)["placement"]["heap_global"]


@pytest.mark.parametrize("case", ["small_b100", "small_mp"])
def test_trellis_capacity_overflow_is_reported(case):
    """At -b 2500 the utterances store more trellis words than the default room (64 a frame): the decoder must flag
    it (overflow 1) and end the utterance's search, not read the word ends it had no room to store."""
    g = _golden(case)
    want = _oracle(case, 2500)
    dec = _decoder(g, 2500, {"JB200_ATOMS_PER_FRAME": "64"})
    res = dec.decode_scores([u.outprob for u in g.utts])
    for r, o, u in zip(res, want, g.utts):
        assert r["overflow"] == (1 if len(o["atoms"]) > 64 * len(u.outprob) + 64 else 0)
    assert any(r["overflow"] for r in res)
    # the decoder stays usable: 10 frames fit
    from oracle import ffi
    short = [u.outprob[:10] for u in g.utts]
    for r, x in zip(dec.decode_scores(short), short):
        _same(r, ffi.beam_decode(g.ds, x), f"{case} -b 2500, 10 frames after an overflow")


def _coverage():
    tab = {}
    for case in CASES:
        for beam in _widths(case):
            s = _run(case, beam)
            t = tab.setdefault(s["kernel"], dict(up_closed=0, up_relocated=0, up_replay=0, down_shared=0, down_global=0,
                                                 global_whole_copy=0))
            h, pl = s["heap"], s["placement"]
            t["up_closed"] += h["closed_form"] - h["closed_form_relocated"]
            t["up_relocated"] += h["closed_form_relocated"]
            t["up_replay"] += h["upward_selects"] - h["closed_form"]
            t["down_global" if pl["heap_global"] else "down_shared"] += s["cells"]["down"]
            t["global_whole_copy"] += pl["whole_copy_replays"]
    return tab


def test_every_branch_of_the_cut_was_reached():
    """Per kernel, summed over all cases and widths above: each branch of the cut ran at least once, so the self-check
    and the trellis comparison above covered it.  The upward cut on a global-memory heap is not among them: the small
    models never hold more than 2 x 2500 tokens a frame; the full-size -b 4000 tests in test_gpu_full.py cover it."""
    tab = _coverage()
    print("\nbeam-cut coverage (frames / cuts):")
    for k, t in sorted(tab.items()):
        print(f"  {k:10s}", "  ".join(f"{n}={v}" for n, v in t.items()))
    assert set(tab) == {"normal", "multipath", "grammar"}
    for k, t in tab.items():
        for cell in ("up_closed", "up_relocated", "up_replay", "down_shared", "down_global", "global_whole_copy"):
            assert t[cell] > 0, f"{k} kernel: no {cell} cut in any case/width ({t})"
