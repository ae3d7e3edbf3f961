"""GPU: decoder groups (jb200_group_*), Julius' multi-decoding.

Several recognition instances on one acoustic model read one score matrix per input (every RecogProcess on a PROCESS_AM
shares its HMMWork, m_fusion.c:1182).  A group scores each batch or stream feed once and runs every active member's beam
on the group's rows, so each member must decode bit for bit what it decodes on its own, whatever its tree kind, beam
width or LM weight, and a group call must cost one scoring plus one beam launch per member."""
import numpy as np
import pytest
import torch

from julius_b200 import capi, desc, synth
from oracle import ffi
from util import Golden, atoms_equal

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY = -1, -5
CASES = ["small_b100", "small_mp", "small_dfa"]
# Members on one scorer: small_b100 and small_mp have identical gmm.* and am.* entries (Gaussians and pseudo-phone sets);
# small_dfa was exported with another pseudo-phone set layout (-iwcd1), so its grammar trees get a scorer of their own.
# Each set: (case whose model builds the scorer, members as (case, tree overrides)).
SETS = {"ngram": ("small_b100", [("small_b100", {}), ("small_mp", {}), ("small_b100", dict(beam_width=40, lm_weight=10.0))]),
        "grammar": ("small_dfa", [("small_dfa", {}), ("small_dfa", dict(beam_width=40))])}


def _same(r, w, what):
    assert r["overflow"] == 0 and w["overflow"] == 0, what
    assert r["status"] == w["status"], what
    assert r["n_frames"] == w["n_frames"], what
    assert np.float32(r["score"]).view(np.uint32) == np.float32(w["score"]).view(np.uint32), what
    ok, why = atoms_equal(r["atoms"], w["atoms"])
    assert ok, f"{what}: {why}"
    assert r["words"] == w["words"], what


def _same_as_golden(r, u, what):
    ok, why = atoms_equal(r["atoms"], u.atoms)
    assert ok, f"{what}: {why}"
    assert r["status"] == u.status and r["words"] == u.words, what
    assert np.float32(r["score"]) == np.float32(u.score), what


def _variant(blob, **tree):
    """the model with some tree.* scalars replaced (same dtype)"""
    b = dict(blob)
    for k, v in tree.items():
        b["tree." + k] = np.array([v], b["tree." + k].dtype)
    return desc.Descriptors(b)


@pytest.fixture(scope="module")
def goldens():
    return {c: Golden(c) for c in CASES}


def _member_set(goldens, name):
    """one scorer, its members and their own decodes of the union of the goldens' utterances; owner[u] = (case, index)
    of utterance u, golden[k] = the case member k is the unmodified model of (None for a variant)"""
    am_case, members = SETS[name]
    am = capi.GmmScorer(goldens[am_case].ds, mode=capi.GMM_EXACT)
    dss = [_variant(goldens[c].blob, **kw) if kw else goldens[c].ds for c, kw in members]
    feats, owner = [], []
    for c in CASES:
        for i, x in enumerate(goldens[c].feats):
            feats.append(x); owner.append((c, i))
    n, mf = len(feats), sum(len(x) for x in feats)
    decs = [capi.Decoder(ds, am, max_utts=n, max_frames=mf) for ds in dss]
    own = [d.decode(feats) for d in decs]
    return dict(am=am, dss=dss, decs=decs, feats=feats, owner=owner, own=own, golden=[None if kw else c for c, kw in members])


@pytest.fixture(scope="module")
def mixed(goldens):
    """the N-gram set: normal and multipath trees, and the normal tree at beam width 40 and LM weight 10"""
    return _member_set(goldens, "ngram")


@pytest.mark.parametrize("which", ["ngram", "grammar"])
def test_group_equals_own_decodes_the_restatement_and_the_goldens(which, mixed, goldens):
    ms = mixed if which == "ngram" else _member_set(goldens, which)
    decs, feats, owner, own = ms["decs"], ms["feats"], ms["owner"], ms["own"]
    g = capi.DecoderGroup(decs)
    off = np.zeros(len(feats) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in feats])
    cat = np.ascontiguousarray(np.concatenate(feats), np.float32)
    d_cat = torch.from_numpy(cat).cuda()
    # the golden state-score matrices (bit-identical to the scorer's: the gmm.* entries are the same) for the score-row
    # entry point and the restatement
    scores = [goldens[c].utts[i].outprob for c, i in owner]
    runs = {"host": g.decode(feats), "scores": g.decode_scores(scores)}
    g.decode_device(d_cat.data_ptr(), off)
    runs["device"] = [d.results() for d in decs]
    for k, ds in enumerate(ms["dss"]):
        for u, (c, i) in enumerate(owner):
            o = ffi.beam_decode(ds, goldens[c].utts[i].outprob)
            for name, res in runs.items():
                r = res[k][u]
                what = f"{name}: member {k}, utterance {u} ({c}/{i})"
                _same(r, own[k][u], what)
                ok, why = atoms_equal(r["atoms"], o["atoms"])
                assert ok, f"{what} vs restatement: {why}"
                assert r["words"] == o["words"], what
                if ms["golden"][k] == c:
                    _same_as_golden(r, goldens[c].utts[i], what + " vs golden")
    t = g.timing()
    assert t["score"] > 0 and t["beams"] > 0
    g.close()


def test_a_group_batch_costs_one_scoring_and_one_beam_per_member(mixed):
    decs, feats = mixed["decs"], mixed["feats"]
    decs[0].decode(feats)                                   # warm
    c0 = capi.launch_count()
    decs[0].decode(feats)
    single = capi.launch_count() - c0
    for n in (1, 2, 3):
        g = capi.DecoderGroup(decs[:n])
        g.decode(feats)                                     # warm
        c0 = capi.launch_count()
        g.decode(feats)
        assert capi.launch_count() - c0 == single + n - 1, n
        g.close()


def test_an_inactive_member_is_skipped_and_keeps_its_results(mixed):
    decs, feats, own = mixed["decs"], mixed["feats"], mixed["own"]
    g = capi.DecoderGroup(decs[:3])
    first = g.decode(feats[:2])
    g.set_active(1, False)
    c0 = capi.launch_count()
    got = g.decode(feats)
    launches = capi.launch_count() - c0
    g.set_active(1, True)
    c0 = capi.launch_count()
    g.decode(feats)
    assert launches == capi.launch_count() - c0 - 1
    assert got[1] is None
    for u, r in enumerate(decs[1].results(2)):              # still the two-utterance batch of the first call
        _same(r, first[1][u], f"inactive member, utterance {u}")
    for k in (0, 2):
        for u, r in enumerate(got[k]):
            _same(r, own[k][u], f"member {k}, utterance {u}")
    g.close()


def test_dnn_group_with_device_splice():
    gd = Golden("small_dnn")
    ctx = 3
    fl = gd.ds.dnn.in_dim // ctx
    am = capi.GmmScorer(gd.ds, gmm_desc=gd.ds.cd_only_gmm())
    dnn = capi.DnnScorer(gd.ds, context_len=ctx)
    dss = [gd.ds, _variant(gd.blob, beam_width=max(8, gd.ds.tree.beam_width // 2))]
    rng = np.random.default_rng(5)
    utts = [np.ascontiguousarray(x[:, :fl]) for x in gd.feats] + [synth.sample_dnn_input(rng, n, fl) for n in (90, ctx, ctx - 1)]
    decs = []
    for ds in dss:
        d = capi.Decoder(ds, am, max_utts=len(utts), max_frames=4096)
        d.attach_dnn(dnn)
        decs.append(d)
    own = [d.decode(utts) for d in decs]
    g = capi.DecoderGroup(decs)
    got = g.decode(utts)
    for k in range(2):
        for u, r in enumerate(got[k]):
            _same(r, own[k][u], f"member {k}, utterance {u}")
    # decoders sharing the DNN, each on its own stream with no synchronisation between them: the handle orders its
    # forwards, whose activation buffers it holds once
    off = np.zeros(len(utts) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in utts])
    d_cat = torch.from_numpy(np.ascontiguousarray(np.concatenate(utts), np.float32)).cuda()
    for d in decs:
        d.decode_device(d_cat.data_ptr(), off, fetch=False)
    g.decode_device(d_cat.data_ptr(), off, fetch=False)
    for k, d in enumerate(decs):
        for u, r in enumerate(d.results()):
            _same(r, own[k][u], f"shared DNN, member {k}, utterance {u}")
    # streams: the carry of the last ctx - 1 frames is kept once, in the group
    x = utts[0]
    want = []
    for d in decs:
        d.stream_open(1)
        for a in range(0, len(x), 7):
            d.stream_feed([x[a:a + 7]], last=[a + 7 >= len(x)])
        want.append(d.stream_result(0))
    g.stream_open(1)
    for a in range(0, len(x), 7):
        g.stream_feed([x[a:a + 7]], last=[a + 7 >= len(x)])
    for k, d in enumerate(decs):
        _same(d.stream_result(0), want[k], f"stream, member {k}")
    g.close()


def _pieces(T, size):
    return [(a, min(a + size, T)) for a in range(0, T, size)]


def _run_streams(feed, status, partial, result, members, feats, size):
    """every utterance on its own stream, fed size frames at a time with an interim result asked on every feed; returns
    per member the (status, partial) after every feed and the final results"""
    n = len(feats)
    plans = [_pieces(len(x), size) for x in feats]
    trace = [[] for _ in members]
    for step in range(max(len(p) for p in plans)):
        chunks, last = [], []
        for s in range(n):
            if step < len(plans[s]):
                a, b = plans[s][step]
                chunks.append(feats[s][a:b]); last.append(int(step == len(plans[s]) - 1))
            else:
                chunks.append(None); last.append(0)
        feed(chunks, last)
        for k, m in enumerate(members):
            trace[k].append([(status(m, s), partial(m, s)) for s in range(n)])
    return trace, [[result(m, s) for s in range(n)] for m in members]


@pytest.mark.parametrize("size", [1, 7, 10000])
def test_group_streams_equal_each_members_own_streams(mixed, size):
    decs = mixed["decs"]                                    # N-gram, multipath, narrow beam
    feats = mixed["feats"][:3]
    st, pa, re = (lambda m, s: m.stream_status(s)), (lambda m, s: m.stream_partial(s)), (lambda m, s: m.stream_result(s))
    want = []
    for d in decs:
        d.stream_open(len(feats))
        want.append(_run_streams(lambda c, l, d=d: d.stream_feed(c, last=l, interim=True), st, pa, re, [d], feats, size))
    g = capi.DecoderGroup(decs)
    g.stream_open(len(feats))
    trace, res = _run_streams(lambda c, l: g.stream_feed(c, last=l, interim=True), st, pa, re, decs, feats, size)
    for k in range(len(decs)):
        assert trace[k] == want[k][0][0], f"member {k}: status / partials differ"
        for s in range(len(feats)):
            _same(res[k][s], want[k][1][0][s], f"member {k}, stream {s}")
    g.close()


def test_group_stream_restart_and_inactive_member(mixed):
    decs = mixed["decs"][:2]
    x = mixed["feats"][0]
    want = []
    for d in decs:
        d.stream_open(1)
        d.stream_feed([x], last=[1])
        want.append(d.stream_result(0))
    g = capi.DecoderGroup(decs)
    g.stream_open(1)
    g.stream_feed([x[:50]], interim=True)
    g.stream_restart(0)                                      # the utterance starts over
    for a, b in _pieces(len(x), 33):
        g.stream_feed([x[a:b]], last=[b == len(x)])
    for k, d in enumerate(decs):
        _same(d.stream_result(0), want[k], f"restarted stream, member {k}")
    # member 1 inactive for the next utterance: it is neither restarted nor fed, and keeps the result of the last one
    g.set_active(1, False)
    g.stream_restart(0)
    y = mixed["feats"][1]
    g.stream_feed([y], last=[1])
    _same(decs[1].stream_result(0), want[1], "inactive member")
    fresh = capi.Decoder(mixed["dss"][0], mixed["am"], max_utts=1, max_frames=1024)
    _same(decs[0].stream_result(0), fresh.decode([y])[0], "active member")
    g.close()


def test_refusals_leave_the_device_alone(mixed):
    L = capi.lib()
    decs, feats = mixed["decs"], mixed["feats"]
    gs = Golden("small_safe")
    am_safe = capi.GmmScorer(gs.ds, mode=capi.GMM_EXACT)
    other = capi.Decoder(gs.ds, am_safe, max_utts=2, max_frames=512)
    gd = Golden("small_dnn")
    am_dnn = capi.GmmScorer(gd.ds, gmm_desc=gd.ds.cd_only_gmm())
    with_dnn = capi.Decoder(gd.ds, am_dnn, max_utts=2, max_frames=512)
    with_dnn.attach_dnn(capi.DnnScorer(gd.ds))
    plain = capi.Decoder(gd.ds, am_dnn, max_utts=2, max_frames=512)
    small = capi.Decoder(mixed["dss"][0], mixed["am"], max_utts=2, max_frames=512)

    def create(ms):
        hs = (capi.C.c_void_p * max(len(ms), 1))(*[m.handle_ptr() for m in ms])
        h = capi.C.c_void_p()
        rc = L.jb200_group_create(hs, len(ms), capi.C.byref(h))
        if rc == 0:
            L.jb200_group_destroy(h)
        return rc

    c0 = capi.launch_count()
    assert create([decs[0], other]) == ERR_ARG              # another jb200_gmm
    assert create([with_dnn, plain]) == ERR_ARG             # a DNN-attached member beside a plain one
    assert create([decs[0], decs[1], decs[0]]) == ERR_ARG   # the same decoder twice
    assert create([]) == ERR_ARG
    assert create(decs * 6) == ERR_ARG                      # more than 16 (and duplicates)
    assert capi.launch_count() == c0
    g = capi.DecoderGroup([decs[0], small])
    off = np.array([0, 200, 400, 600], np.int32)            # three utterances: over the smaller member's 2
    cat = np.ascontiguousarray(np.concatenate(feats[:3]), np.float32)
    c0 = capi.launch_count()
    assert L.jb200_group_decode_batch_host(g._h, capi._f(cat), off.ctypes.data_as(desc.I), 3) == ERR_CAPACITY
    assert L.jb200_group_decode_batch_host(g._h, capi._f(cat), off.ctypes.data_as(desc.I), 0) == ERR_ARG
    assert capi.launch_count() == c0
    g.stream_open(1)
    n_new = np.array([10], np.int32)
    last = np.zeros(1, np.uint8)
    c0 = capi.launch_count()
    assert L.jb200_stream_feed_host(small.handle_ptr(), capi._f(cat), n_new.ctypes.data_as(desc.I),
                                    last.ctypes.data_as(capi.C.POINTER(capi.C.c_uint8)), 0) == ERR_ARG
    assert capi.launch_count() == c0
    g.close()


def test_activity_changes_wait_for_the_end_of_the_utterance(mixed):
    """a member's stream that missed feeds (or got feeds the others did not) cannot go on: while one of its streams is
    inside an utterance, the group refuses to change whether it is active"""
    decs = mixed["decs"][:2]
    x = mixed["feats"][0]
    g = capi.DecoderGroup(decs)
    with pytest.raises(capi.Jb200Error, match="jb200_group_stream_feed"):
        g.stream_feed([x[:10]])                            # no stream_open yet
    g.stream_open(1)
    g.stream_feed([x[:50]])
    L = capi.lib()
    c0 = capi.launch_count()
    assert L.jb200_group_set_active(g._h, 1, 0) == ERR_ARG
    assert capi.launch_count() == c0
    g.stream_feed([x[50:]], last=[1])
    g.set_active(1, False)                                 # the utterance has ended
    g.set_active(1, True)
    g.stream_restart(0)
    g.stream_feed([x], last=[1])
    fresh = capi.Decoder(mixed["dss"][1], mixed["am"], max_utts=1, max_frames=1024)
    _same(decs[1].stream_result(0), fresh.decode([x])[0], "member 1 after an activity change between utterances")
    g.close()
