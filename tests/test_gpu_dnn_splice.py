"""GPU: DNN-HMM input as front-end frames (jb200_dnn_set_context): the context window is spliced on the device.

Julius splices context_len consecutive front-end frames into each network input (wav2mfcc.c:160-183, splice_mfcc
realtime-1stpass.c:445-460): decoded frame t is concat(x[t], ..., x[t + ctx - 1]), left-aligned and unpadded, so N input
frames decode max(0, N - ctx + 1) frames.  Whatever the entry point -- scorer, batch decoder or streams -- the result must
be bit for bit that of the same DNN with context 1 on the vectors spliced on the host."""
import numpy as np
import pytest

from julius_b200 import capi, desc, synth
from util import DNN_CASES, Golden, atoms_equal, full_dnn_blob, rel_err

pytestmark = pytest.mark.gpu

CTX = {"small_dnn": 3, "small_dnn_iwsp": 3, "full": 11}     # dnnconf context_len of each model (40 x 3, 48 x 11)


def splice(f, ctx):
    """host splice: row t = frames t .. t + ctx - 1, for t in [0, N - ctx + 1)"""
    T = max(0, len(f) - ctx + 1)
    return np.ascontiguousarray(np.concatenate([f[j:j + T] for j in range(ctx)], axis=1), np.float32)


@pytest.fixture(scope="module")
def models():
    out = {c: Golden(c).ds for c in DNN_CASES}
    out["full"] = desc.Descriptors(full_dnn_blob())
    return out


@pytest.fixture(scope="module")
def scorers(models):
    """one context-1 and one splicing handle per model, created on first use"""
    cache = {}

    def get(case, ctx):
        if (case, ctx) not in cache:
            cache[(case, ctx)] = capi.DnnScorer(models[case], context_len=ctx)
        return cache[(case, ctx)]
    return get


@pytest.mark.parametrize("case", DNN_CASES + ["full"])
@pytest.mark.parametrize("extra", [-1, 0, 1, 127, 129, 999])
def test_scores_equal_the_host_spliced_input(case, extra, models, scorers, oracle_lib):
    """N = ctx + extra input frames: ctx - 1 (no window), ctx, ctx + 1, 128 + ctx - 1, 129 + ctx, 1000 + ctx - 1"""
    ctx = CTX[case]
    N = ctx + extra
    fl = models[case].dnn.in_dim // ctx
    x = synth.sample_dnn_input(np.random.default_rng(1000 * ctx + N), N, fl)
    got = scorers(case, ctx).score(x)
    xs = splice(x, ctx)
    assert got.shape == (max(0, N - ctx + 1), models[case].dnn.out_dim)
    if len(xs) == 0:
        return
    want = scorers(case, 1).score(xs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    ref = oracle_lib.dnn_score(models[case], xs)
    err = rel_err(got, ref, floor=1.0)
    assert err.max() <= 1e-4, f"max rel err {err.max():.3e}"


def test_set_context_rejects_what_it_cannot_honour(models):
    L = capi.lib()
    ds = models["small_dnn"]                                   # in_dim 120
    d = capi.DnnScorer(ds)
    assert L.jb200_dnn_set_context(d.handle, 0) == -1
    assert L.jb200_dnn_set_context(d.handle, -3) == -1
    assert L.jb200_dnn_set_context(d.handle, 7) == -1          # 120 % 7 != 0
    assert L.jb200_dnn_set_context(d.handle, 3) == 0
    assert L.jb200_dnn_set_context(d.handle, 1) == 0           # still unused: the layout may change
    d.score(np.zeros((4, 120), np.float32))
    assert L.jb200_dnn_set_context(d.handle, 3) == -1          # it has scored frames
    e = capi.DnnScorer(ds)
    am = capi.GmmScorer(ds, gmm_desc=ds.cd_only_gmm())
    dec = capi.Decoder(ds, am, max_utts=1, max_frames=64)
    dec.attach_dnn(e)
    assert L.jb200_dnn_set_context(e.handle, 3) == -1          # it is attached to a decoder
    with pytest.raises(capi.Jb200Error):
        capi.DnnScorer(ds, context_len=0)


def _same(r, w, what):
    assert r["overflow"] == 0 and w["overflow"] == 0, what
    assert r["status"] == w["status"], what
    assert r["n_frames"] == w["n_frames"], what
    assert np.float32(r["score"]).view(np.uint32) == np.float32(w["score"]).view(np.uint32), what
    ok, why = atoms_equal(r["atoms"], w["atoms"])
    assert ok, f"{what}: {why}"
    assert r["words"] == w["words"], what


def _utterances(g, ctx, fl, rng):
    """five utterances of input frames: two taken from the golden vectors, a random one, one of ctx - 1 frames (no
    window) and one of exactly ctx frames (one decoded frame)"""
    return [np.ascontiguousarray(g.feats[0][:, :fl]), np.ascontiguousarray(g.feats[1][:, :fl]),
            synth.sample_dnn_input(rng, 90, fl), synth.sample_dnn_input(rng, ctx - 1, fl), synth.sample_dnn_input(rng, ctx, fl)]


def _decoders(g, ctx, n):
    """a decoder on a splicing DNN and one on a context-1 DNN of the same net"""
    out = []
    for c in (ctx, 1):
        am = capi.GmmScorer(g.ds, gmm_desc=g.ds.cd_only_gmm())
        dec = capi.Decoder(g.ds, am, max_utts=n, max_frames=n * 1024)
        dec.attach_dnn(capi.DnnScorer(g.ds, context_len=c))
        out.append(dec)
    return out


@pytest.mark.parametrize("case", DNN_CASES)
def test_batch_equals_the_host_spliced_batch(case):
    g = Golden(case)
    ctx = CTX[case]
    fl = g.ds.dnn.in_dim // ctx
    utts = _utterances(g, ctx, fl, np.random.default_rng(7))
    dec, dec1 = _decoders(g, ctx, len(utts))
    got = dec.decode(utts)
    want = dec1.decode([splice(x, ctx) for x in utts])
    for u, (r, w) in enumerate(zip(got, want)):
        assert r["n_frames"] == max(0, len(utts[u]) - ctx + 1)
        _same(r, w, f"utterance {u} ({len(utts[u])} input frames)")
    # the same batch again on the same decoder: nothing of the first one is carried over
    for u, (r, w) in enumerate(zip(dec.decode(utts), want)):
        _same(r, w, f"second batch, utterance {u}")


def _stream_plans(utts, ctx, rng):
    """per stream, a list of actions: ("feed", utterance, a, b, last) or ("restart",)"""
    def feeds(u, sizes, end_apart, stop=None):
        N = len(utts[u]) if stop is None else stop
        out, t, i = [], 0, 0
        while t < N:
            n = min(sizes[i] if i < len(sizes) else int(rng.integers(1, 20)), N - t)
            out.append(["feed", u, t, t + n, False]); t += n; i += 1
        if stop is not None:
            return out
        if end_apart or not out:
            out.append(["feed", u, N, N, True])                # end mark with no frames
        else:
            out[-1][4] = True
        return out
    return [
        # golden frames fed 1, ctx - 1, 7, then random; after its end the stream restarts on an utterance shorter
        # than ctx, fed one frame and then the rest, ended by an end mark alone
        feeds(0, [1, ctx - 1, 7], False) + [["restart"]] + feeds(3, [1], True),
        # a first feed shorter than ctx, abandoned half way and restarted, then the whole of another utterance
        feeds(1, [ctx - 1, 1], False, stop=12) + [["restart"]] + feeds(1, [1, ctx - 1], True),
        # random frames in random pieces; then an utterance of exactly ctx frames
        feeds(2, [ctx - 1, 7], False) + [["restart"]] + feeds(4, [ctx], False),
    ]


@pytest.mark.parametrize("case", DNN_CASES)
def test_streams_equal_the_batch_and_the_host_spliced_streams(case):
    g = Golden(case)
    ctx = CTX[case]
    fl = g.ds.dnn.in_dim // ctx
    utts = _utterances(g, ctx, fl, np.random.default_rng(11))
    spliced = [splice(x, ctx) for x in utts]
    dec, dec1 = _decoders(g, ctx, len(utts))
    batch = dec.decode(utts)
    plans = _stream_plans(utts, ctx, np.random.default_rng(12))
    n = len(plans)
    dec.stream_open(n)
    dec1.stream_open(n)
    have = [0] * n                                             # input frames of the stream's current utterance
    step, ended, interims = 0, 0, 0
    while any(plans):
        chunks, rows, last = [], [], []
        for s in range(n):
            act = plans[s].pop(0) if plans[s] else None
            if act is not None and act[0] == "restart":
                dec.stream_restart(s)
                dec1.stream_restart(s)
                have[s] = 0
                act = None
            if act is None:
                chunks.append(None); rows.append(None); last.append(0)
                continue
            _, u, a, b, fin = act
            assert a == have[s]
            chunks.append(utts[u][a:b])
            rows.append(spliced[u][max(0, a - ctx + 1):max(0, b - ctx + 1)])
            last.append(1 if fin else 0)
            have[s] = b
            if fin:
                plans[s] = [("done", u)] + plans[s]            # compared after the feed
        interim = step % 2 == 0
        dec.stream_feed(chunks, last=last, interim=interim)
        dec1.stream_feed(rows, last=last, interim=interim)
        for s in range(n):
            st = dec.stream_status(s)
            assert st == dec1.stream_status(s)
            assert st["frames"] == max(0, have[s] - ctx + 1)
            if interim:
                assert dec.stream_partial(s) == dec1.stream_partial(s), f"stream {s}, feed {step}"
                interims += 1
            if plans[s] and plans[s][0][0] == "done":
                u = plans[s].pop(0)[1]
                _same(dec.stream_result(s), batch[u], f"stream {s}, utterance {u}")
                _same(dec1.stream_result(s), batch[u], f"context-1 stream {s}, utterance {u}")
                ended += 1
        step += 1
    assert ended == 5 and interims > 0
