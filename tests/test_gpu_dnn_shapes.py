"""GPU: K2 (dnn.cu) at the layer shapes, frame counts and output distributions where a GEMM or a normaliser goes wrong.

Most checks are bit-exact.  The designed nets of tests/util.py have logits that are exact in fp32 whatever the summation
order (tests/test_dnn_design.py checks that on the CPU), so the scores must equal the restatement of dnn_calc_outprob bit
for bit: any layout, padding, pipeline or normaliser error shows, however small.  Multi-layer nets, whose hidden
activations go through bf16x3 and the logistic table, are held to the 1e-4 (floor 1) parity tolerance."""
import math

import numpy as np
import pytest
import torch

from julius_b200 import capi, desc, synth
from util import EXACT_PATTERNS, Golden, atoms_equal, dnn_blob, exact_grid_layer, exact_grid_net, full_dnn_blob, \
    one_hot_softmax_net, random_prior, rel_err

pytestmark = pytest.mark.gpu

NORMALISER_N = [1, 2, 3, 255, 256, 257, 3000, 9001]
IN_DIMS = [1, 7, 8, 9, 16, 63, 64, 65, 120, 129, 429, 528]
OUT_DIMS = [1, 2, 3, 5, 127, 128, 129, 240, 257, 3001]
BN = 128                                    # output columns per GEMM tile (dnn.cu)


def assert_bits_equal(got, want, what=""):
    assert got.shape == want.shape, (got.shape, want.shape)
    diff = got.view(np.uint32) != want.view(np.uint32)
    if diff.any():
        t, i = np.argwhere(diff)[0]
        pytest.fail(f"{what}: {int(diff.sum())} of {diff.size} scores differ, first at frame {t} output {i} "
                    f"({got[t, i]!r} vs {want[t, i]!r}), max abs {np.abs(got - want).max():.3e}, "
                    f"max rel (floor 1) {rel_err(got, want).max():.3e}")


def score_exact(oracle_lib, blob, x, what):
    ds = desc.Descriptors(blob)
    assert_bits_equal(capi.DnnScorer(ds).score(x), oracle_lib.dnn_score(ds, x), what)


# ---- a. the normaliser replays addlog_array ---------------------------------------------------------------------
@pytest.mark.parametrize("n", NORMALISER_N)
def test_normaliser_replays_addlog_array_bit_exact(n, oracle_lib):
    """Frame t is one-hot, so its logits are design t exactly; the log-softmax must be addlog_array's, bit for bit."""
    blob, x, names = one_hot_softmax_net(n, seed=n)
    ds = desc.Descriptors(blob)
    got, want = capi.DnnScorer(ds).score(x), oracle_lib.dnn_score(ds, x)
    bad = [f"{names[t]}: max abs {np.abs(got[t] - want[t]).max():.2e}, rel {rel_err(got[t], want[t]).max():.2e}"
           for t in range(len(names)) if not np.array_equal(got[t].view(np.uint32), want[t].view(np.uint32))]
    assert not bad, f"N = {n}: " + "; ".join(bad)


# ---- b. GEMM layout on exact-grid nets ----------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", list(EXACT_PATTERNS))
@pytest.mark.parametrize("out_dim", OUT_DIMS)
@pytest.mark.parametrize("in_dim", IN_DIMS)
def test_gemm_layout_bit_exact(in_dim, out_dim, pattern, oracle_lib):
    for T in (1, 129):
        blob, x = exact_grid_net(in_dim, out_dim, T, pattern, seed=in_dim * 10007 + out_dim + (T == 1) * 7919)
        score_exact(oracle_lib, blob, x, f"{in_dim} -> {out_dim}, {pattern}, T = {T}")


def _many_tiles_T(out_dim):
    """a frame count giving about 2.5 tiles per SM, so every CTA walks several tiles"""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_nblk = (out_dim + BN - 1) // BN
    T = math.ceil(2.5 * n_sm / n_nblk) * 128 + 1
    assert n_nblk * ((T + 127) // 128) > n_sm
    return T


@pytest.mark.parametrize("in_dim,out_dim,pattern", [(120, 240, "lo_hi"), (429, 3001, "hi_lo"), (64, 129, "hi_hi")])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 255, 257])
def test_gemm_frame_count_sweep_bit_exact(in_dim, out_dim, pattern, T, oracle_lib):
    blob, x = exact_grid_net(in_dim, out_dim, T, pattern, seed=31 * T + in_dim)
    score_exact(oracle_lib, blob, x, f"{in_dim} -> {out_dim}, {pattern}, T = {T}")


@pytest.mark.parametrize("in_dim,out_dim,pattern", [
    (64, 257, "lo_hi"),      # one k-block per tile: fewer than the 3-stage ring, the phases turn over between tiles
    (100, 257, "hi_lo"),     # two k-blocks per tile
    (429, 3001, "lo_hi"),    # the BASELINE output width
])
def test_gemm_more_tiles_than_sms_bit_exact(in_dim, out_dim, pattern, oracle_lib):
    T = _many_tiles_T(out_dim)
    blob, x = exact_grid_net(in_dim, out_dim, T, pattern, seed=in_dim + out_dim)
    score_exact(oracle_lib, blob, x, f"{in_dim} -> {out_dim}, {pattern}, T = {T}")


# ---- c. multi-layer nets within the parity tolerance ----------------------------------------------------------------
ARCHS = {
    "2_layers": [429, 100, 3001],
    "16_layers": [39, 129, 200, 7, 100, 1000, 129, 1, 200, 100, 7, 129, 200, 1000, 100, 129, 257],
    "hidden_1": [120, 1, 240],
    "hidden_7": [120, 7, 7, 240],
    "hidden_100": [429, 100, 100, 257],
    "hidden_129": [429, 129, 129, 3001],
    "hidden_200": [39, 200, 200, 5],
    "hidden_1000": [528, 1000, 1000, 3000],
    "widths_change": [429, 2048, 100, 2048, 3001],
    "saturated": [429, 256, 256, 3001],
}


def random_net(dims, seed, peaked, hidden_scale=1.5):
    """hidden W ~ N(0, hidden_scale/sqrt(in)), output layer 3/sqrt(in).  Peaked: the output layer x 2.5, which puts the
    best output about 15 nats above the median one and leaves some 40 % of the outputs within LOG_ADDMIN of it, as in
    the trained-model designs of util.softmax_designs (the broad nets: about 6 nats, all outputs within)"""
    rng = np.random.default_rng(seed)
    ws, bs = [], []
    for i in range(len(dims) - 1):
        last = i == len(dims) - 2
        scale = (3.0 * (2.5 if peaked else 1.0) if last else hidden_scale) / np.sqrt(dims[i])
        ws.append((rng.standard_normal((dims[i + 1], dims[i])) * scale).astype(np.float32))
        bs.append((rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32))
    return dnn_blob(ws, bs, random_prior(rng, dims[-1])), ws, bs


ARCH_SEEDS = {k: i for i, k in enumerate(ARCHS)}


# One hidden unit drives all 240 logits of "hidden_1" through output weights up to 23.  bf16x3 moves that unit's
# pre-activation by up to 2e-5, which moves its logistic table index by one step in 35 of the 300 frames; one step
# (1.25e-5) times a weight of 23 is 1.3e-4 in log10, and the peaked net shows it: 2.8e-4 absolute, 1.1e-4 relative on
# an H100.  That is a limit of the bf16x3 scheme, not of a layout or the normaliser.
_BF16X3_LIMIT = pytest.mark.xfail(strict=True, reason="bf16x3 + logistic table step through a single hidden unit")


@pytest.mark.parametrize("arch,peaked", [pytest.param(a, p, id=f"{a}-{'peaked' if p else 'broad'}",
                                                      marks=[_BF16X3_LIMIT] if (a, p) == ("hidden_1", True) else [])
                                         for a in ARCHS for p in (False, True)])
def test_multilayer_within_1e4_of_the_oracle(arch, peaked, oracle_lib):
    dims = ARCHS[arch]
    # the saturated net's hidden pre-activations pass +-8, where the logistic is clamped
    blob, ws, bs = random_net(dims, ARCH_SEEDS[arch] + 100 * peaked, peaked, 8.0 if arch == "saturated" else 1.5)
    x = synth.sample_dnn_input(np.random.default_rng(ARCH_SEEDS[arch]), 300, dims[0])
    if arch == "saturated":
        pre = x.astype(np.float64) @ ws[0].T.astype(np.float64) + bs[0]
        assert (np.abs(pre) > 8).mean() > 0.05
    ds = desc.Descriptors(blob)
    got, want = capi.DnnScorer(ds).score(x), oracle_lib.dnn_score(ds, x)
    err = rel_err(got, want, floor=1.0)
    print(f"{arch} {'peaked' if peaked else 'broad'}: max rel err {err.max():.3e}, max abs {np.abs(got - want).max():.3e}")
    assert err.max() <= 1e-4, f"max rel err {err.max():.3e}, max abs {np.abs(got - want).max():.3e}"


# ---- d. a frame's scores do not depend on its batch -----------------------------------------------------------------
def test_scores_do_not_depend_on_the_batch():
    ds = desc.Descriptors(full_dnn_blob(seed=11, in_dim=429, hidden=512, layers=2, n_out=3001))
    x = synth.sample_dnn_input(np.random.default_rng(5), 800, 429)
    X = x[:100]
    a = capi.DnnScorer(ds)
    ref = a.score(X)                                                          # reserves 100 frames
    assert_bits_equal(a.score(X), ref, "repeated call")
    assert_bits_equal(a.score(np.concatenate([x[100:300], X]))[200:], ref, "200 frames prepended (regrowth)")
    assert_bits_equal(a.score(X[:37]), ref[:37], "37 frames, below the reserved 300")
    big = a.score(np.concatenate([x[100:617], X, x[617:800]]))
    assert_bits_equal(big[517:617], ref, "inside 800 frames (regrowth)")
    b = capi.DnnScorer(ds)
    other = b.score(x[300:700])
    assert_bits_equal(a.score(X), ref, "with a second scorer alive")
    assert_bits_equal(b.score(X[::-1])[::-1], ref, "second scorer, frames reversed")
    assert_bits_equal(b.score(x[300:700]), other, "second scorer, repeated")
    assert_bits_equal(other[:100], big[200:300], "same frames in two scorers")


# ---- e. the decoder's scoring path ---------------------------------------------------------------------------------
def test_decoder_on_an_exact_dnn_equals_the_restatement(oracle_lib):
    """small_dnn's HMM with a peaked 120 -> 240 exact-grid net and its features rounded to 1/16: Decoder.decode scores
    through dnn_forward_device into the decoder's score rows; the trellis must equal the restatement's beam on the
    restatement's scores, atom for atom."""
    g = Golden("small_dnn")
    feats = [(np.round(f * 16) / 16).astype(np.float32) for f in g.feats]
    m_x = np.round(np.concatenate(feats) * 16).astype(np.int64)
    _, w, b = exact_grid_layer(np.random.default_rng(2), m_x, 4, 240, 8, 8, nnz=32)
    blob = {k: v for k, v in g.blob.items() if not k.startswith("dnn.")}
    blob.update(dnn_blob([w], [b], g.blob["dnn.state_prior"]))
    ds = desc.Descriptors(blob)
    logits = m_x * 2.0 ** -4 @ w.T.astype(np.float64) + b
    top2 = np.sort(logits, axis=1)[:, -2:]
    assert np.median(top2[:, 1] - np.median(logits, axis=1)) > 14      # peaked: most outputs are dropped by addlog_array
    dnn = capi.DnnScorer(ds)
    am = capi.GmmScorer(ds, gmm_desc=ds.cd_only_gmm())
    dec = capi.Decoder(ds, am, max_utts=4, max_frames=2048)
    dec.attach_dnn(dnn)
    res = dec.decode(feats)
    for u, (r, f) in enumerate(zip(res, feats)):
        sc = oracle_lib.dnn_score(ds, f)
        assert_bits_equal(dnn.score(f), sc, f"utterance {u} scores")
        o = oracle_lib.beam_decode(ds, sc)
        ok, why = atoms_equal(r["atoms"], o["atoms"])
        assert ok, f"utterance {u}: {why}"
        assert r["words"] == o["words"] and r["status"] == o["status"] and r["overflow"] == 0
        assert np.float32(r["score"]) == np.float32(o["score"])
