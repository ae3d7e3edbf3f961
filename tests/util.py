import hashlib
import json
import os
import re
from types import SimpleNamespace

import numpy as np

from julius_b200 import desc, refdump

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# small_userlm: user-defined LM functions (-userlm) on top of the N-gram, tabulated by the exporter
CASES = ["tiny", "small_b100", "small_safe", "small_mp", "small_iwsp", "small_userlm"]
DNN_CASES = ["small_dnn", "small_dnn_iwsp"]
# pinned on the CPU only so far (the GPU suite does not run them yet)
ORACLE_ONLY_CASES = ["small_tr", "small_tm", "small_dfa"]


class Golden:
    def __init__(self, name):
        d = os.path.join(GOLDEN, name)
        self.dir = d
        self.meta = json.load(open(os.path.join(d, "meta.json")))
        self.blob = load_golden_model(d, self.meta)
        self.ds = desc.Descriptors(self.blob)
        self.utts = refdump.load_refdump(os.path.join(d, "out.jrf"))
        z = np.load(os.path.join(d, "feats.npz"))
        self.feats = [z[f"u{i}"] for i in range(len(self.utts))]


def atoms_equal(a, b):
    """bit-exact comparison of two structured atom arrays (wid, begin, end, backscore, lscore, last)."""
    if len(a) != len(b):
        return False, f"atom count {len(a)} != {len(b)}"
    for k in ("wid", "begin", "end", "last"):
        if not np.array_equal(a[k], b[k]):
            i = int(np.nonzero(a[k] != b[k])[0][0])
            return False, f"field {k} differs first at atom {i}: {a[i]} vs {b[i]}"
    for k in ("backscore", "lscore"):
        if not np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)):
            i = int(np.nonzero(a[k].view(np.uint32) != b[k].view(np.uint32))[0][0])
            return False, f"field {k} differs (bits) first at atom {i}: {a[i]} vs {b[i]}"
    return True, ""


def rel_err(a, b, floor=1.0):
    """|a-b| / max(|a|,|b|,floor): the relative criterion with an absolute floor (SURVEY 7, hard parts)."""
    return np.abs(a - b) / np.maximum(np.maximum(np.abs(a), np.abs(b)), floor)


def full_dnn_blob(seed=3, in_dim=528, hidden=2048, layers=7, n_out=3000):
    """A random-init DNN of the BASELINE configs[3] shape (528 = 48 x 11 inputs, 7 x 2048 logistic, n_out states) as a
    flattened-model blob dict, with the initialisation of julius_b200.synth.write_dnn (W ~ N(0, 1.5/sqrt(in)), output
    layer 3/sqrt(in), b ~ N(0, 0.1), Dirichlet priors stored as log10, calc_dnn.c:699-703)."""
    rng = np.random.default_rng(seed)
    dims = [in_dim] + [hidden] * layers + [n_out]
    b = {"dnn.n_layers": np.array([layers + 1], np.int32), "dnn.in_dim": np.array([in_dim], np.int32),
         "dnn.out_dim": np.array([n_out], np.int32), "gmm.n_states": np.array([n_out], np.int32)}
    for i in range(layers + 1):
        scale = (3.0 if i == layers else 1.5) / np.sqrt(dims[i])
        b[f"dnn.l{i}.in"] = np.array([dims[i]], np.int32)
        b[f"dnn.l{i}.out"] = np.array([dims[i + 1]], np.int32)
        b[f"dnn.l{i}.w"] = (rng.standard_normal((dims[i + 1], dims[i])) * scale).astype(np.float32).ravel()
        b[f"dnn.l{i}.b"] = (rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)
    prior = rng.dirichlet(np.full(n_out, 5.0))
    b["dnn.state_prior"] = np.log10(prior).astype(np.float32)
    return b


def dnn_blob(ws, bs, prior):
    """A DNN blob dict (the layout of full_dnn_blob) from per-layer weights [out, in] and biases [out]."""
    b = {"dnn.n_layers": np.array([len(ws)], np.int32), "dnn.in_dim": np.array([ws[0].shape[1]], np.int32),
         "dnn.out_dim": np.array([ws[-1].shape[0]], np.int32), "gmm.n_states": np.array([ws[-1].shape[0]], np.int32)}
    for i, (w, bias) in enumerate(zip(ws, bs)):
        b[f"dnn.l{i}.in"] = np.array([w.shape[1]], np.int32)
        b[f"dnn.l{i}.out"] = np.array([w.shape[0]], np.int32)
        b[f"dnn.l{i}.w"] = np.ascontiguousarray(w, np.float32).ravel()
        b[f"dnn.l{i}.b"] = np.ascontiguousarray(bias, np.float32)
    b["dnn.state_prior"] = np.ascontiguousarray(prior, np.float32)
    return b


def random_prior(rng, n):
    return np.log10(rng.dirichlet(np.full(n, 5.0))).astype(np.float32)


# ---- designed DNNs whose output the restatement gives bit for bit (tests/test_gpu_dnn_shapes.py) -------------------
# K2 splits every operand into bf16 hi + lo and sums hi.hi + hi.lo + lo.hi in fp32.  A value with at most 16 significant
# bits splits exactly, and when one operand of each product is hi-only (8 bits) the dropped lo.lo term is zero.  If every
# product and every partial sum is a multiple of one grid and stays below 2^20 grid units, each sum is exact in fp32 in
# any order, so the logits equal the restatement's; what remains is the normaliser, which replays addlog_array.

def round_sig16(a):
    """float32 rounded to 16 significant bits (nearest, ties to even)"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7F + ((u >> 8) & 1)) & 0xFFFFFF00
    return u.astype(np.uint32).view(np.float32)


def softmax_designs(n, rng):
    """Designed logit vectors of length n: flat, broad, peaked like a trained acoustic model with the peak early or late
    in addlog_array's walk (which runs from n-1 down to 0), ties, a -1e10 entry, a 1e4 spread, clusters around the
    LOG_ADDMIN cut.  Each value has at most 16 significant bits."""
    def nrm(mu, s):
        return mu + s * rng.standard_normal(n)

    def put(a, idx, v):
        a = a.copy()
        a[idx] = v
        return a

    last = n - 1
    two = rng.choice(n, size=min(2, n), replace=False)
    near = -13.8155 + rng.integers(-8, 9, n) * 2.0 ** -12          # both sides of the cut, 2^-12 apart
    cluster = np.where(rng.random(n) < 0.5, -13.7, -13.9)
    d = {
        "flat": np.zeros(n),
        "n3_top15_first": put(nrm(0, 3), 0, 15.0),
        "n3_top15_last": put(nrm(0, 3), last, 15.0),
        "n2_top12_first": put(nrm(0, 2), 0, 12.0),
        "top10_first_rest_n-4": put(nrm(-4, 1), 0, 10.0),
        "top10_last_rest_n-4": put(nrm(-4, 1), last, 10.0),
        "top0_first_rest_-13.9": put(np.full(n, -13.9), 0, 0.0),
        "top0_last_rest_-13.9": put(np.full(n, -13.9), last, 0.0),
        "n1": nrm(0, 1), "n3": nrm(0, 3), "n5": nrm(0, 5),
        "two_equal_maxima": put(nrm(0, 3), two, 15.0),
        "minus_1e10": put(nrm(0, 3), rng.integers(n), -1e10),
        "spread_1e4": rng.uniform(-5e3, 5e3, n),
        "clusters_-13.7_-13.9_first": put(cluster, 0, 0.0),
        "clusters_-13.7_-13.9_last": put(cluster, last, 0.0),
        "near_cut_first": put(near, 0, 0.0),
        "near_cut_last": put(near, last, 0.0),
    }
    return {k: round_sig16(v.astype(np.float32)) for k, v in d.items()}


def one_hot_softmax_net(n, seed):
    """Single layer, one input per design: frame t is one-hot at t, so its logits are design t exactly (bias 0)."""
    rng = np.random.default_rng(seed)
    designs = softmax_designs(n, rng)
    w = np.stack(list(designs.values()), axis=1)                  # [n, K]
    x = np.eye(w.shape[1], dtype=np.float32)
    return dnn_blob([w], [np.zeros(n, np.float32)], random_prior(rng, n)), x, list(designs)


# operand patterns: (input bits, input exponent, weight bits, weight exponent); values are m * 2^-e with |m| < 2^bits
EXACT_PATTERNS = {"hi_hi": (7, 4, 7, 6),      # both operands hi-only: hi.hi alone
                  "lo_hi": (11, 10, 4, 2),    # inputs with lo parts: pins lo.hi
                  "hi_lo": (4, 2, 11, 10)}    # weights with lo parts: pins hi.lo
EXACT_LIMIT = 2 ** 20                         # grid units; fp32 has 24 bits, 4 are kept as margin


def exact_grid_layer(rng, m_x, ax, out_dim, wb, aw, nnz=24):
    """Weights and bias for integer inputs m_x [T, in] on the grid 2^-ax: nnz non-zero weights per output, m_w * 2^-aw
    with 0 < |m_w| < 2^wb, bias on the product grid 2^-(ax+aw).  Returns (x, w, b); asserts the exactness bound."""
    T, in_dim = m_x.shape
    k = min(in_dim, nnz)
    m_w = np.zeros((out_dim, in_dim), np.int64)
    mag = rng.integers(1, 2 ** wb, (out_dim, k)) * rng.choice([-1, 1], (out_dim, k))
    cols = np.argsort(rng.random((out_dim, in_dim)), axis=1)[:, :k]
    np.put_along_axis(m_w, cols, mag, axis=1)
    m_b = rng.integers(-2 ** 16, 2 ** 16 + 1, out_dim)
    bound = (np.abs(m_x).astype(np.int64) @ np.abs(m_w).T).max(initial=0) + np.abs(m_b).max()
    assert bound < EXACT_LIMIT, f"design error: sum of |x w| + |b| reaches {bound} grid units (limit {EXACT_LIMIT})"
    x = (m_x * 2.0 ** -ax).astype(np.float32)
    w = (m_w * 2.0 ** -aw).astype(np.float32)
    b = (m_b * 2.0 ** -(ax + aw)).astype(np.float32)
    assert np.array_equal(x, m_x * 2.0 ** -ax) and np.array_equal(w, m_w * 2.0 ** -aw)
    return x, w, b


def exact_grid_net(in_dim, out_dim, T, pattern, seed):
    """A single-layer exact-grid net and inputs (see EXACT_PATTERNS) -> (blob, x)."""
    rng = np.random.default_rng(seed)
    xb, ax, wb, aw = EXACT_PATTERNS[pattern]
    m_x = rng.integers(-(2 ** xb - 1), 2 ** xb, (T, in_dim))
    x, w, b = exact_grid_layer(rng, m_x, ax, out_dim, wb, aw)
    return dnn_blob([w], [b], random_prior(rng, out_dim)), x


def addlog_table_np():
    """addlog.c:39-57 in numpy"""
    f = -(np.float32(15) * np.arange(500000, dtype=np.float32) / np.float32(500000))
    return np.log(1 + np.exp(f.astype(np.float64))).astype(np.float32)


def addlog_array_np(a, tbl):
    """addlog_array (addlog.c:102-123) on every row of a [T, N] float32, in float32 with the same double promotions"""
    a = np.asarray(a, np.float32)
    y = np.full(a.shape[0], -1000000.0, np.float32)
    for n in range(a.shape[1] - 1, -1, -1):
        x = a[:, n]
        hi, lo = np.maximum(x, y), np.minimum(x, y)
        tmp = lo - hi
        keep = tmp.astype(np.float64) >= -13.815510558
        idx = np.where(keep, (-tmp).astype(np.float64) * 33333.3333 + 0.5, 0).astype(np.uint32)
        y = np.where(keep, hi + tbl[idx], hi)
    return y


def single_layer_scores_np(blob, x, tbl):
    """Exact float64 logits of a single-layer net (asserted representable in float32), then addlog_array and the prior
    line of calc_dnn.c:862-865 in numpy"""
    n, k = int(blob["dnn.out_dim"][0]), int(blob["dnn.in_dim"][0])
    w = blob["dnn.l0.w"].reshape(n, k).astype(np.float64)
    logits = x.astype(np.float64) @ w.T + blob["dnn.l0.b"].astype(np.float64)
    l32 = logits.astype(np.float32)
    assert np.array_equal(l32.astype(np.float64), logits), "design error: the logits are not exact in float32"
    lp = addlog_array_np(l32, tbl)
    out = 0.434294482 * (l32 - lp[:, None]).astype(np.float64) - blob["dnn.state_prior"].astype(np.float64)
    return out.astype(np.float32)


# ---- designed GMMs (tests/test_gmm_design.py, tests/test_gpu_gmm_shapes.py) -----------------------------------------
# K1 is instantiated for these feature dimensions; even ones keep gconst / ln w in an extra quad of the record.
GMM_DIMS = [25, 26, 38, 39]
LOG_ZERO = np.float32(-1000000.0)
LOG_ADDMIN = -13.815510558                        # a double: the drop test compares a float difference with it
ADDMIN_KEPT = np.float32(np.nextafter(np.float32(LOG_ADDMIN), np.float32(0)))
if float(ADDMIN_KEPT) < LOG_ADDMIN:               # the float just above LOG_ADDMIN, whichever way the cast rounded
    ADDMIN_KEPT = np.nextafter(ADDMIN_KEPT, np.float32(0))
ADDMIN_DROPPED = np.nextafter(ADDMIN_KEPT, np.float32(-np.inf))   # the float just below it
TILE_STATES, TILE_GAUSS = 4, 64                   # K1's tile caps (gmm.cu)

# mixture counts in tiling order: empty states at the start, a tile ending at exactly 64 Gaussians, a 64-mixture state,
# 65 Gaussians (40 + 25: a split), empty states right after a full 4-state tile (a run of 1 and a run of 4), a single
# empty state in the middle, more than 4 one-mixture states, ragged counts, empty states at the end after a full tile
TILING_PATTERN = ([0, 0, 3, 61, 64, 8, 8, 8, 8, 0, 40, 25, 39, 8, 8, 8, 8, 0, 0, 0, 0, 8, 5, 0, 7] + [1] * 9
                  + [20, 20, 24, 2, 0, 1, 16])
TILING_TAIL = [8, 8, 8, 8, 0]
# the two examples of states no tile used to cover
EMPTY_STATE_PATTERNS = {"4full_then_1empty": [8, 8, 8, 8, 0], "4full_4empty_8": [8, 8, 8, 8, 0, 0, 0, 0, 8]}


def gmm_tiles(counts):
    """K1's tiling (gmm_build) in Python: [(first state, states, Gaussians)]"""
    tiles, s, S = [], 0, len(counts)
    while s < S:
        s0, ng, filled = s, 0, 0
        while s < S and (counts[s] == 0 or (filled < TILE_STATES and ng + counts[s] <= TILE_GAUSS)):
            ng += counts[s]
            filled += counts[s] > 0
            s += 1
        if ng > 0:
            tiles.append((s0, s - s0, ng))
    return tiles


def tiles_per_cta(T, n_tiles, sms):
    """the tiles one CTA of K1 walks for T frames (launch_gmm: about 8 CTAs per SM)"""
    fblocks = -(-T // 256)
    chunks = min(max(1, -(-sms * 8 // fblocks)), n_tiles)
    return -(-n_tiles // chunks)


def gmm_blob(counts, dim, mean, ivar, gconst, lnw, valid, cdsets=(), iwcd=(2, 3), gprune=(0, 2)):
    """A GMM blob dict (the entries desc.Descriptors reads) from per-state mixture counts, per-Gaussian parameters and
    pseudo-phone (cd) sets given as lists of member states."""
    counts = np.asarray(counts, np.int64)
    off = np.zeros(len(counts) + 1, np.int32)
    np.cumsum(counts, out=off[1:])
    G = int(off[-1])
    cd_off = np.zeros(len(cdsets) + 1, np.int32)
    np.cumsum([len(c) for c in cdsets], out=cd_off[1:])
    cd_states = np.array([s for c in cdsets for s in c], np.int32)
    i32 = lambda v: np.array([v], np.int32)
    return {"gmm.n_states": i32(len(counts)), "gmm.dim": i32(dim), "gmm.n_gauss": i32(G),
            "gmm.max_mix": i32(max(1, int(counts.max(initial=0)))), "gmm.gprune_method": i32(gprune[0]),
            "gmm.gprune_num": i32(gprune[1]), "gmm.state_off": off,
            "gmm.mean": np.ascontiguousarray(mean, np.float32).reshape(G * dim),
            "gmm.ivar": np.ascontiguousarray(ivar, np.float32).reshape(G * dim),
            "gmm.gconst": np.ascontiguousarray(gconst, np.float32), "gmm.lnweight": np.ascontiguousarray(lnw, np.float32),
            "gmm.valid": np.ascontiguousarray(valid, np.uint8),
            "am.iwcd_method": i32(iwcd[0]), "am.iwcd_nbest": i32(iwcd[1]), "am.n_cdsets": i32(len(cdsets)),
            "am.n_cdset_states": i32(len(cd_states)), "am.cd_off": cd_off, "am.cd_states": cd_states}


def random_gmm_counts(seed, n_ragged=300):
    rng = np.random.default_rng(seed)
    return TILING_PATTERN + rng.integers(1, 17, n_ragged).tolist() + TILING_TAIL


def cdset_designs(counts, rng):
    """cd sets over a model's states: 1 member, 2..17 members (below, at and above every best N), 24 and 40 members,
    sets with a repeated member (tied scores), sets holding empty (LOG_ZERO) states and a set of empty states only"""
    counts = np.asarray(counts)
    full, empty = np.nonzero(counts > 0)[0], np.nonzero(counts == 0)[0]
    pick = lambda n: rng.choice(full, n, replace=n > len(full)).tolist()
    sets = [pick(n) for n in [1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 24, 40]]
    for n in (3, 5, 9, 17):
        m = pick(n - 1)
        sets.append(m + [m[n // 2]])                                       # a tie
        sets.append(m[:n // 2] + [int(empty[0])] + m[n // 2:])             # a member at LOG_ZERO
    sets.append([int(e) for e in empty[:3]])                               # all LOG_ZERO: 0/0 in AVG and best N
    return sets


def random_gmm(counts, dim, seed, null_frac=0.1):
    """Means N(0,1), inverse variances in [0.2, 5] with their gconst, Dirichlet weights, about null_frac NULL densities,
    one 8-mixture state with all densities NULL and states with a NULL first, last, and first and last mixture."""
    rng = np.random.default_rng(seed)
    counts = list(counts)
    G = int(sum(counts))
    mean = rng.standard_normal((G, dim)).astype(np.float32)
    ivar = rng.uniform(0.2, 5.0, (G, dim)).astype(np.float32)
    gconst = (dim * np.log(2 * np.pi) - np.log(ivar.astype(np.float64)).sum(1)).astype(np.float32)
    lnw = np.concatenate([np.log(rng.dirichlet(np.full(c, 2.0))) for c in counts if c > 0]).astype(np.float32)
    valid = (rng.random(G) >= null_frac).astype(np.uint8)
    off = np.concatenate([[0], np.cumsum(counts)])
    eight = [s for s, c in enumerate(counts) if c == 8]
    valid[off[eight[0]]:off[eight[0] + 1]] = 0
    big = [s for s, c in enumerate(counts) if c >= 12]
    valid[off[big[0]]] = 0
    valid[off[big[1] + 1] - 1] = 0
    valid[off[big[2]]] = valid[off[big[2] + 1] - 1] = 0
    return gmm_blob(counts, dim, mean, ivar, gconst, lnw, valid, cdset_designs(counts, rng))


def random_frames(dim, T, seed, n_far=32):
    """features N(0, 1.2), then n_far far frames (scale 30 .. 3000) whose Gaussian sums cross LOG_ZERO"""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.2, (T, dim))
    x[T - n_far:] *= np.geomspace(25.0, 2500.0, n_far)[:, None]
    return x.astype(np.float32)


def index_rounding_diffs(n_each=4):
    """differences d (floats in (LOG_ADDMIN, 0)) whose table index (double)(-d) * 33333.3333 + 0.5 lies within a few
    float ulps below / above an integer, picked where the same index taken in float arithmetic lands on the other side"""
    d = -np.float32(np.linspace(0.5, 13.5, 2_000_003)).astype(np.float32)
    r = (-d).astype(np.float64) * 33333.3333 + 0.5
    i_d = r.astype(np.int64)
    i_mul = (np.float32(-d) * np.float32(33333.3333) + np.float32(0.5)).astype(np.int64)
    i_fma = ((-d).astype(np.float64) * np.float64(np.float32(33333.3333)) + 0.5).astype(np.float32).astype(np.int64)
    frac = r - np.rint(r)
    near = np.abs(frac) < 4 * np.spacing(r.astype(np.float32)).astype(np.float64)
    pick = []
    for side in (frac < 0, frac > 0):
        idx = np.nonzero(near & side & (i_d != i_mul) & (i_d != i_fma))[0]
        pick += idx[np.linspace(0, len(idx) - 1, n_each).astype(int)].tolist()
    return d[pick]


def addlog_designs():
    """{name: weighted terms} for states with ivar = 0, where every term is exactly gconst * -0.5 + ln w (ln w = 0)"""
    rng = np.random.default_rng(5)
    f = lambda *v: np.array(v, np.float32)
    d = {"addmin_kept": f(-1.5, np.float32(-1.5) + ADDMIN_KEPT), "addmin_dropped": f(-1.5, np.float32(-1.5) + ADDMIN_DROPPED),
         "addmin_kept_rev": f(np.float32(-1.5) + ADDMIN_KEPT, -1.5),
         "equal64": np.full(64, -3.0, np.float32),
         "peak_first": np.concatenate([[4.0], rng.normal(-6, 2, 11)]).astype(np.float32),
         "peak_last": np.concatenate([rng.normal(-6, 2, 11), [4.0]]).astype(np.float32),
         "below_log_zero": f(-2e6, -1.5e6, -3e6), "at_log_zero": f(-1e6), "near_log_zero": f(-1000003.0, -1000001.0),
         "exact_zero": f(0.0), "exact_zero_2": f(0.0, -20.0)}
    for i, x in enumerate(index_rounding_diffs()):
        d[f"index_{i}"] = f(0.0, x)
    return d


EXACT_ZERO_DESIGNS = ("exact_zero", "exact_zero_2")


def prune_designs(n):
    """{name: (scores, ln w, kept list)} for -tmix n: the kept list is the top-n list the pruned walk must end with, in
    list order (best first).  Scores are 0.25-grid values; the weights make every kept id visible in the sum."""
    w = lambda k: np.log(np.arange(1, k + 1, dtype=np.float64) / (k * (k + 1) / 2))
    highs = [6.0 + i for i in range(max(n - 2, 0))][::-1]
    d = {}
    # a later equal score goes in front of an earlier one; the next insertion then drops the earlier one
    if n >= 2:
        sc = highs + [4.0, 3.0, 4.0, 4.5]
        k = len(highs)
        d["tie_order"] = (sc, w(len(sc)), list(range(k)) + [k + 3, k + 2])
    # a candidate equal to the n-th best is dropped
    sc = [5.0 + i for i in range(n)][::-1] + [5.0]
    d["equal_nth"] = (sc, w(len(sc))[::-1], list(range(n)))
    # equal scores: the first n mixtures stay, whatever their weights
    d["equal_scores"] = ([-2.0] * (n + 3), w(n + 3)[::-1], list(range(n)))
    # fewer mixtures than -tmix
    d["fewer_than_tmix"] = ([1.0, 3.0], w(2), [1, 0][:n])
    return {k: (np.array(s, np.float32), np.array(l, np.float32), kept) for k, (s, l, kept) in d.items()}


def design_gmm(dim, seed, tmix=None):
    """A model with one state per addlog design (ln w = 0), and with tmix the prune designs for -tmix tmix, separated by
    empty states; ivar = 0 so that each Gaussian's log-likelihood is gconst * -0.5 on every frame.
    -> (blob, [state name or None for an empty state])"""
    rng = np.random.default_rng(seed)
    states = [(k, v, np.zeros(len(v), np.float32)) for k, v in addlog_designs().items()]
    if tmix is not None:
        states += [(k, s, l) for k, (s, l, _) in prune_designs(tmix).items()]
    names, counts, scores, lnws = [], [], [], []
    for i, (k, s, l) in enumerate(states):
        if i % 3 == 0:
            names.append(None); counts.append(0)
        names.append(k); counts.append(len(s)); scores.append(s); lnws.append(l)
    names.append(None); counts.append(0)
    sc = np.concatenate(scores)
    G = len(sc)
    gconst = (sc * np.float32(-2.0)).astype(np.float32)
    assert np.array_equal(gconst * np.float32(-0.5), sc)
    mean = rng.standard_normal((G, dim)).astype(np.float32)
    blob = gmm_blob(counts, dim, mean, np.zeros((G, dim), np.float32), gconst, np.concatenate(lnws),
                    np.ones(G, np.uint8), cdset_designs(counts, rng))
    return blob, names


def finish_np(lp):
    """calc_mix.c:72-80 for one stream of weight 1 on float32 log-sums"""
    lp = np.asarray(lp, np.float32)
    out = (lp.astype(np.float64) * 0.434294482).astype(np.float32)
    return np.where((lp <= LOG_ZERO) | (lp == 0), LOG_ZERO, out).astype(np.float32)


# A golden model is stored whole (model.jb2m), or, where that file would exceed 1 MB, as model_delta.npz: the entries that
# differ from the model of the golden case meta["base"] (all of them when there is no base), compressed; meta["drop"] lists
# the base's entries the model does not have.
def load_golden_model(d, meta):
    p = os.path.join(d, "model.jb2m")
    if os.path.exists(p):
        return refdump.load_blob(p)
    return _apply_delta(meta.get("base"), dict(np.load(os.path.join(d, "model_delta.npz"))), meta.get("drop", []))


def _golden_blob(name):
    d = os.path.join(GOLDEN, name)
    return load_golden_model(d, json.load(open(os.path.join(d, "meta.json"))))


def _apply_delta(base_name, delta, drop):
    base = _golden_blob(base_name) if base_name else {}
    blob = {k: delta.get(k, v) for k, v in base.items() if k not in drop}
    blob.update(delta)
    return blob


def _model_delta(blob, base_name):
    base = _golden_blob(base_name) if base_name else {}
    return {k: v for k, v in blob.items() if k not in base or not _same(base[k], v)}, [k for k in base if k not in blob]


def write_golden_model(d, blob, base_name, meta):
    """writes model_delta.npz and records base / drop in meta (the caller writes meta.json)"""
    delta, drop = _model_delta(blob, base_name)
    np.savez_compressed(os.path.join(d, "model_delta.npz"), **delta)
    meta.update(base=base_name, drop=drop)


# ---- option sweeps pinned against the compiled reference (tests/golden/sweep/<case>.npz, made by make_golden.py sweep).
# A case stores only what its exported model has that differs from the golden case of the same synthetic preset
# (the GMM parameters are the same), the input features, the reference's word trellis / pass-1 best, and a SHA-256
# of the reference's [T x S] state-score matrix, which the state scores of the code under test must reproduce bit for bit.
SWEEP_DIR = os.path.join(GOLDEN, "sweep")
SWEEP_BASE = {("small", False): "small_b100", ("small_sp", False): "small_iwsp", ("small_tr", False): "small_tr",
              ("small_tm", False): "small_tm", ("small", True): "small_dfa"}


def sweep_name(preset, extra, grammar=False):
    return re.sub(r"[^A-Za-z0-9.]+", "_", " ".join((["dfa"] if grammar else []) + [preset] + list(extra))).strip("_")


def scores_sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def write_sweep_case(preset, extra, grammar, blob, feats, utts):
    """one compressed .npz per case: model/<entry> (the delta), u<i> (features), atoms<i> / words<i> / status<i> /
    score<i> (the reference's results) and meta (JSON)"""
    base_name = SWEEP_BASE[(preset, grammar)]
    delta, drop = _model_delta(blob, base_name)
    meta = {"preset": preset, "extra_args": list(extra), "grammar": grammar, "base": base_name, "drop": drop,
            "outprob_sha256": [scores_sha(u.outprob) for u in utts]}
    z = {f"model/{k}": v for k, v in delta.items()}
    for i, (x, u) in enumerate(zip(feats, utts)):
        z.update({f"u{i}": x, f"atoms{i}": u.atoms, f"words{i}": np.array(u.words, np.int32),
                  f"status{i}": np.array([u.status], np.int32), f"score{i}": np.array([u.score], np.float32)})
    os.makedirs(SWEEP_DIR, exist_ok=True)
    p = os.path.join(SWEEP_DIR, sweep_name(preset, extra, grammar) + ".npz")
    np.savez_compressed(p, meta=np.array(json.dumps(meta)), **z)
    return p


def load_sweep_case(preset, extra, grammar=False):
    """-> (Descriptors, [features], [reference utterance: atoms, words, status, score, outprob_sha256])"""
    z = np.load(os.path.join(SWEEP_DIR, sweep_name(preset, extra, grammar) + ".npz"))
    meta = json.loads(str(z["meta"]))
    blob = _apply_delta(meta["base"], {k[6:]: z[k] for k in z.files if k.startswith("model/")}, meta["drop"])
    n = len(meta["outprob_sha256"])
    utts = [SimpleNamespace(atoms=z[f"atoms{i}"], words=z[f"words{i}"].tolist(), status=int(z[f"status{i}"][0]),
                            score=z[f"score{i}"][0], outprob_sha256=meta["outprob_sha256"][i]) for i in range(n)]
    return desc.Descriptors(blob), [z[f"u{i}"] for i in range(n)], utts
