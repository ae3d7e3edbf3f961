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
