"""Regenerate the committed golden fixtures by running the UNMODIFIED compiled reference
(oracle/_ref/jref, built by oracle/Makefile from /root/reference) on seeded synthetic models.

    python tests/golden/make_golden.py [case ...]

Each fixture directory holds
    model.jb2m  the reference's loaded models, flattened by the export plugin
    out.jrf     reference outputs: [T x S] state scores, word trellis, pass-1 best
    feats.npz   the input feature matrices (u0, u1, ...)
    meta.json   the jconf-style options used

    python tests/golden/make_golden.py sweep

writes the option sweeps of tests/test_oracle_sweep.py as sweep/<case>.npz, in a compact form (tests/util.py).

    python tests/golden/make_golden.py sweep --missing

writes only the sweep cases that have no file yet and leaves the existing ones untouched.
"""
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from julius_b200 import refdump, synth  # noqa: E402
from oracle import ffi, fixtures  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# grammar (DFA) mode cases: the LM is the synthetic finite-state grammar of julius_b200.synth.write_grammar
GRAMMAR_CASES = {"small_dfa"}

CASES = {
    # name: (preset, n_utts, n_frames, noise_utts, extra args)
    "tiny": ("tiny", 2, 150, 0, []),
    "small_b100": ("small", 2, 200, 1, ["-b", "100"]),
    "small_safe": ("small", 1, 150, 0, ["-gprune", "safe", "-tmix", "2", "-b", "60", "-iwcd1", "max"]),
    # multipath tree (non-emitting word-begin/word-end nodes), beam.c:2752-2828
    "small_mp": ("small", 2, 200, 1, ["-multipath", "-b", "120"]),
    # inter-word short pause (tee model => multipath by necessity), BASELINE configs[4] flavour
    "small_iwsp": ("small_sp", 2, 200, 1, ["-iwsp", "-iwcd1", "max", "-b", "150"]),
    # 40 transparent (filler) words: last_cword differs from the last word, beam.c:2300-2330
    "small_tr": ("small_tr", 2, 200, 1, ["-b", "100"]),
    # phonetic tied-mixture AM (<TMIX> codebooks, calc_tied_mix.c), flattened by the exporter; safe pruning
    "small_tm": ("small_tm", 2, 200, 1, ["-gprune", "safe", "-tmix", "4", "-b", "100"]),
    # grammar mode (category tree + category-pair constraint, beam.c:1669-1760, :2404-2455), BASELINE configs[0] flavour
    "small_dfa": ("small", 2, 200, 1, ["-b", "80", "-penalty1", "-1.0"]),
    # user-defined LM functions on top of the N-gram (-userlm, wchmm.h:274-276; registered by the driver, JREF_USERLM=1)
    "small_userlm": ("small", 2, 200, 1, ["-userlm", "-b", "100"]),
}
# cases whose model.jb2m would exceed 1 MB: stored as a compressed delta against the model of another case (tests/util.py)
COMPACT = {"small_userlm": "small_b100", "small_tm": None}
# cases that need something in the driver's environment
CASE_ENV = {"small_userlm": {"JREF_USERLM": "1"}}
# DNN-HMM: (preset, DnnConfig kwargs, n_utts, n_frames, extra args)
DNN_CASES = {
    "small_dnn": ("small", dict(in_dim=120, feature_len=40, context_len=3, hidden=128, layers=3), 2, 150, ["-b", "150"]),
    # configs[4] flavour: DNN-HMM on a multipath tree with -iwsp and a wide beam
    "small_dnn_iwsp": ("small_sp", dict(in_dim=120, feature_len=40, context_len=3, hidden=128, layers=3), 2, 150,
                       ["-iwsp", "-iwcd1", "max", "-b", "600"]),
}


def export_case(name, outdir):
    """runs the recipe of golden case `name` (CASES or DNN_CASES) in outdir -> (model, files, dump, stdout)"""
    if name in DNN_CASES:
        preset, dkw, nu, nf, extra = DNN_CASES[name]
        return fixtures.make_dnn_fixture(preset, outdir, dkw, n_utts=nu, n_frames=nf, extra_args=extra)
    preset, nu, nf, nn, extra = CASES[name]
    return fixtures.make_fixture(preset, outdir, n_utts=nu, n_frames=nf, noise_utts=nn, extra_args=extra,
                                 grammar=name in GRAMMAR_CASES, env_extra=CASE_ENV.get(name))


def sweep_cases():
    """[(preset, extra args, grammar, make_fixture kwargs)] of every sweep case"""
    from test_oracle_sweep import SWEEP, GRAMMAR_SWEEP
    cases = [(p, e, False, dict(n_utts=2, n_frames=150, noise_utts=1)) for p, e in SWEEP]
    return cases + [("small", e, True, dict(n_utts=2, n_frames=180, noise_utts=1)) for e in GRAMMAR_SWEEP]


def make_sweep(missing_only=False):
    for preset, extra, grammar, kw in sweep_cases():
        if missing_only and os.path.exists(os.path.join(util.SWEEP_DIR, util.sweep_name(preset, extra, grammar) + ".npz")):
            continue
        tmp = tempfile.mkdtemp(prefix="jb200_golden_")
        m, files, dump, out = fixtures.make_fixture(preset, tmp, extra_args=extra, grammar=grammar, **kw)
        blob = refdump.load_blob(os.path.join(tmp, "model.jb2m"))
        feats = [synth.read_htk_param(fn)[0] for fn in files]
        dst = util.write_sweep_case(preset, extra, grammar, blob, feats, refdump.load_refdump(dump))
        shutil.rmtree(tmp)
        print(" ".join([preset] + extra), "->", dst)


def main():
    ffi.build()
    if sys.argv[1:2] == ["sweep"]:
        return make_sweep(missing_only=sys.argv[2:] == ["--missing"])
    only = set(sys.argv[1:])
    for name, (preset, nu, nf, nn, extra) in CASES.items():
        if only and name not in only:
            continue
        tmp = tempfile.mkdtemp(prefix="jb200_golden_")
        m, files, dump, out = export_case(name, tmp)
        dst = os.path.join(HERE, name)
        os.makedirs(dst, exist_ok=True)
        meta = {"preset": preset, "extra_args": extra, "n_utts": len(files), "grammar": name in GRAMMAR_CASES, "env": CASE_ENV.get(name, {}),
                "summary": out.strip().splitlines()[-1]}
        if name in COMPACT:
            util.write_golden_model(dst, refdump.load_blob(os.path.join(tmp, "model.jb2m")), COMPACT[name], meta)
        else:
            shutil.copy(os.path.join(tmp, "model.jb2m"), dst)
        shutil.copy(dump, os.path.join(dst, "out.jrf"))
        feats = {f"u{i}": synth.read_htk_param(fn)[0] for i, fn in enumerate(files)}
        np.savez_compressed(os.path.join(dst, "feats.npz"), **feats)
        with open(os.path.join(dst, "meta.json"), "w") as f:
            json.dump(meta, f, indent=1)
        shutil.rmtree(tmp)
        print(name, "->", dst)
    for name, (preset, dkw, nu, nf, extra) in DNN_CASES.items():
        if only and name not in only:
            continue
        tmp = tempfile.mkdtemp(prefix="jb200_golden_")
        m, files, dump, out = export_case(name, tmp)
        dst = os.path.join(HERE, name)
        os.makedirs(dst, exist_ok=True)
        shutil.copy(os.path.join(tmp, "model.jb2m"), dst)
        shutil.copy(dump, os.path.join(dst, "out.jrf"))
        np.savez_compressed(os.path.join(dst, "feats.npz"), **{f"u{i}": synth.read_htk_param(fn)[0] for i, fn in enumerate(files)})
        with open(os.path.join(dst, "meta.json"), "w") as f:
            json.dump({"preset": preset, "dnn": dkw, "extra_args": extra, "n_utts": len(files), "summary": out.strip().splitlines()[-1]}, f, indent=1)
        shutil.rmtree(tmp)
        print(name, "->", dst)


if __name__ == "__main__":
    main()
