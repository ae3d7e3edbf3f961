"""CPU: host-side logic -- blob container round trip, descriptor structs, C-ABI symbols."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from julius_b200 import capi, desc, refdump, synth
from util import GOLDEN, ROOT, Golden


def test_blob_roundtrip(tmp_path):
    g = Golden("tiny")
    p = tmp_path / "x.jb2m"
    refdump.save_blob(str(p), g.blob)
    b2 = refdump.load_blob(str(p))
    assert list(b2) == list(g.blob)
    for k in g.blob:
        assert b2[k].dtype == g.blob[k].dtype and np.array_equal(b2[k], g.blob[k])


def test_descriptor_fields():
    g = Golden("small_b100")
    t = g.ds.tree
    assert t.n_nodes == len(g.blob["tree.self_a"])
    assert t.n_iso + t.n_shared == t.n_start
    assert t.beam_width == 100
    assert g.ds.gmm.n_gauss == g.blob["gmm.state_off"][-1]
    assert C.sizeof(desc.TreeDesc) % 8 == 0


def test_capi_library_exports_every_declared_symbol():
    assert os.path.exists(capi.LIBPATH), "libjb200.so not built (python -m julius_b200.build)"
    L = C.CDLL(capi.LIBPATH)
    hdr = open(os.path.join(ROOT, "include", "julius_b200.h")).read()
    names = set(re.findall(r"\b(jb200_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 15
    missing = [n for n in sorted(names) if not hasattr(L, n)]
    assert not missing, f"declared in julius_b200.h but not exported: {missing}"


def test_synth_is_seeded(tmp_path):
    a = synth.SynthModel(synth.SynthConfig.preset("tiny"))
    b = synth.SynthModel(synth.SynthConfig.preset("tiny"))
    assert np.array_equal(a.mean, b.mean) and a.words == b.words and a.bigrams == b.bigrams
    x, _ = a.sample_utterance(np.random.default_rng(3), 120)
    assert x.shape == (120, 39) and x.dtype == np.float32
    p = tmp_path / "f.mfc"
    synth.write_htk_param(str(p), x)
    y, kind = synth.read_htk_param(str(p))
    assert np.array_equal(x, y) and kind == synth.PARMKIND_MFCC_E_D_A


def test_descriptor_layouts_match_the_c_header(tmp_path):
    """The ctypes mirrors in julius_b200/desc.py must lay the descriptors out exactly as include/jb200_model.h does
    (the product library, the plugin and the oracle all read them through that header)."""
    import ctypes as C
    import shutil
    import subprocess
    from julius_b200 import desc
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    fields = {"jb200_tree_desc": (desc.TreeDesc, ["n_nodes", "lm_unk_num_log", "self_a", "bi_prob", "lm_type", "penalty1", "init_word", "cp_allowed"]),
              "jb200_gmm_desc": (desc.GmmDesc, ["n_states", "state_off", "valid", "cd_states"]),
              "jb200_dnn_desc": (desc.DnnDesc, ["n_layers", "layer_out", "w", "state_prior"])}
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "jb200_model.h"', 'int main(void) {']
    for st, (_, names) in fields.items():
        src.append(f'  printf("{st} %zu", sizeof({st}));')
        for n in names:
            src.append(f'  printf(" %zu", offsetof({st}, {n}));')
        src.append('  printf("\\n");')
    src.append('  return 0; }')
    cfile = tmp_path / "layout.c"
    cfile.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(cfile)], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    for line in out:
        if not line.strip():
            continue
        parts = line.split()
        cls, names = fields[parts[0]]
        want = [C.sizeof(cls)] + [getattr(cls, n).offset for n in names]
        assert [int(x) for x in parts[1:]] == want, parts[0]


def test_c_descriptor_readers_match_python(tmp_path):
    """jb200_gmm_from_blob on a GMM model and jb200_cd_gmm_from_blob (the beam shim's layout-only scorer of a DNN
    model) read what desc.py reads; a cd-set table shorter than declared is refused; a long entry name is cut to 47
    characters."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    src = r'''#include "jb200_model.h"
static void show(const char *what, int rc, const jb200_gmm_desc *g) {
  printf("%s %d %d %d %d %d %d %d %d %d %d\n", what, rc, g->n_states, g->dim, g->n_gauss, g->iwcd_method, g->iwcd_nbest,
         g->n_cdsets, g->n_cdset_states, g->cd_off ? g->cd_off[g->n_cdsets] : -1, g->mean != NULL);
}
int main(int argc, char **argv) {
  jb200_blob b; jb200_gmm_desc g; jb200_blob_entry *x;
  if (argc != 3 || jb200_blob_load(&b, argv[1]) != 0) return 1;
  show("gmm", jb200_gmm_from_blob(&b, &g), &g);
  jb200_blob_free(&b);
  if (jb200_blob_load(&b, argv[2]) != 0) return 1;
  show("cd", jb200_cd_gmm_from_blob(&b, &g), &g);
  x = (jb200_blob_entry *)jb200_blob_find(&b, "am.cd_off");
  x->count -= 1;
  show("short", jb200_cd_gmm_from_blob(&b, &g), &g);
  jb200_blob_add_i(&b, "LONG", 7);
  printf("name %s %d\n", b.e[b.n - 1].name, jb200_blob_get_i(&b, "CUT", 0));
  jb200_blob_free(&b);
  return 0;
}
'''
    cfile = tmp_path / "readers.c"
    long_name = "x" * 40 + "_cut_here"
    cfile.write_text(src.replace("LONG", long_name).replace("CUT", long_name[:47]))
    exe = str(tmp_path / "readers")
    subprocess.run(["gcc", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", exe, str(cfile)],
                   check=True)
    tiny, dnn = Golden("tiny"), Golden("small_dnn")
    out = subprocess.run([exe, os.path.join(tiny.dir, "model.jb2m"), os.path.join(dnn.dir, "model.jb2m")],
                         capture_output=True, text=True, check=True).stdout.splitlines()
    rows = {ln.split()[0]: [int(v) if v.lstrip("-").isdigit() else v for v in ln.split()[1:]] for ln in out}

    def want(g, rc, dim, n_gauss, has_mean):
        return [rc, g.n_states, dim, n_gauss, g.iwcd_method, g.iwcd_nbest, g.n_cdsets, g.n_cdset_states,
                int(g.cd_off[g.n_cdsets]), has_mean]
    g = tiny.ds.gmm
    assert rows["gmm"] == want(g, 0, g.dim, g.n_gauss, 1)
    c = dnn.ds.cd_only_gmm()
    assert c.n_cdsets > 0
    assert rows["cd"] == want(c, 0, 0, 0, 0)
    assert rows["short"][0] == -1
    assert rows["name"] == [long_name[:47], 7]


def test_product_path_fails_loudly_without_a_device():
    """No CPU fallback: on a machine without an sm_90 GPU every create call of the C-ABI must return an error (and the
    Python mirror raise), never hand back a handle that computes on the host."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    g = Golden("tiny")
    with pytest.raises(capi.Jb200Error):
        capi.GmmScorer(g.ds, mode=capi.GMM_EXACT)
    d = Golden("small_dnn")
    with pytest.raises(capi.Jb200Error):
        capi.DnnScorer(d.ds)
    assert capi.lib().jb200_device_count() <= 0 or True      # the call itself must not crash


def test_dnn_create_refuses_inconsistent_widths():
    """jb200_dnn_create checks the net's widths before it looks for a device: an in_dim other than the first layer's
    input, an out_dim other than the last layer's output, a layer input other than the previous layer's output, or a
    width below 1 is JB200_ERR_ARG, with or without a GPU."""
    from util import dnn_blob
    rng = np.random.default_rng(0)
    w0, w1 = rng.standard_normal((8, 5)).astype(np.float32), rng.standard_normal((3, 8)).astype(np.float32)
    good = dnn_blob([w0, w1], [np.zeros(8, np.float32), np.zeros(3, np.float32)], np.zeros(3, np.float32))
    bad = {"in_dim": {"dnn.in_dim": 6}, "out_dim": {"dnn.out_dim": 4}, "zero_width": {"dnn.l0.out": 0, "dnn.l1.in": 0},
           "zero_in": {"dnn.in_dim": 0, "dnn.l0.in": 0}, "zero_out": {"dnn.out_dim": 0, "dnn.l1.out": 0},
           "chain": {"dnn.l0.out": 9}}

    def create(blob):
        h = C.c_void_p()
        rc = capi.lib().jb200_dnn_create(C.byref(desc.Descriptors(blob).dnn), 0, C.byref(h))
        if h:
            capi.lib().jb200_dnn_destroy(h)
        return rc

    for name, change in bad.items():
        blob = dict(good)
        blob.update({k: np.array([v], np.int32) for k, v in change.items()})
        assert create(blob) == -1, name                           # JB200_ERR_ARG
    assert create(good) in (0, -3)                               # JB200_OK, or JB200_ERR_NODEVICE without a GPU


def test_gmm_create_refuses_unsupported_descriptors():
    """jb200_gmm_create checks -tmix, -iwcd1 best, the mixtures per state and the feature dimension (25, 26, 38 or 39
    when the model has Gaussians) before it looks for a device: each is JB200_ERR_UNSUPPORTED, with or without a GPU."""
    g = Golden("tiny")
    too_many_mix = g.blob["gmm.state_off"].copy()
    too_many_mix[1] = too_many_mix[0] + 65

    def create(blob, **fields):
        ds = desc.Descriptors(blob)
        for k, v in fields.items():
            setattr(ds.gmm, k, v)
        h = C.c_void_p()
        rc = capi.lib().jb200_gmm_create(C.byref(ds.gmm), 0, capi.GMM_EXACT, C.byref(h))
        if h:
            capi.lib().jb200_gmm_destroy(h)
        return rc

    assert create(g.blob, gprune_method=1, gprune_num=0) == -4               # -tmix 0 with pruning on
    assert create(g.blob, iwcd_method=2, iwcd_nbest=17) == -4                # -iwcd1 best 17
    assert create(dict(g.blob, **{"gmm.state_off": too_many_mix})) == -4     # a state with 65 mixtures
    assert create(g.blob, dim=13) == -4                                      # a feature dimension K1 is not built for
    assert create(g.blob, dim=13, n_gauss=0) in (0, -3)                      # cd sets only: the dimension is not used
    assert create(g.blob) in (0, -3)                                         # JB200_OK, or JB200_ERR_NODEVICE without a GPU


def test_decoder_create_refuses_bad_trees():
    """jb200_decoder_create checks the tree before it looks at the acoustic model or the device, so each bad tree gets its
    own error code even with no acoustic model, with or without a GPU; a good tree then gets JB200_ERR_ARG for the
    missing model.  The too-many-roots refusal is not covered: it needs a tree with 2^18 roots."""
    def tree(case, mutate=None, **fields):
        blob = dict(Golden(case).blob)
        if mutate:
            mutate(blob)
        ds = desc.Descriptors(blob)
        for k, v in fields.items():
            setattr(ds.tree, k, v)
        return ds

    def put(blob, name, i, v):
        blob["tree." + name] = a = blob["tree." + name].copy()
        a[i] = v

    cases = {
        "unknown lm_type": (tree("small_b100", lm_type=7), -4),
        "grammar on a multipath tree": (tree("small_dfa", multipath=1), -4),
        "grammar without start nodes": (tree("small_dfa", n_init=0), -1),
        "grammar with a transparent word": (tree("small_dfa", lambda b: put(b, "is_transparent", 0, 1)), -4),
        "tree too large": (tree("small_b100", n_nodes=1 << 28), -4),
        "no head silence": (tree("small_b100", head_silwid=-1), -4),
        "transparent head silence": (tree("small_b100", lambda b: put(b, "is_transparent", b["tree.head_silwid"][0], 1)), -4),
        "beam width 0": (tree("small_b100", beam_width=0), -4),
        "beam width 8001": (tree("small_b100", beam_width=8001), -4),
        "non-emitting node in a non-multipath tree": (tree("tiny", lambda b: put(b, "outstyle", 0, 255)), -4),
        "shared root without a factoring value": (tree("small_b100", lambda b: put(b, "scid", b["tree.shared_node"][0], 0)), -1),
    }
    for case in ("tiny", "small_b100", "small_dfa"):
        cases[f"{case} without an acoustic model"] = (tree(case), -1)
    for name, (ds, want) in cases.items():
        h = C.c_void_p()
        assert capi.lib().jb200_decoder_create(C.byref(ds.tree), None, 1, 64, C.byref(h)) == want, name
        assert not h, name


def test_nothing_in_the_product_imports_the_oracle():
    """oracle/ is test infrastructure: no module of julius_b200/ and none of the C/CUDA sources may reference it."""
    pkg = os.path.join(ROOT, "julius_b200")
    bad = []
    for dirpath, _, files in os.walk(pkg):
        if "_obj" in dirpath:
            continue
        for fn in files:
            if not fn.endswith((".py", ".cu", ".cuh", ".inc", ".c", ".h")):
                continue
            txt = open(os.path.join(dirpath, fn), errors="ignore").read()
            if re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M) or "liboracle" in txt or "oracle/restate" in txt or '#include "oracle' in txt:
                bad.append(os.path.relpath(os.path.join(dirpath, fn), ROOT))
    assert not bad, bad


def test_user_lm_export_limits_are_loud(tmp_path):
    """-userlm is tabulated densely over the dictionary by the export step: a dictionary above the limit must make the
    start-up fail with a message, not produce a model that silently ignores the user functions."""
    import os
    import pytest
    from oracle import ffi, fixtures
    if not ffi.have_ref():
        pytest.skip("oracle/_ref not built")
    d = str(tmp_path)
    with pytest.raises(RuntimeError):
        fixtures.make_fixture("small", d, n_utts=1, n_frames=50, extra_args=["-userlm", "-b", "60"],
                              env_extra={"JREF_USERLM": "1", "JB200_USERLM_MAXWORDS": "100"})
    assert not os.path.exists(os.path.join(d, "model.jb2m"))
    # within the limit the same call exports (402 words)
    m, files, dump, out = fixtures.make_fixture("small", d, n_utts=1, n_frames=50, extra_args=["-userlm", "-b", "60"],
                                                env_extra={"JREF_USERLM": "1"})
    assert os.path.getsize(os.path.join(d, "model.jb2m")) > 402 * 402 * 8
