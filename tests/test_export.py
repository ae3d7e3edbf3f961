"""CPU: the export plugin, run again through the compiled reference with the recipe that made each committed model,
writes that model entry for entry.  Every golden and sweep model was made by the exporter, so a change in what it writes
shows up here, at its cause, rather than later as a score or trellis mismatch."""
import importlib.util
import json
import os

import pytest

from julius_b200 import refdump
from util import GOLDEN, ROOT, load_golden_model, load_sweep_case

JREF = os.path.join(ROOT, "oracle", "_ref", "jref")
pytestmark = pytest.mark.skipif(not os.path.exists(JREF), reason="compiled reference (oracle/_ref/jref) not present")

_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(GOLDEN, "make_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)

SWEEP_CASES = make_golden.sweep_cases()


def assert_same_model(got, want):
    assert sorted(got) == sorted(want), f"entries differ: missing {sorted(set(want) - set(got))}, " \
                                        f"extra {sorted(set(got) - set(want))}"
    for k in want:
        assert (got[k].dtype, got[k].size) == (want[k].dtype, want[k].size), f"{k}: dtype or count differs"
        assert got[k].tobytes() == want[k].tobytes(), f"{k}: bytes differ"


@pytest.mark.parametrize("name", list(make_golden.CASES) + list(make_golden.DNN_CASES))
def test_export_reproduces_golden_model(name, tmp_path):
    make_golden.export_case(name, str(tmp_path))
    d = os.path.join(GOLDEN, name)
    with open(os.path.join(d, "meta.json")) as f:
        want = load_golden_model(d, json.load(f))
    assert_same_model(refdump.load_blob(str(tmp_path / "model.jb2m")), want)


@pytest.mark.parametrize("preset,extra,grammar,kw", SWEEP_CASES,
                         ids=[" ".join((["dfa"] if g else []) + [p] + e) for p, e, g, _ in SWEEP_CASES])
def test_export_reproduces_sweep_model(preset, extra, grammar, kw, tmp_path):
    from oracle import fixtures
    fixtures.make_fixture(preset, str(tmp_path), extra_args=extra, grammar=grammar, **kw)
    want = load_sweep_case(preset, extra, grammar)[0].blob
    assert_same_model(refdump.load_blob(str(tmp_path / "model.jb2m")), want)
