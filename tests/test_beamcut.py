"""CPU: the models of the beam cut in tools/beamcut.cpp -- the pipelined replay (heap_pipe.cuh), the closed form with
its relocation pass as heap_select_closed / closed_relocate run it, and the invariant (I) it rests on -- each against the
reference's sort_token_upward/_downward loop (beam.c:1342-1447); and the candidate sort network against std::sort."""
import os
import re
import shutil
import subprocess

import pytest

from util import ROOT

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")

DISTINCT = ["20000", "300", "8", "2"]       # distinct scores: hardly any exact ties ... nothing but ties


@pytest.fixture(scope="module")
def beamcut(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("beamcut") / "beamcut")
    subprocess.run(["g++", "-O2", "-o", exe, os.path.join(ROOT, "tools", "beamcut.cpp")], check=True)
    return exe


@pytest.fixture(scope="module")
def random_run(beamcut):
    """`beamcut random <distinct> 800` (upward and downward selects of up to 2600 tokens), run once per tie level:
    (the line with the selects it ran, the line with the mismatches of every model)."""
    runs = {}

    def run(distinct):
        if distinct not in runs:
            p = subprocess.run([beamcut, "random", distinct, "800"], capture_output=True, text=True)
            assert p.returncode == 0, p.stdout + p.stderr
            ran = re.search(r"selects: upward (\d+), downward (\d+); relocation pass in (\d+)", p.stdout)
            mism = re.search(r"mismatches (\d+) \(replay (\d+), closed form (\d+), invariant (\d+)\)", p.stdout)
            assert ran and mism, p.stdout
            runs[distinct] = (tuple(map(int, ran.groups())), tuple(map(int, mism.groups())))
        return runs[distinct]
    return run


@pytest.mark.parametrize("distinct", DISTINCT)
def test_replay_equals_the_reference_loop(random_run, distinct):
    """The pipelined replay: upward extraction order with and without the loser cut, the whole array select_exact
    leaves, and the downward arrangement with its extracted roots."""
    (up, down, _), (total, replay, _, _) = random_run(distinct)
    assert up > 0 and down > 0
    assert replay == 0 and total == 0


@pytest.mark.parametrize("distinct", DISTINCT)
def test_closed_form_with_relocations_equals_the_reference_loop(random_run, distinct):
    """The closed form as the kernel runs it (packed keys, the sort network, the flagging test, closed_relocate lane by
    lane) and the invariant (I) with subtree queries, on every upward select."""
    (up, _, relocated), (total, _, closed, invariant) = random_run(distinct)
    assert up > 0 and relocated > 0
    assert closed == 0 and invariant == 0 and total == 0


def test_tiled_bitonic_network_sorts_descending_at_every_power_of_two(beamcut):
    p = subprocess.run([beamcut, "sort", "13"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "mismatches 0" in p.stdout
    assert "np  8192" in p.stdout and "np     2" in p.stdout
    assert "np  1024: 10 barriers" in p.stdout
