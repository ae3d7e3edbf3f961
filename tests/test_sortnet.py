"""CPU: the candidate sort of the closed-form beam cut as the kernel runs it (tools/sortnet.cpp: the bitonic network with
its short-distance stages done per 128-key tile over (tile, lane, register) indices, as sort_tile_pass in csrc/beam.cu)
against std::sort."""
import os
import shutil
import subprocess

import pytest

from util import ROOT


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_tiled_bitonic_network_sorts_descending_at_every_power_of_two(tmp_path):
    exe = str(tmp_path / "sortnet")
    subprocess.run(["g++", "-O2", "-o", exe, os.path.join(ROOT, "tools", "sortnet.cpp")], check=True)
    p = subprocess.run([exe, "12"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "mismatches 0" in p.stdout
    assert "np  8192" in p.stdout and "np     2" in p.stdout
    assert "np  1024: 10 barriers" in p.stdout
