"""CPU: the designed DNNs of tests/test_gpu_dnn_shapes.py are what they claim to be.  For the one-hot nets and the
exact-grid nets, the restatement of dnn_calc_outprob must give, bit for bit, what numpy gives from the exact float64
logits (asserted representable in float32) followed by a float32 emulation of addlog_array.  This shows without a GPU
that the logits of those nets leave no room for rounding, so the GPU test may ask for identical bits."""
import numpy as np
import pytest

from julius_b200 import desc
from util import EXACT_PATTERNS, addlog_array_np, addlog_table_np, exact_grid_net, one_hot_softmax_net, \
    single_layer_scores_np

NORMALISER_N = [1, 2, 3, 255, 256, 257, 3000, 9001]
IN_DIMS = [1, 7, 8, 9, 16, 63, 64, 65, 120, 129, 429, 528]
OUT_DIMS = [1, 2, 3, 5, 127, 128, 129, 240, 257, 3001]


@pytest.fixture(scope="module")
def tbl(oracle_lib):
    t = addlog_table_np()
    assert np.array_equal(t, oracle_lib.addlog_table())
    return t


def test_addlog_emulation_against_fp64(tbl):
    """the emulation is a log-sum-exp: within the table's step of the float64 value on broad rows"""
    a = np.random.default_rng(1).standard_normal((4, 3000)).astype(np.float32) * 3
    want = np.log(np.exp(a.astype(np.float64)).sum(1))
    assert np.abs(addlog_array_np(a, tbl) - want).max() < 1e-3


@pytest.mark.parametrize("n", NORMALISER_N)
def test_one_hot_nets_are_exact(n, tbl, oracle_lib):
    blob, x, _ = one_hot_softmax_net(n, seed=n)
    got = oracle_lib.dnn_score(desc.Descriptors(blob), x)
    want = single_layer_scores_np(blob, x, tbl)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("pattern", list(EXACT_PATTERNS))
@pytest.mark.parametrize("in_dim", IN_DIMS)
def test_exact_grid_nets_are_exact(in_dim, pattern, tbl, oracle_lib):
    for out_dim in OUT_DIMS:
        blob, x = exact_grid_net(in_dim, out_dim, 129, pattern, seed=in_dim * 10007 + out_dim)
        got = oracle_lib.dnn_score(desc.Descriptors(blob), x)
        want = single_layer_scores_np(blob, x, tbl)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (in_dim, out_dim)
