"""wgmma (bf16x3 split) contraction kernel vs the fp32 SIMT kernel on random data."""
import pytest

from herro_b200 import api

pytestmark = pytest.mark.gpu

SHAPES = [  # M, N, K, act, res, lda_extra  — the shapes the forward uses (C=128, F=512, D=256) and edge cases
    (128, 128, 64, 0, 0, 0),
    (256, 384, 128, 0, 0, 0),      # QKV
    (1024, 128, 128, 0, 1, 0),     # out-proj + residual
    (1024, 512, 128, 2, 0, 0),     # FFN1 + ReLU, split-bf16 output
    (1024, 128, 512, 0, 1, 0),     # FFN2 + residual
    (256, 256, 3968, 1, 0, 128),   # read-axis collapse, lda = 32*C
    (384, 256, 192, 0, 0, 64),     # odd sizes, padded lda
    (128 * 301, 384, 128, 0, 0, 0),  # more work items than SMs: persistent loop, ring wrap-around
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_tc_matches_simt(shape):
    M, N, K, act, res, extra = shape
    r = api.selftest_gemm(M, N, K, act, res, extra)
    # bf16x3: ~2^-17 relative per product on top of fp32 accumulation-order noise of both kernels
    assert r["max_abs_err"] <= 3e-5 * max(1.0, r["max_abs_ref"]), r
