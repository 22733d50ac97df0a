"""The fused FFN kernel (k_ffn_ws) against the chain of separate contractions, at launch shapes where its weight ring and
tile barriers wrap many times (every CTA runs many 128-token tiles) and where a launch has fewer tiles than SMs."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def _assert_same(a, b):
    assert a["segments"] == b["segments"]
    worst = 0.0
    for key, wa in a["windows"].items():
        wb = b["windows"][key]
        worst = max(worst, float(np.abs(wa["bases_logits"] - wb["bases_logits"]).max(initial=0.0)),
                    float(np.abs(wa["info_logits"] - wb["info_logits"]).max(initial=0.0)))
    assert worst <= 1e-4, worst


def test_fused_ffn_many_tiles_per_cta(monkeypatch):
    """One forward pass with at least 10 tiles per CTA and layer: the 4-stage weight ring, the resident tile's barriers and
    their phases cycle many times within and across tiles.  Both kernel variants (out-projection fused in front, and not)
    against the unfused chain."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rs = helpers.small_readset(n_reads=80, mean_len=20000, seed=21, coverage=40.0, min_ovl=2048)
    model = helpers.model_path(seed=3)
    fused = helpers.run_product(rs, model, 4096, 64, keep_debug=True)
    assert fused["stats"]["supported"] >= 10 * 4 * sms  # a tile is 4 supported positions of 32 read tokens
    monkeypatch.setenv("HERRO_B200_NO_FUSE_OPROJ", "1")
    ffn_only = helpers.run_product(rs, model, 4096, 64, keep_debug=True)
    monkeypatch.delenv("HERRO_B200_NO_FUSE_OPROJ")
    monkeypatch.setenv("HERRO_B200_NO_FUSE_FFN", "1")
    unfused = helpers.run_product(rs, model, 4096, 64, keep_debug=True)
    assert unfused["stats"]["kernel_launches"] > ffn_only["stats"]["kernel_launches"] > fused["stats"]["kernel_launches"]
    _assert_same(fused, unfused)
    _assert_same(ffn_only, unfused)


def test_fused_ffn_fewer_tiles_than_sms(monkeypatch):
    """Forward passes of 128 positions (32 tiles): the grid is smaller than the SM count and each CTA runs one tile."""
    rs = helpers.small_readset(n_reads=30, mean_len=7000, seed=22)
    model = helpers.model_path(seed=3)
    monkeypatch.setenv("HERRO_B200_CHUNK_POS", "128")
    fused = helpers.run_product(rs, model, 4096, 64, keep_debug=True)
    assert fused["stats"]["supported"] > 3 * 128
    monkeypatch.setenv("HERRO_B200_NO_FUSE_FFN", "1")
    unfused = helpers.run_product(rs, model, 4096, 64, keep_debug=True)
    assert unfused["stats"]["kernel_launches"] > fused["stats"]["kernel_launches"]
    _assert_same(fused, unfused)
