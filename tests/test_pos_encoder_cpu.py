"""The optional encoder stage across each window's supported positions: model files, the reference graph, TorchScript."""
import struct

import numpy as np
import pytest

import helpers
from herro_b200 import api, weights as hbw

torch = pytest.importorskip("torch")
from tools import pos_forward_ref  # noqa: E402
from oracle import forward_ref  # noqa: E402

HB_ERR_MODEL = -3
POS = hbw.NetConfig(pos_layers=2, pos_heads=8, pos_ffn=1024)


def _header(path):
    with open(path, "rb") as f:
        magic, ver, nt, *cfg = struct.unpack("<8sII16I", f.read(struct.calcsize("<8sII16I")))
    return ver, cfg


def test_blob_round_trip_and_version(tmp_path):
    T = hbw.random_weights(POS, 4)
    p = str(tmp_path / "pos.hbw")
    hbw.save_blob(p, POS, T)
    ver, cfg = _header(p)
    assert ver == 2 and cfg[10:13] == [2, 8, 1024] and cfg[13:] == [0, 0, 0]
    cfg2, T2 = hbw.load_blob(p)
    assert cfg2 == POS and T2.keys() == T.keys() and all(np.array_equal(T[k], T2[k]) for k in T)
    assert list(T)[-24:] == [n for n in hbw.tensor_shapes(POS) if n.startswith("p")]
    ver, cfg = _header(helpers.model_path(seed=3))
    assert ver == 1 and cfg[10:16] == [0] * 6


def test_random_weights_keep_the_draws_of_the_graph_without_the_stage():
    a, b = hbw.random_weights(hbw.NetConfig(), 3), hbw.random_weights(POS, 3)
    assert set(a) < set(b)
    assert all(np.array_equal(a[k], b[k]) for k in a)


def _net(cfg=POS, seed=3):
    return pos_forward_ref.from_weights(cfg, hbw.random_weights(cfg, seed))


def _batch(lens, L=60, seed=0):
    rng = np.random.default_rng(seed)
    B = len(lens)
    bases = rng.integers(0, 11, (B, L, 31)).astype(np.uint8)
    quals = rng.integers(33, 80, (B, L, 31)).astype(np.uint8)
    idx = [np.sort(rng.choice(L, n, replace=False)).astype(np.int32) for n in lens]
    return bases, quals, np.asarray(lens, dtype=np.int32), idx


def _close(info_a, bl_a, info_b, bl_b):
    # fp32 contractions of other batch shapes round differently: within 1e-6 of the window's largest logit (or of 1)
    tol = 1e-6 * max(1.0, float(np.abs(bl_b).max(initial=0)))
    return np.abs(bl_a - bl_b).max(initial=0) <= tol and np.abs(info_a - info_b).max(initial=0) <= tol


def test_without_the_stage_the_graph_is_unchanged():
    cfg = hbw.NetConfig()
    T = hbw.random_weights(cfg, 3)
    a = forward_ref.run_batch(forward_ref.from_weights(cfg, T), *_batch([7, 3, 12]))
    b = forward_ref.run_batch(pos_forward_ref.from_weights(cfg, T), *_batch([7, 3, 12]))
    for x, y in zip(a[1] + a[0], b[1] + b[0]):
        assert np.array_equal(x, y)


def test_a_window_alone_equals_the_window_padded_in_a_batch():
    net = _net()
    bases, quals, lens, idx = _batch([5, 0, 23, 9, 1])
    info, bl = forward_ref.run_batch(net, bases, quals, lens, idx)
    for k in np.flatnonzero(lens):  # a batch of one empty window is not a call the graph accepts
        i1, b1 = forward_ref.run_batch(net, bases[k:k + 1], quals[k:k + 1], lens[k:k + 1], idx[k:k + 1])
        assert _close(i1[0], b1[0], info[k], bl[k])


def test_padding_rows_do_not_matter():
    net = _net()
    lens = torch.tensor([3, 11, 6])
    pad = torch.arange(11)[None, :] >= lens[:, None]
    x = torch.randn(3, 11, POS.collapse)
    y = x.clone()
    y[pad] = 1e3 * torch.randn(int(pad.sum()), POS.collapse)
    with torch.no_grad():
        assert torch.equal(net.pos_stage(x, pad)[~pad], net.pos_stage(y, pad)[~pad])


def test_permuting_the_windows_permutes_the_outputs():
    net = _net()
    bases, quals, lens, idx = _batch([4, 17, 9])
    info, bl = forward_ref.run_batch(net, bases, quals, lens, idx)
    perm = [2, 0, 1]
    info2, bl2 = forward_ref.run_batch(net, bases[perm], quals[perm], lens[perm], [idx[i] for i in perm])
    for j, k in enumerate(perm):
        assert _close(info2[j], bl2[j], info[k], bl[k])


def test_positions_attend_across_their_window():
    net = _net()
    bases, quals, lens, idx = _batch([8])
    _, bl = forward_ref.run_batch(net, bases, quals, lens, idx)
    _, bl_first = forward_ref.run_batch(net, bases, quals, np.array([4], np.int32), [idx[0][:4]])
    assert np.abs(bl[0][:4] - bl_first[0]).max() > 1e-4


def test_scripted_archive_of_the_stage_equals_the_blob(tmp_path):
    blob = helpers.model_path(seed=3, cfg=POS)
    pt = str(tmp_path / "pos.pt")
    torch.jit.script(_net()).save(pt)
    d_blob, h_blob = api.inspect_model(blob)
    d_pt, h_pt = api.inspect_model(pt)
    assert d_blob == d_pt == hbw.config_dict(POS)
    assert h_blob == h_pt


def test_export_of_the_stage_graph_round_trips(tmp_path):
    from tools import export_weights
    net = _net()
    dims, T = export_weights.state_dict_to_tensors(net.state_dict())
    assert dims == dict(stem_k=33, channels=128, layers=2, ffn=512, collapse=256, pos_layers=2, pos_ffn=1024)
    ref = hbw.random_weights(POS, 3)
    assert T.keys() == ref.keys() and all(np.array_equal(T[k], ref[k]) for k in T)


def test_foreign_position_layers_are_rejected(tmp_path):
    sd = _net().state_dict()
    bad = dict(sd)
    bad["pos_layers.1.ff1.weight"] = torch.zeros(1000, POS.collapse)
    p = str(tmp_path / "bad.pt")
    torch.save(bad, p)
    with pytest.raises(api.HerroError) as e:
        api.inspect_model(p)
    assert e.value.code == HB_ERR_MODEL
    p = str(tmp_path / "noh.pt")
    torch.save(sd, p)  # a plain state_dict carries no head count
    with pytest.raises(api.HerroError) as e:
        api.inspect_model(p)
    assert e.value.code == HB_ERR_MODEL and "pos_layers.0.H" in str(e.value)


def test_the_stage_is_in_the_abi():
    with open(helpers.os.path.join(helpers.ROOT, "include", "herro_b200.h")) as f:
        h = f.read()
    assert "HB_K_POS_ATTN" in h and api.KERNEL_CLASSES.index("pos_attn") == 15 < 16
    assert {"hb_inspect_model_ex", "hb_selftest_pos_attention"} <= set(api.EXPORTED_SYMBOLS)
