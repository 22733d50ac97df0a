"""The encoder stage across each window's supported positions on the GPU: the masked variable-length attention kernel
against float64, and whole runs against the reference graph (tools/pos_forward_ref.py)."""
import numpy as np
import pytest

import helpers
from herro_b200 import api, weights as hbw

pytestmark = pytest.mark.gpu
HB_ERR_MODEL = -3
POS2 = hbw.NetConfig(pos_layers=2, pos_heads=8, pos_ffn=1024)
POS1 = hbw.NetConfig(pos_layers=1, pos_heads=4, pos_ffn=512)


def _attention64(lens, heads, dh, qkv):
    D = heads * dh
    out = np.zeros((qkv.shape[0], D))
    o = 0
    for n in lens:
        x = qkv[o:o + n].astype(np.float64)
        for h in range(heads):
            q, k, v = (x[:, s * D + h * dh:s * D + (h + 1) * dh] for s in range(3))
            s_ = q @ k.T / np.sqrt(dh)
            p = np.exp(s_ - s_.max(axis=1, keepdims=True))
            out[o:o + n, h * dh:(h + 1) * dh] = (p / p.sum(axis=1, keepdims=True)) @ v
        o += n
    return out


@pytest.mark.parametrize("heads,dh", [(8, 32), (4, 64)])
def test_masked_attention_kernel_against_float64(heads, dh):
    rng = np.random.default_rng(dh)
    worst = 0.0
    cases = [[n] for n in (1, 2, 15, 16, 17, 31, 63, 64, 65, 127, 128, 129, 255, 1000, 3000)]
    cases.append(list(rng.integers(1, 41, 5000)))
    for lens in cases:
        qkv = rng.uniform(-1, 1, (int(sum(lens)), 3 * heads * dh)).astype(np.float32)
        got, _ = api.selftest_pos_attention(lens, heads, dh, qkv)
        err = float(np.abs(got - _attention64(lens, heads, dh, qkv)).max())
        assert err <= 3e-5, (lens[:3], len(lens), err)  # measured on an H100: at most 9.4e-6
        worst = max(worst, err)
    print(f"dh {dh}: max |error| {worst:.2e}")


def _run_oracle(monkeypatch, rs, model, W, b):
    from oracle import forward_ref
    from tools import pos_forward_ref
    monkeypatch.setattr(forward_ref, "from_weights", pos_forward_ref.from_weights)
    return helpers.run_oracle(rs, model, window_size=W, batch_size=b)


@pytest.mark.parametrize("cfg", [POS2, POS1], ids=["L2H8F1024", "L1H4F512"])
@pytest.mark.parametrize("profile,W,b,seed", [("r10", 4096, 64, 11), ("r10", 1024, 4, 5), ("r9", 4096, 64, 7)],
                         ids=["r10-W4096-b64", "r10-W1024-b4", "r9"])
def test_stage_graph_against_the_reference(monkeypatch, cfg, profile, W, b, seed):
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=seed, profile=profile)
    model = helpers.model_path(seed=3, cfg=cfg)
    ora = _run_oracle(monkeypatch, rs, model, W, b)
    if b == 4:  # groups of unequal windows: the reference graph really pads and masks
        assert any(len({len(ora["windows"][(t, w)].sup_rows) for w in range(g, g + 4) if (t, w) in ora["windows"]}) > 1
                   for t in ora["segments"] for g in range(0, 64, 4))
    got = helpers.run_product(rs, model, W, b, keep_debug=True)
    r = helpers.compare(ora, got, logits_tol=1e-3)
    assert r["windows"] > 0 and got["stats"]["n_kernel"]["pos_attn"] > 0 and got["stats"]["class_flops"]["pos_attn"] > 0
    print(r)


def test_forward_passes_hold_whole_windows(monkeypatch):
    """HERRO_B200_CHUNK_POS=128 splits the launch into passes of whole windows; a window with more supported positions is
    a pass of its own.  The outputs are bit-identical to a single pass."""
    rs = helpers.small_readset(n_reads=24, mean_len=12000, seed=1, profile="r9")
    model = helpers.model_path(seed=3, cfg=POS2)
    one = helpers.run_product(rs, model, 8192, 64, keep_debug=True)
    assert max(len(w["sup_rows"]) for w in one["windows"].values()) > 128
    monkeypatch.setenv("HERRO_B200_CHUNK_POS", "128")
    many = helpers.run_product(rs, model, 8192, 64, keep_debug=True)
    assert many["stats"]["n_kernel"]["heads"] > one["stats"]["n_kernel"]["heads"]
    assert many["segments"] == one["segments"]
    for key, w in one["windows"].items():
        assert np.array_equal(w["bases_logits"], many["windows"][key]["bases_logits"]), key
        assert np.array_equal(w["info_logits"], many["windows"][key]["info_logits"]), key


def test_torchscript_archive_of_the_stage_graph(tmp_path):
    import torch
    from tools import pos_forward_ref
    blob = helpers.model_path(seed=3, cfg=POS2)
    pt = str(tmp_path / "pos.pt")
    torch.jit.script(pos_forward_ref.from_weights(*hbw.load_blob(blob))).save(pt)
    rs = helpers.small_readset(n_reads=30, mean_len=8000, seed=4)
    a = helpers.run_product(rs, blob, 4096, 64)
    b = helpers.run_product(rs, pt, 4096, 64)
    assert a["segments"] == b["segments"] and any(a["segments"].values())


@pytest.mark.parametrize("cfg,word", [(hbw.NetConfig(pos_layers=1, pos_heads=16, pos_ffn=512), "pos_heads"),
                                      (hbw.NetConfig(pos_layers=1, pos_heads=8, pos_ffn=200), "pos_ffn")])
def test_unsupported_stage_dimensions_are_rejected(tmp_path, cfg, word):
    from herro_b200 import Context
    p = str(tmp_path / "m.hbw")
    hbw.save_blob(p, cfg, hbw.random_weights(cfg, 1))
    with pytest.raises(api.HerroError) as e:
        Context(p, 0, 4096, 64)
    assert e.value.code == HB_ERR_MODEL and word in str(e.value)


def test_warm_context_with_the_stage_allocates_nothing():
    from herro_b200 import Context
    rs = helpers.small_readset(n_reads=30, mean_len=7000, seed=12)
    ctx = Context(helpers.model_path(seed=3, cfg=POS2), 0, 4096, 64, launch_targets=4)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)

    def run():
        for t in range(rs.n):
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            if a1 > a0:
                ctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
        ctx.flush()
        return {r.rid: r.segments for r in ctx.drain()}

    first = run()
    run()
    ctx.reset_stats()
    assert run() == first
    st = ctx.stats()
    assert st["device_launches"] >= 3 and st["n_kernel"]["pos_attn"] > 0
    assert st["host_allocs"] == 0, st["host_allocs"]
