"""The device forward at every kernel path the model loader can select, against the reference graph evaluated in float64.

forward.cu picks its kernels from the model's shape: the tensor-core stem `k_stem_tc` (C 128, at most 64 taps) or the SIMT
`k_stem`; the first LayerNorm fused into the stem or run by `k_layernorm`; the fused QKV + attention kernel (C 128, 4 heads) or
the QKV contraction and `k_attention<16|32>`; the fused FFN (C 128, F 512) or the chain of contractions.  Each model below
takes another combination.  Every model has a non-zero pad-token embedding emb[11]: the reference evaluates its stem over the
batch-padding rows (token 11), so the supported rows within K/2 of a window that is shorter than its batch depend on it."""
from typing import NamedTuple

import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api, weights as hbw

pytestmark = pytest.mark.gpu
HB_ERR_MODEL = -3


class Shape(NamedTuple):
    cfg: hbw.NetConfig
    tc_stem: bool      # the tensor-core stem, with the first LayerNorm in its epilogue
    fused_attn: bool   # k_qkv_attn_ws, else the QKV contraction and k_attention
    fused_ffn: bool    # k_ffn_ws with the out-projection in front, else out-projection, FFN1 and FFN2 as contractions


def _cfg(k, c, h, layers, f, d):
    return hbw.NetConfig(stem_k=k, channels=c, heads=h, layers=layers, ffn=f, collapse=d)


SHAPES = {
    "default": Shape(_cfg(33, 128, 4, 2, 512, 256), True, True, True),
    # tensor-core stem in 5 k-blocks, head_dim 16, F 256: the FFN with LayerNorm-fused contractions, D 128
    "ts-shape": Shape(_cfg(17, 128, 8, 3, 256, 128), True, False, False),
    # C 256: SIMT stem, k_layernorm at C 256, every contraction through k_gemm_ws (N 256 / 768, collapse K 7936)
    "wide": Shape(_cfg(33, 256, 8, 2, 512, 256), False, False, False),
    # too many taps for the tensor-core stem at C 128: SIMT stem, separate LayerNorm, then fused; one layer, D 384
    "long-stem": Shape(_cfg(65, 128, 4, 1, 512, 384), False, True, True),
    # the most taps of the tensor-core stem (16 k-blocks) and the most layers
    "max-tc-taps": Shape(_cfg(63, 128, 4, 8, 512, 256), True, True, True),
    "one-tap": Shape(_cfg(1, 128, 4, 2, 512, 256), True, True, True),
    "stem-129": Shape(_cfg(129, 128, 4, 2, 512, 256), False, True, True),
}


def pad_model(cfg, path, pad_embedding=True):
    """random_weights(cfg, 3) with emb[11] drawn from N(0, 1) (or left zero) -> the blob at `path`."""
    T = hbw.random_weights(cfg, 3)
    if pad_embedding:
        T["emb"][11] = np.random.default_rng(11).standard_normal(hbw.EMB_DIM).astype(np.float32)
    hbw.save_blob(path, cfg, T)
    return path


def readset():
    return helpers.small_readset(n_reads=120, mean_len=9000, seed=5, coverage=25.0, min_ovl=600)


# ------------------------------------------------------------------------------------------ the float64 reference
def run_batch64(net, bases_u8, quals_u8, lens, indices):
    """forward_ref.run_batch with the network in float64: the qualities are normalised as the contract does (u8 -> f32, then
    fl(2/93) * q - fl(66/93 + 1) as two fp32 operations) and only then converted."""
    from oracle import forward_ref
    q = forward_ref.QUAL_SCALE * torch.from_numpy(quals_u8).to(torch.float32) - forward_ref.QUAL_OFFSET
    bases = torch.from_numpy(bases_u8).to(torch.int32)
    lens_t = torch.from_numpy(np.asarray(lens, dtype=np.int32))
    idx = [torch.from_numpy(np.asarray(i, dtype=np.int32)) for i in indices]
    with torch.no_grad():
        info, bl = net(bases, q.to(torch.float64), lens_t, idx)
    sizes = [int(n) for n in lens]
    return [t.numpy() for t in torch.split(info, sizes)], [t.numpy() for t in torch.split(bl, sizes)]


def run_oracle64(monkeypatch, rs, model, W, b, targets):
    from oracle import forward_ref
    build = forward_ref.from_weights
    with monkeypatch.context() as m:
        m.setattr(forward_ref, "from_weights", lambda cfg, T: build(cfg, T).double())
        m.setattr(forward_ref, "run_batch", run_batch64)
        return helpers.run_oracle(rs, model, window_size=W, batch_size=b, targets=targets)


# ------------------------------------------------------------------------------------------ rows that see the padding
def pad_reach(batch, wins, K):
    """Per window of a reference batch: which of its supported rows have a stem neighbourhood (rows r - K/2 .. r + K/2) that
    reaches the batch's padding rows (row >= the window's length L and < the batch's Lmax)."""
    lmax = batch.bases.shape[1]
    out = []
    for k, wi in enumerate(batch.win_index):
        L = wins[int(wi)].bases.shape[0]
        out.append((np.asarray(batch.indices[k]) + K // 2 >= L) & (L < lmax))
    return out


def pad_reach_by_window(ora, K):
    """{(rid, wid): bool per supported row} over the oracle's batches."""
    out = {}
    for t, T in ora["targets"].items():
        wins = T.windows()
        for bi in range(T.n_batches):
            B = T.batch(bi)
            for wi, m in zip(B.win_index, pad_reach(B, wins, K)):
                out[(t, wins[int(wi)].wid)] = m
    return out


def targets_reaching_padding(rs, W, b, K, want=20):
    """The first targets, in read order, whose supported rows reach padding rows at least `want` times in all: the float64
    forward is slow on the host, so it runs where the stem's padding rows matter."""
    from oracle import pyoracle as po
    reads = po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)])
    chosen, n = [], 0
    for t in range(rs.n):
        ovl, cigs = rs.target_alns(t)
        if len(ovl) == 0:
            continue
        T = po.Target(reads, t, ovl, cigs, W, b)
        wins = T.windows()
        hit = sum(int(m.sum()) for bi in range(T.n_batches) for m in pad_reach(T.batch(bi), wins, K))
        if hit:
            chosen.append(t)
            n += hit
            if n >= want:
                break
    return chosen


def split_errors(ora, got, reach):
    """Worst |logit - float64| over the rows that reach padding rows and over all other rows."""
    worst = [0.0, 0.0]
    for key, (info, bl) in ora["logits"].items():
        g = got["windows"][key]
        d = np.maximum(np.abs(g["bases_logits"] - bl).max(axis=1, initial=0.0), np.abs(g["info_logits"] - info))
        for i, sel in enumerate((reach[key], ~reach[key])):
            if sel.any():
                worst[i] = max(worst[i], float(d[sel].max()))
    return worst


def expected_launches(shape, tc_stem):
    """Kernel launches per forward pass, by class."""
    L, ln_fused = shape.cfg.layers, shape.cfg.channels == 128
    return dict(stem=1, heads=1, layernorm=(0 if tc_stem else 1) + (0 if ln_fused else 2 * L),
                qkv_attn=L if shape.fused_attn else 0, attention=0 if shape.fused_attn else L,
                ffn=L if shape.fused_ffn else 0, gemm=1 + L * ((0 if shape.fused_attn else 1) + (0 if shape.fused_ffn else 3)))


# ------------------------------------------------------------------------------------------ the forward against float64
CASES = [(name, 1024, 4) for name in SHAPES] + [("default", 4096, 64)]


@pytest.mark.parametrize("name,W,b", CASES, ids=[f"{n}-W{W}-b{b}" for n, W, b in CASES])
def test_forward_against_float64(monkeypatch, tmp_path, name, W, b):
    """The device logits of every supported position within the 1e-3 bound of the float64 graph, segments identical up to
    argmax near-ties.  A shape the tensor-core stem can take runs again with the SIMT stem (HERRO_B200_STEM_SIMT): both
    meet the bound and agree with each other within 1e-4."""
    shape = SHAPES[name]
    K = shape.cfg.stem_k
    model = pad_model(shape.cfg, str(tmp_path / f"{name}_pad_emb.hbw"))
    rs = readset()
    # one tap never reaches another row: its windows are still chosen where 33 taps would reach padding
    targets = targets_reaching_padding(rs, W, b, K if K > 1 else 33)
    ora = run_oracle64(monkeypatch, rs, model, W, b, targets)
    reach = pad_reach_by_window(ora, K)
    n_reach = sum(int(m.sum()) for m in reach.values())
    if K > 1:
        assert n_reach >= 10, n_reach  # otherwise the pad embedding is not exercised
    runs = {}
    for stem in (["simt", "tc"] if shape.tc_stem else ["simt"]):
        with monkeypatch.context() as m:
            if stem == "simt" and shape.tc_stem:
                m.setenv("HERRO_B200_STEM_SIMT", "1")  # read when the context is created
            got = helpers.run_product(rs, model, W, b, targets=targets, keep_debug=True)
        n_kernel = got["stats"]["n_kernel"]
        passes = n_kernel["heads"]
        assert passes > 0
        want = {k: passes * v for k, v in expected_launches(shape, stem == "tc").items()}
        assert {k: n_kernel[k] for k in want} == want
        pad_err, other_err = split_errors(ora, got, reach)
        print(f"{name} W{W} -b{b} {stem} stem: worst |logit - float64| {max(pad_err, other_err):.2e} "
              f"({n_reach} rows reaching padding: {pad_err:.2e}; other rows: {other_err:.2e})")
        r = helpers.compare(ora, got, 1e-3)
        assert r["windows"] > 0
        runs[stem] = got
    if len(runs) == 2:
        a, c = runs["tc"], runs["simt"]
        assert a["segments"] == c["segments"]
        worst = max(max(float(np.abs(w["bases_logits"] - c["windows"][key]["bases_logits"]).max(initial=0.0)),
                        float(np.abs(w["info_logits"] - c["windows"][key]["info_logits"]).max(initial=0.0)))
                    for key, w in a["windows"].items())
        print(f"{name}: worst |tensor-core stem - SIMT stem| {worst:.2e}")
        assert worst <= 1e-4, worst


# ------------------------------------------------------------------------------------------ shapes the loader refuses
REJECTED = {
    "C192": _cfg(33, 192, 6, 2, 512, 256),
    "head-dim-64": _cfg(33, 256, 4, 2, 512, 256),
    "even-taps": _cfg(32, 128, 4, 2, 512, 256),
    "taps-131": _cfg(131, 128, 4, 2, 512, 256),
    "layers-9": _cfg(33, 128, 4, 9, 512, 256),
    "F200": _cfg(33, 128, 4, 2, 200, 256),
    "D200": _cfg(33, 128, 4, 2, 512, 200),
}


@pytest.mark.parametrize("name", list(REJECTED))
def test_unsupported_model_shapes_are_rejected(tmp_path, name):
    from herro_b200 import Context
    p = pad_model(REJECTED[name], str(tmp_path / f"{name}.hbw"))
    with pytest.raises(api.HerroError) as e:
        Context(p, 0, 4096, 64)
    assert e.value.code == HB_ERR_MODEL
