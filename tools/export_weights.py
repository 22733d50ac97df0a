#!/usr/bin/env python
"""Convert a torch state_dict / TorchScript archive of the HerroNet architecture
(oracle/forward_ref.py naming) into the HB200W1 blob that hb_create() loads.
BatchNorm after the stem, if present (`stem_bn.*`), is folded into the conv (eval mode, eps 1e-5).

  python tools/export_weights.py model.pt out.hbw
"""
import sys
import os

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from herro_b200 import weights as hbw  # noqa: E402


def state_dict_to_tensors(sd):
    g = lambda k: np.asarray(sd[k].detach().cpu().numpy() if hasattr(sd[k], "detach") else sd[k], dtype=np.float32)
    stem_w = g("stem.weight")[..., 0]            # [C,7,K,1] -> [C,7,K]
    stem_b = g("stem.bias")
    if "stem_bn.weight" in sd:                    # fold BN: y = (conv - mean) * gamma / sqrt(var + eps) + beta
        s = g("stem_bn.weight") / np.sqrt(g("stem_bn.running_var") + 1e-5)
        stem_w = stem_w * s[:, None, None]
        stem_b = (stem_b - g("stem_bn.running_mean")) * s + g("stem_bn.bias")
    C, _, K = stem_w.shape
    layers = 0
    while f"layers.{layers}.qkv.weight" in sd:
        layers += 1
    F = g("layers.0.ff1.weight").shape[0]
    D = g("collapse.weight").shape[0]
    dh_heads = None
    T = {"emb": g("embedding.weight"), "stem_w": stem_w, "stem_b": stem_b, "read_pos": g("read_pos")}
    for l in range(layers):
        p, q = f"layers.{l}.", f"l{l}."
        T.update({q + "ln1_g": g(p + "ln1.weight"), q + "ln1_b": g(p + "ln1.bias"), q + "wqkv": g(p + "qkv.weight"),
                  q + "bqkv": g(p + "qkv.bias"), q + "wo": g(p + "out.weight"), q + "bo": g(p + "out.bias"),
                  q + "ln2_g": g(p + "ln2.weight"), q + "ln2_b": g(p + "ln2.bias"), q + "w1": g(p + "ff1.weight"),
                  q + "b1": g(p + "ff1.bias"), q + "w2": g(p + "ff2.weight"), q + "b2": g(p + "ff2.bias")})
    T.update({"lnf_g": g("lnf.weight"), "lnf_b": g("lnf.bias"), "wc": g("collapse.weight"), "bc": g("collapse.bias"),
              "wb": g("base_head.weight"), "bb": g("base_head.bias"), "wi": g("info_head.weight"), "bi": g("info_head.bias")})
    dims = dict(stem_k=K, channels=C, layers=layers, ffn=F, collapse=D)
    pos_layers = 0  # the optional encoder stage across a window's supported positions (tools/pos_forward_ref.py naming)
    while f"pos_layers.{pos_layers}.qkv.weight" in sd:
        pos_layers += 1
    for l in range(pos_layers):
        p, q = f"pos_layers.{l}.", f"p{l}."
        T.update({q + "ln1_g": g(p + "ln1.weight"), q + "ln1_b": g(p + "ln1.bias"), q + "wqkv": g(p + "qkv.weight"),
                  q + "bqkv": g(p + "qkv.bias"), q + "wo": g(p + "out.weight"), q + "bo": g(p + "out.bias"),
                  q + "ln2_g": g(p + "ln2.weight"), q + "ln2_b": g(p + "ln2.bias"), q + "w1": g(p + "ff1.weight"),
                  q + "b1": g(p + "ff1.bias"), q + "w2": g(p + "ff2.weight"), q + "b2": g(p + "ff2.bias")})
    if pos_layers:
        dims.update(pos_layers=pos_layers, pos_ffn=g("pos_layers.0.ff1.weight").shape[0])
    return dims, T


def main():
    import torch
    src, dst = sys.argv[1], sys.argv[2]
    heads = int(sys.argv[3]) if len(sys.argv) > 3 else 4
    pos_heads = int(sys.argv[4]) if len(sys.argv) > 4 else 0
    try:
        m = torch.jit.load(src, map_location="cpu")
        sd = m.state_dict()
        sub = dict(m.named_modules()).get("pos_layers.0")
        if sub is not None:
            pos_heads = int(sub.H)
    except Exception:
        sd = torch.load(src, map_location="cpu")
        sd = sd.get("state_dict", sd)
    dims, T = state_dict_to_tensors(sd)
    if dims.get("pos_layers"):
        if not pos_heads:
            raise SystemExit("the model has position layers: give their head count (pos_layers.0.H) as the 4th argument")
        dims["pos_heads"] = pos_heads
    cfg = hbw.NetConfig(heads=heads, **dims)
    hbw.save_blob(dst, cfg, T)
    print("wrote", dst, cfg)


if __name__ == "__main__":
    main()
