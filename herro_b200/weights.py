"""Weights container for the forward stage ("HB200W1" flat blob).

The reference loads an opaque TorchScript archive (src/inference.rs:185) whose production
files (model_v0.1.pt / model_R9_v0.1.pt, Zenodo 12683277) are not available offline
(SURVEY.md §0 F1).  The forward implemented here is the architecture named by
BASELINE.json:north_star — conv stem, read-axis multi-head attention, per-position FFN,
base head + informative-position head — behind the reference's exact model I/O contract
(bases i32 [B,L,31], quals f32 [B,L,31], lens i32 [B], indices List[i32] ->
info_logits [sum lens], bases_logits [sum lens,5]; src/inference.rs:155-172).

Tensors are stored in *inference form* (BatchNorm folded into the stem conv), fp32, with
PyTorch `nn.Linear` orientation ([out, in]).  This module is numpy-only: it can create a
deterministic random-init model (there is no network to fetch checkpoints) and read/write
the blob that `hb_create()` loads.  tools/export_weights.py converts a torch state_dict /
TorchScript archive of this architecture into the same blob.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, asdict

import numpy as np

MAGIC = b"HB200W1\0"
VERSION = 1         # a blob with position layers is VERSION_POS, so that a library without the stage rejects it
VERSION_POS = 2
N_READS = 31        # TOP_K_SORT + 1, src/features.rs:22
N_TOKENS = 12       # BASES_MAP alphabet + padding, src/inference.rs:15,23-31
EMB_DIM = 6         # as in the only shipped graph (resources/model.pt: Embedding(12, 6, padding_idx=11))
N_CLASSES = 5       # A C G T *, src/consensus.rs:142-149


@dataclass(frozen=True)
class NetConfig:
    stem_k: int = 33        # taps along positions, per read (legacy stem: Conv2d(7->128, k=(33,1)))
    channels: int = 128     # d_model
    heads: int = 4
    layers: int = 2
    ffn: int = 512
    collapse: int = 256     # read-axis collapse (legacy: Conv2d(128->256, k=(1,31)))
    pos_layers: int = 0     # encoder layers across each window's supported positions (0: no such stage)
    pos_heads: int = 0
    pos_ffn: int = 0

    @property
    def head_dim(self):
        return self.channels // self.heads


def tensor_shapes(cfg: NetConfig):
    C, F, D, K = cfg.channels, cfg.ffn, cfg.collapse, cfg.stem_k
    shapes = {
        "emb": (N_TOKENS, EMB_DIM),
        "stem_w": (C, EMB_DIM + 1, K),
        "stem_b": (C,),
        "read_pos": (N_READS, C),
    }
    for l in range(cfg.layers):
        p = f"l{l}."
        shapes.update({
            p + "ln1_g": (C,), p + "ln1_b": (C,),
            p + "wqkv": (3 * C, C), p + "bqkv": (3 * C,),
            p + "wo": (C, C), p + "bo": (C,),
            p + "ln2_g": (C,), p + "ln2_b": (C,),
            p + "w1": (F, C), p + "b1": (F,),
            p + "w2": (C, F), p + "b2": (C,),
        })
    shapes.update({
        "lnf_g": (C,), "lnf_b": (C,),
        "wc": (D, N_READS * C), "bc": (D,),
        "wb": (N_CLASSES, D), "bb": (N_CLASSES,),
        "wi": (1, D), "bi": (1,),
    })
    P = cfg.pos_ffn
    for l in range(cfg.pos_layers):  # after "bi": the random draws of every other tensor stay those of the graph without the stage
        p = f"p{l}."
        shapes.update({
            p + "ln1_g": (D,), p + "ln1_b": (D,),
            p + "wqkv": (3 * D, D), p + "bqkv": (3 * D,),
            p + "wo": (D, D), p + "bo": (D,),
            p + "ln2_g": (D,), p + "ln2_b": (D,),
            p + "w1": (P, D), p + "b1": (P,),
            p + "w2": (D, P), p + "b2": (D,),
        })
    return shapes


def random_weights(cfg: NetConfig = NetConfig(), seed: int = 0) -> dict:
    """Deterministic random init, scaled so logits are O(1-5) (decisive argmax)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shp in tensor_shapes(cfg).items():
        base = name.split(".")[-1]
        if base.endswith("_g"):
            t = 1.0 + 0.1 * rng.standard_normal(shp)
        elif base.startswith("b") or base.endswith("_b"):
            t = 0.05 * rng.standard_normal(shp)
        elif base == "emb":
            t = rng.standard_normal(shp)
            t[N_TOKENS - 1] = 0.0          # padding_idx = 11
        elif base == "read_pos":
            t = 0.5 * rng.standard_normal(shp)
        elif base in ("wb", "wi"):
            t = rng.standard_normal(shp) * (3.0 / np.sqrt(shp[-1]))
        else:
            fan_in = int(np.prod(shp[1:]))
            t = rng.standard_normal(shp) * (1.0 / np.sqrt(fan_in))
            if base == "stem_w":
                t *= 2.0
        out[name] = np.ascontiguousarray(t, dtype=np.float32)
    return out


_HDR = struct.Struct("<8sII16I")
_ENT = struct.Struct("<48sII4IQQ")


def save_blob(path: str, cfg: NetConfig, tensors: dict) -> None:
    shapes = tensor_shapes(cfg)
    names = list(shapes.keys())
    for n in names:
        if tuple(tensors[n].shape) != tuple(shapes[n]):
            raise ValueError(f"{n}: shape {tensors[n].shape} != {shapes[n]}")
    cfgv = [N_TOKENS, EMB_DIM, N_READS, cfg.stem_k, cfg.channels, cfg.heads, cfg.layers, cfg.ffn, cfg.collapse,
            N_CLASSES, cfg.pos_layers, cfg.pos_heads, cfg.pos_ffn] + [0] * 3
    off = _HDR.size + _ENT.size * len(names)
    off = (off + 63) // 64 * 64
    ents, blobs = [], []
    for n in names:
        a = np.ascontiguousarray(tensors[n], dtype="<f4")
        shp = list(a.shape) + [1] * (4 - a.ndim)
        ents.append(_ENT.pack(n.encode(), 0, a.ndim, *shp, off, a.nbytes))
        blobs.append((off, a.tobytes()))
        off = (off + a.nbytes + 63) // 64 * 64
    with open(path, "wb") as f:
        f.write(_HDR.pack(MAGIC, VERSION_POS if cfg.pos_layers else VERSION, len(names), *cfgv))
        for e in ents:
            f.write(e)
        for o, b in blobs:
            f.seek(o)
            f.write(b)
        f.truncate(off)


def load_blob(path: str):
    with open(path, "rb") as f:
        buf = f.read()
    magic, ver, nt, *cfgv = _HDR.unpack_from(buf, 0)
    if magic != MAGIC or ver not in (VERSION, VERSION_POS):
        raise ValueError("not an HB200W1 weights blob")
    if cfgv[0] != N_TOKENS or cfgv[1] != EMB_DIM or cfgv[2] != N_READS or cfgv[9] != N_CLASSES:
        raise ValueError("unsupported fixed dimensions in weights blob")
    cfg = NetConfig(stem_k=cfgv[3], channels=cfgv[4], heads=cfgv[5], layers=cfgv[6], ffn=cfgv[7], collapse=cfgv[8],
                    pos_layers=cfgv[10], pos_heads=cfgv[11], pos_ffn=cfgv[12])
    tensors = {}
    for i in range(nt):
        name, dt, nd, s0, s1, s2, s3, off, nb = _ENT.unpack_from(buf, _HDR.size + i * _ENT.size)
        name = name.rstrip(b"\0").decode()
        shp = (s0, s1, s2, s3)[:nd]
        tensors[name] = np.frombuffer(buf, dtype="<f4", count=nb // 4, offset=off).reshape(shp).copy()
    return cfg, tensors


def config_dict(cfg: NetConfig):
    return asdict(cfg)
