"""Plain PyTorch fp32 reference of the forward with the position-axis encoder stage (TEST INFRASTRUCTURE ONLY).

The graph of oracle/forward_ref.py, followed by `pos_layers` pre-LN encoder layers across each window's supported
positions.  Each window of a reference batch group (`lens[b]` positions) is one sequence; the sequences are padded to the
group's longest, a sinusoidal encoding of the position's index in its window is added, and the padding keys are masked
out of every softmax, so a window's result does not depend on the other windows of its group.  No LayerNorm follows the
stage.  The encoding is evaluated in float64 and rounded to float32, as on the device.

`PosHerroNet` is scriptable (torch.jit.script); with no position layers it computes exactly what `forward_ref.HerroNet`
computes.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import forward_ref
from oracle.forward_ref import run_batch  # noqa: F401  (the reference's inference() call, for any HerroNet)

_base_from_weights = forward_ref.from_weights  # the tensors of the graph without the stage (callers may rebind the name)


class PosEncoderLayer(forward_ref.EncoderLayer):
    """forward_ref.EncoderLayer with a key-padding mask (True = padding key: its score is -inf before the softmax)."""

    def forward(self, x: torch.Tensor, pad: Optional[torch.Tensor] = None) -> torch.Tensor:  # [N, S, C], [N, S]
        N, S, C = x.shape
        H = self.H
        dh = C // H
        h = self.ln1(x)
        qkv = self.qkv(h).view(N, S, 3, H, dh)
        q = qkv[:, :, 0].transpose(1, 2)
        k = qkv[:, :, 1].transpose(1, 2)
        v = qkv[:, :, 2].transpose(1, 2)
        att = torch.matmul(q, k.transpose(-1, -2)) * (1.0 / math.sqrt(dh))
        if pad is not None:
            att = att.masked_fill(pad[:, None, None, :], float("-inf"))
        att = torch.softmax(att, dim=-1)
        o = torch.matmul(att, v).transpose(1, 2).reshape(N, S, C)
        x = x + self.out(o)
        h = self.ln2(x)
        x = x + self.ff2(F.relu(self.ff1(h)))
        return x


def sinusoid(S: int, D: int) -> torch.Tensor:
    """pe[k, 2i] = sin(k * 10000^(-2i/D)), pe[k, 2i+1] = cos(...), in float64, rounded to float32: [S, D]."""
    k = torch.arange(S, dtype=torch.float64)[:, None]
    two_i = torch.arange(0, D, 2, dtype=torch.float64)[None, :]
    a = k * torch.pow(torch.full_like(two_i, 10000.0), -(two_i / D))
    pe = torch.zeros((S, D), dtype=torch.float64)
    pe[:, 0::2] = torch.sin(a)
    pe[:, 1::2] = torch.cos(a)
    return pe.to(torch.float32)


class PosHerroNet(forward_ref.HerroNet):
    def __init__(self, stem_k: int = 33, channels: int = 128, heads: int = 4, layers: int = 2, ffn: int = 512,
                 collapse: int = 256, pos_layers: int = 0, pos_heads: int = 8, pos_ffn: int = 1024):
        super().__init__(stem_k, channels, heads, layers, ffn, collapse)
        self.pos_layers = nn.ModuleList([PosEncoderLayer(collapse, pos_heads, pos_ffn) for _ in range(pos_layers)])

    def pos_stage(self, x: torch.Tensor, pad: torch.Tensor) -> torch.Tensor:
        """[B, Smax, D] padded windows, pad [B, Smax] (True = padding) -> the encoded windows (padding rows undefined)."""
        x = x + sinusoid(x.shape[1], x.shape[2])
        for layer in self.pos_layers:
            x = layer(x, pad)
        return x

    def forward(self, bases: torch.Tensor, quals: torch.Tensor, lens: torch.Tensor,
                indices: List[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        x = self.stem_features(bases, quals)
        sel: List[torch.Tensor] = []
        for b in range(len(indices)):
            sel.append(x[b].index_select(0, indices[b].to(torch.long)))
        t = torch.cat(sel, dim=0) + self.read_pos
        for layer in self.layers:
            t = layer(t)
        t = self.lnf(t)
        z = F.relu(self.collapse(t.reshape(t.shape[0], -1)))            # [sum lens, D]
        if len(self.pos_layers) > 0:
            B = lens.shape[0]
            smax = int(lens.max()) if B > 0 else 0
            xp = torch.zeros((B, smax, z.shape[1]), dtype=z.dtype)
            o = 0
            for b in range(B):
                n = int(lens[b])
                xp[b, :n] = z[o:o + n]
                o += n
            pad = torch.arange(smax)[None, :] >= lens.to(torch.long)[:, None]
            z = self.pos_stage(xp, pad)[~pad]                           # back to [sum lens, D], same order
        return self.info_head(z).squeeze(-1), self.base_head(z)


def from_weights(cfg, tensors: dict) -> PosHerroNet:
    """Build the module from a herro_b200.weights blob (cfg: NetConfig, tensors: name->ndarray)."""
    net = PosHerroNet(cfg.stem_k, cfg.channels, cfg.heads, cfg.layers, cfg.ffn, cfg.collapse, cfg.pos_layers,
                      cfg.pos_heads or 1, cfg.pos_ffn)
    base = _base_from_weights(cfg, tensors)
    net.load_state_dict(base.state_dict(), strict=False)
    T = {k: torch.from_numpy(np.asarray(v, dtype=np.float32)) for k, v in tensors.items()}
    with torch.no_grad():
        for l, layer in enumerate(net.pos_layers):
            p = f"p{l}."
            layer.ln1.weight.copy_(T[p + "ln1_g"]); layer.ln1.bias.copy_(T[p + "ln1_b"])
            layer.qkv.weight.copy_(T[p + "wqkv"]); layer.qkv.bias.copy_(T[p + "bqkv"])
            layer.out.weight.copy_(T[p + "wo"]); layer.out.bias.copy_(T[p + "bo"])
            layer.ln2.weight.copy_(T[p + "ln2_g"]); layer.ln2.bias.copy_(T[p + "ln2_b"])
            layer.ff1.weight.copy_(T[p + "w1"]); layer.ff1.bias.copy_(T[p + "b1"])
            layer.ff2.weight.copy_(T[p + "w2"]); layer.ff2.bias.copy_(T[p + "b2"])
    net.eval()
    return net
