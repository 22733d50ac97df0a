#!/usr/bin/env python
"""Emit a TorchScript archive of the forward (oracle/forward_ref.HerroNet, or tools/pos_forward_ref.PosHerroNet when the
blob has a position-axis encoder stage) from an HB200W1 blob:
the unmodified reference binary can load it with CModule::load_on_device (src/inference.rs:185)
and call it with its 4 inputs (src/inference.rs:155-163).  Test/diagnostic tool."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from herro_b200 import weights as hbw
    from oracle import forward_ref
    from tools import pos_forward_ref
    cfg, T = hbw.load_blob(sys.argv[1])
    net = (pos_forward_ref if cfg.pos_layers else forward_ref).from_weights(cfg, T)
    torch.jit.script(net).save(sys.argv[2])
    print("wrote", sys.argv[2])


if __name__ == "__main__":
    main()
