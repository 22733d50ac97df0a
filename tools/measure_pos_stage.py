#!/usr/bin/env python
"""Cost of the position-axis encoder stage on the GPU: the same read set run with the default model and with a model that
adds `pos_layers` encoder layers across each window's supported positions, alternating the two in one process.

Per model and round it reports the device-resident replay rate of the last launch (Mbases/s of corrected bases) and, from a
separate launch with per-kernel CUDA-event timing, the milliseconds per kernel class.  The card's name and power limit are
read in the same call.  Prints one JSON object.

  python tools/measure_pos_stage.py --reads 2000 --read-len 15000 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (x.strip() for x in out.split(","))))
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2000)
    ap.add_argument("--read-len", type=int, default=15000)
    ap.add_argument("--window", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--replays", type=int, default=5)
    ap.add_argument("--pos-layers", type=int, default=2)
    ap.add_argument("--pos-heads", type=int, default=8)
    ap.add_argument("--pos-ffn", type=int, default=1024)
    args = ap.parse_args()

    from herro_b200 import Context, weights as hbw
    from tools import synth
    synth.build()
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=1024)
    tmp = tempfile.mkdtemp(prefix="herro_pos_stage_")
    models = {}
    for name, cfg in (("default", hbw.NetConfig()),
                      ("pos", hbw.NetConfig(pos_layers=args.pos_layers, pos_heads=args.pos_heads, pos_ffn=args.pos_ffn))):
        p = os.path.join(tmp, f"{name}.hbw")
        hbw.save_blob(p, cfg, hbw.random_weights(cfg, seed=7))
        models[name] = p
    ctxs = {}
    for name, p in models.items():
        ctx = Context(p, 0, args.window, args.batch_size)
        ctx.upload_reads(rs.seqs, rs.quals, rs.off)
        ctxs[name] = ctx

    def launch(ctx):
        for t in range(rs.n):
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            if a1 > a0:
                ctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
        ctx.flush()
        ctx.drain(skip_failed=True)

    for ctx in ctxs.values():  # warm-up: module loads, region growth
        launch(ctx)
    res = {name: dict(replay_mbases_s=[], ms_kernel=[]) for name in ctxs}
    info = card()
    for _ in range(args.rounds):
        for name, ctx in ctxs.items():
            ctx.reset_stats()
            ctx.set_kernel_timing(True)
            launch(ctx)
            ctx.set_kernel_timing(False)
            st = ctx.stats()
            res[name]["ms_kernel"].append({k: round(v, 3) for k, v in st["ms_kernel"].items() if v > 0})
            res[name]["supported"] = st["supported"]
            res[name]["class_flops"] = {k: v for k, v in st["class_flops"].items() if v}
            launch(ctx)  # the replayed launch ran without event timing
            ms = ctx.replay_last_launch(args.replays)
            bases = ctx.stats()["last_launch_bases"]
            res[name]["replay_mbases_s"].append(round(bases * args.replays / ms / 1e3, 2))
    out = dict(card=info, workload=f"synthetic {args.reads} reads x {args.read_len} bp, r10, 40x, W={args.window}, "
                                   f"-b {args.batch_size}", pos_model=dict(pos_layers=args.pos_layers,
                                                                           pos_heads=args.pos_heads, pos_ffn=args.pos_ffn),
               results=res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
