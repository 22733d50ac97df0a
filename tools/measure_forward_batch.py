#!/usr/bin/env python
"""Cost of the model call alone (hb_forward_batch) on the GPU, beside the pipeline's forward on the same windows.

A cfg3-shaped read set (2 000 targets x 20 kb, R10, 40x, W 4096, the default model) runs through the pipeline once with the
debug taps on; each read's reference batches are rebuilt from them (the windows of a 20 kb read form one batch of about five).
Then, in one process:
  - per-read batches from host memory, one call each: the reference's call shape (one small forward per read, SURVEY.md F7);
  - 64-window batches as uint8 CUDA tensors (windows of consecutive reads, padded to the longest of the 64);
  - the repack kernel's time (CUDA events, kernel class `lists`) and its bytes/s against HBM3's 3.35 TB/s;
  - the pipeline's ms_forward per supported position on the same targets.
Call times are host wall time around the synchronous call.  The card's name and power limit are read in the same run.  Prints
one JSON object.

  python tools/measure_forward_batch.py --reads 2000 --read-len 20000
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.measure_pos_stage import card  # noqa: E402

HBM_BYTES_S = 3.35e12  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2000)
    ap.add_argument("--read-len", type=int, default=20000)
    ap.add_argument("--window", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from herro_b200 import Context, weights as hbw
    from tools import synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    synth.build()
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048)
    path = os.path.join(tempfile.mkdtemp(prefix="herro_fwd_batch_"), "default.hbw")
    hbw.save_blob(path, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
    ctx = Context(path, 0, args.window, args.batch_size, launch_targets=1 << 20, keep_debug=True)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    targets = [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]]

    def pipeline():
        for t in targets:
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            ctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
        ctx.flush()
        ctx.drain(skip_failed=True)

    pipeline()  # warm-up
    pipe = []
    for _ in range(args.rounds):
        ctx.reset_stats()
        pipeline()
        s = ctx.stats()
        pipe.append(dict(ms_forward=s["ms_forward"], supported=s["supported"]))

    # the windows of the last launch, and each read's reference batch(es): groups of -b windows with supported positions
    W = args.window
    wins = []  # (L, bases, quals, sup_rows) per window with supported positions, read after read
    per_read = []
    for t in targets:
        nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
        for g0 in range(0, nw, args.batch_size):
            grp = [ctx.debug_window(t, w) for w in range(g0, min(g0 + args.batch_size, nw))]
            grp = [d for d in grp if len(d["sup_rows"])]
            if grp:
                wins += grp
                per_read.append(grp)

    def collate(grp):
        lmax = max(d["L"] for d in grp)
        b = np.full((len(grp), lmax, 31), 11, np.uint8)
        q = np.full((len(grp), lmax, 31), 126, np.uint8)
        for k, d in enumerate(grp):
            b[k, :d["L"]], q[k, :d["L"]] = d["bases"], d["quals"]
        return b, q, [len(d["sup_rows"]) for d in grp], [d["sup_rows"].astype(np.int32) for d in grp]

    host_batches = [collate(g) for g in per_read]
    dev_batches = []
    for i in range(0, len(wins), 64):
        b, q, lens, idx = collate(wins[i:i + 64])
        dev_batches.append((torch.from_numpy(b).cuda(), torch.from_numpy(q).cuda(), lens, idx))
    torch.cuda.synchronize()
    n_pos = sum(sum(x[2]) for x in host_batches)

    def timed(batches):
        t0 = time.perf_counter()
        for x in batches:
            ctx.forward_batch(*x)
        return time.perf_counter() - t0

    timed(host_batches[:50]), timed(dev_batches[:4])  # warm-up: region growth, module loads
    res = dict(per_read_host=[], batch64_cuda=[])
    for _ in range(args.rounds):
        for key, batches in (("per_read_host", host_batches), ("batch64_cuda", dev_batches)):
            s = timed(batches)
            res[key].append(dict(ms_per_call=round(s * 1e3 / len(batches), 4), positions_per_s=round(n_pos / s, 1)))
    # the repack kernel, timed with CUDA events over one pass of the 64-window batches
    ctx.reset_stats()
    ctx.set_kernel_timing(True)
    timed(dev_batches)
    ctx.set_kernel_timing(False)
    st = ctx.stats()
    rep_bytes = sum(2 * x[0].shape[0] * x[0].shape[1] * (31 + 32) for x in dev_batches)
    rep_ms = st["ms_kernel"]["lists"]
    out = dict(card=card(), torch_device=torch.cuda.get_device_name(0),
               workload=f"synthetic {args.reads} reads x {args.read_len} bp, r10, 40x, W={W}, -b {args.batch_size}, default model",
               windows=len(wins), positions=n_pos, per_read_calls=len(host_batches), batch64_calls=len(dev_batches),
               per_read_windows_mean=round(len(wins) / len(host_batches), 2), results=res,
               repack=dict(calls=int(st["n_kernel"]["lists"]), ms_total=round(rep_ms, 4), bytes=rep_bytes,
                           bytes_per_s=round(rep_bytes / (rep_ms * 1e-3), 1) if rep_ms else None,
                           share_of_hbm=round(rep_bytes / (rep_ms * 1e-3) / HBM_BYTES_S, 4) if rep_ms else None),
               batch64_ms_forward_per_position_us=round(st["ms_forward"] * 1e3 / max(st["supported"], 1), 5),
               pipeline=[dict(p, ms_forward_per_position_us=round(p["ms_forward"] * 1e3 / max(p["supported"], 1), 5)) for p in pipe])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
