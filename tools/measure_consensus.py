#!/usr/bin/env python
"""Cost of consensus alone (hb_consensus_batch) on the GPU, beside the pipeline's consensus on the same windows and the oracle's
CPU consensus().

A cfg3-shaped read set (2 000 targets x 20 kb, R10, 40x, W 4096, -b 128, the default model) runs through the pipeline with the
debug taps on; every read's ConsensusWindows (tokens, n_alns, supported positions, base logits) are rebuilt from them.  Then, in
one process:
  - the pipeline's ms_consensus per launch (CUDA events around its three consensus kernels);
  - hb_consensus_batch from host memory, one call per read (the reference's call shape: consensus_worker runs once per read)
    and one call over all reads, as host wall time around the synchronous call;
  - k_cons_in's kernel time (torch.profiler, CUDA activities, in a pass of its own) and its bytes/s over its algorithmic bytes
    (31 read + 1 written per row, 8 per key and 20 per logit row, of the windows with n_alns >= 2) against HBM3's 3.35 TB/s;
  - the oracle's consensus() (oracle/herro_oracle.cpp through tests/consensus_oracle.py, one CPU thread) on the same windows.
The card's name and power limit are read in the same run.  Prints one JSON object.

  python tools/measure_consensus.py --reads 2000 --read-len 20000
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
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from herro_b200 import Context, hostio, weights as hbw
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import consensus_oracle
    from tools import synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    synth.build()
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048)
    path = os.path.join(tempfile.mkdtemp(prefix="herro_consensus_"), "default.hbw")
    hbw.save_blob(path, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
    ctx = Context(path, 0, args.window, args.batch_size, launch_targets=1 << 20, keep_debug=True)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    targets = [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]]

    def pipeline():
        for t in targets:
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            ctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
        ctx.flush()
        return {r.rid: r.segments for r in ctx.drain(skip_failed=True)}

    pipeline()  # warm-up
    pipe = []
    for _ in range(args.rounds):
        ctx.reset_stats()
        segs = pipeline()
        s = ctx.stats()
        pipe.append(dict(launches=int(s["device_launches"]), ms_consensus=round(s["ms_consensus"], 4),
                         ms_consensus_per_launch=round(s["ms_consensus"] / max(s["device_launches"], 1), 4)))

    W = args.window
    reads = []
    for t in targets:
        nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
        wins = []
        for w in range(nw):
            d = ctx.debug_window(t, w)
            wins.append(hostio.ConsensusWindow(w, d["n_alns"], d["bases"], d["supported"].reshape(-1, 2), d["bases_logits"].reshape(-1, 5)))
        reads.append(wins)
    per_read = [hostio.consensus_args([r]) for r in reads]
    all_reads = hostio.consensus_args(reads)
    want = [segs.get(t, []) for t in targets]
    assert ctx.consensus_batch(*all_reads) == want, "hb_consensus_batch differs from the pipeline"
    used = [w for r in reads for w in r if w.n_alns >= 2]
    n_rows = sum(w.bases.shape[0] for w in used)
    n_sup = sum(len(w.supported) for w in used)
    algo_bytes = 32 * n_rows + 28 * n_sup

    def timed(calls):
        t0 = time.perf_counter()
        for x in calls:
            ctx.consensus_batch(*x)
        return time.perf_counter() - t0

    timed(per_read[:50]), timed([all_reads])  # warm-up: region growth, module loads
    res = dict(per_read_host=[], all_reads_host=[])
    for _ in range(args.rounds):
        s = timed(per_read)
        res["per_read_host"].append(dict(ms_per_call=round(s * 1e3 / len(per_read), 4), ms_total=round(s * 1e3, 2)))
        s = timed([all_reads])
        res["all_reads_host"].append(dict(ms_per_call=round(s * 1e3, 3)))
    ctx.reset_stats()
    ctx.set_kernel_timing(True)
    timed([all_reads])
    ctx.set_kernel_timing(False)
    st = ctx.stats()
    events_ms = dict(ms_consensus=round(st["ms_consensus"], 4), consensus_class=round(st["ms_kernel"]["consensus"], 4),
                     scan_class=round(st["ms_kernel"]["scan"], 4))
    # k_cons_in alone, by name
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ctx.consensus_batch(*all_reads)
        torch.cuda.synchronize()
    kin = [e for e in prof.key_averages() if "k_cons_in" in e.key]
    kin_us = (getattr(kin[0], "device_time_total", None) or kin[0].cuda_time_total) / max(kin[0].count, 1) if kin else None
    # the oracle's CPU consensus() on the same windows
    ora = [[(w.bases, w.n_alns, w.supported, w.bases_logits) for w in r] for r in reads]
    t0 = time.perf_counter()
    got_ora = consensus_oracle.consensus_windows(ora)
    ora_s = time.perf_counter() - t0
    assert got_ora == want, "the oracle differs from the pipeline"
    out = dict(card=card(), torch_device=torch.cuda.get_device_name(0),
               workload=f"synthetic {args.reads} reads x {args.read_len} bp, r10, 40x, W={W}, -b {args.batch_size}, default model",
               reads=len(reads), windows=sum(len(r) for r in reads), windows_read=len(used), rows_read=n_rows, supported_read=n_sup,
               corrected_bases=sum(len(x) for s in want for x in s), pipeline=pipe, results=res, all_reads_events=events_ms,
               k_cons_in=dict(us_per_call=round(kin_us, 2) if kin_us else None, algo_bytes=algo_bytes,
                              bytes_per_s=round(algo_bytes / (kin_us * 1e-6), 1) if kin_us else None,
                              share_of_hbm=round(algo_bytes / (kin_us * 1e-6) / HBM_BYTES_S, 4) if kin_us else None),
               oracle_cpu=dict(s_total=round(ora_s, 3), ms_per_read=round(ora_s * 1e3 / len(reads), 4),
                               note="one CPU thread, ctypes wrapper included"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
