#!/usr/bin/env python
"""Cost of the read store in host memory (hb_attach_read_store) against the uploaded store, on the cfg3 workload of bench.py
(50 000 reads x 20 kb, R10, 40x, W 4096, -b 128, 2 000 targets per launch), both stores in one process, alternating, `--rounds`
rounds:
  - distinct reads and gathered bytes per launch (computed from the alignments of consecutive 2 000-target launches, and the h2d_bytes
    difference between the two contexts over the same runs);
  - k_reads_in's kernel time (torch.profiler, CUDA activities, over replays of one 2 000-target launch) and its bytes/s, next to one
    cudaMemcpyAsync of a pinned buffer of the same size on the same machine (the DMA rate);
  - replay ms per launch in each mode (hb_replay_last_launch; in host mode it includes the gather);
  - end-to-end corrected Mbases/s through hb_submit_alignments from `-t` feature threads (the C++ harness), in each mode, and
    whether the outputs are byte-identical (the harness's checksum of every record).
The card's name and power limit are read in the same run.  Prints one JSON object.

  python tools/measure_host_store.py --reads 50000 --read-len 20000 --targets 8000
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.measure_pos_stage import card  # noqa: E402


def padded_bytes(n):
    """What k_reads_in moves for a read of n bases: its words and qualities, each rounded up to 16 bytes."""
    return (n + 63) // 64 * 16 + (n + 15) // 16 * 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=50000)
    ap.add_argument("--read-len", type=int, default=20000)
    ap.add_argument("--targets", type=int, default=8000, help="targets corrected per round (alignments are built for these only)")
    ap.add_argument("--launch-targets", type=int, default=2000)
    ap.add_argument("--window", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--threads", type=int, default=8, help="feature threads of the harness")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from herro_b200 import Context, api, weights as hbw
    from tools import synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    synth.build()
    t0 = time.time()
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048, targets=(0, args.targets))
    t_gen = time.time() - t0
    import tempfile
    path = os.path.join(tempfile.mkdtemp(prefix="herro_host_store_"), "default.hbw")
    hbw.save_blob(path, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
    W, b, lt = args.window, args.batch_size, args.launch_targets
    lens = np.diff(rs.off).astype(np.int64)

    # ---- what each launch of consecutive targets gathers
    per_launch = []
    for t0_ in range(0, args.targets, lt):
        tg = range(t0_, min(t0_ + lt, args.targets))
        a0, a1 = int(rs.aln_off[tg[0]]), int(rs.aln_off[tg[-1] + 1])
        reads = np.unique(np.concatenate([np.array(list(tg), np.int64), rs.ovl9[a0:a1, 0].astype(np.int64)]))
        per_launch.append(dict(reads=int(len(reads)), gathered_bytes=int(sum(padded_bytes(int(lens[r])) for r in reads)) + 40 * len(reads)))

    # One context switched between the two stores (two contexts of this launch size do not fit one card together): the lanes keep
    # their scratch across the switch, so both modes run on the same buffers.
    ctx = Context(path, 0, W, b, launch_targets=lt)
    packed = api._pack_reads(rs.seqs, rs.quals, rs.off)
    t0 = time.time()
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    t_store = time.time() - t0
    t_upload = []

    def use(mode):
        if mode == "host":
            ctx.attach_read_store(store)
        else:
            t0 = time.time()
            ctx._check(ctx._L.hb_upload_reads(ctx._h, packed.n, packed.wp.ctypes.data, packed.lens.ctypes.data, packed.qp.ctypes.data))
            t_upload.append(round(time.time() - t0, 2))
    harness = api.HostHarness(ctx, rs.ovl9, rs.cigars, rs.cig_off, rs.aln_off, lens.astype(np.uint32))
    modes = ("device", "host")

    # ---- end to end, alternating
    for k in modes:  # warm-up: every lane and pool at its steady-state size
        use(k)
        harness.run(0, args.targets, 1, None)
        harness.run(0, args.targets, args.threads, None)
    e2e = {k: [] for k in modes}
    checks = {k: set() for k in modes}
    h2d = {k: [] for k in modes}
    for _ in range(args.rounds):
        for k in modes:
            use(k)
            ctx.reset_stats()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = harness.run(0, args.targets, args.threads, None)
            s = time.perf_counter() - t0
            st = ctx.stats()
            checks[k].add(r["checksum"])
            h2d[k].append(int(st["h2d_bytes"]))
            e2e[k].append(dict(s=round(s, 3), corrected_bases=r["bases"], mbases_per_s=round(r["bases"] / s / 1e6, 2),
                               launches=int(st["device_launches"]), ms_features=round(st["ms_features"], 1),
                               ms_worker_phase0=round(st["ms_worker_phase"][0], 1)))

    # ---- one launch of the first lt targets from one thread: replay times, and the gather kernel under the profiler
    one = per_launch[0]
    replay = {}
    for k in modes:
        use(k)
        harness.run(0, min(lt, args.targets), 1, None)
        ctx.replay_last_launch(2)
        replay[k] = [round(ctx.replay_last_launch(5) / 5, 3) for _ in range(args.rounds)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.replay_last_launch(5)
        torch.cuda.synchronize()
    e = [x for x in prof.key_averages() if "k_reads_in" in x.key]
    us = ((getattr(e[0], "device_time_total", None) or e[0].cuda_time_total) / max(e[0].count, 1)) if e else None
    gathered = one["gathered_bytes"] - 40 * one["reads"]
    # ---- the DMA rate of the same bytes
    src = torch.empty(gathered, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(gathered, dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dma = []
    for i in range(args.rounds + 1):
        ev[0].record()
        dst.copy_(src, non_blocking=True)
        ev[1].record()
        torch.cuda.synchronize()
        if i:
            dma.append(round(gathered / (ev[0].elapsed_time(ev[1]) * 1e-3) / 1e9, 2))
    del src, dst
    ctx.close()
    store.close()
    print(json.dumps(dict(
        card=card(), torch_device=torch.cuda.get_device_name(0),
        workload=f"synthetic {args.reads} reads x {args.read_len} bp, r10, 40x, W={W}, -b {b}, default model, {args.targets} targets, "
                 f"{lt} per launch, {args.threads} feature threads",
        generate_s=round(t_gen, 1), upload_s=t_upload, store_create_s=round(t_store, 2),
        store_bytes=int(((lens + 31) // 32 * 8 + lens).sum()),
        per_launch_consecutive=per_launch,
        e2e=e2e, outputs_identical=(len(checks["device"]) == 1 and checks["device"] == checks["host"]),
        h2d_extra_per_round_bytes=[h - d for h, d in zip(h2d["host"], h2d["device"])],
        replay_ms_per_launch=replay,
        k_reads_in=None if not us else dict(us=round(us, 1), bytes=gathered, gb_per_s=round(gathered / (us * 1e-6) / 1e9, 2)),
        dma_pinned_h2d_gb_per_s=dma)))


if __name__ == "__main__":
    main()
