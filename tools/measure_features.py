#!/usr/bin/env python
"""Cost of the features stage alone (hb_features_batch + hb_features_fetch) on the GPU, beside the pipeline's features stage on the
same targets, and `inference --torch` beside the fused pipeline.

A cfg3-shaped read set (2 000 targets x 20 kb, R10, 40x, W 4096, -b 128, the default model) in one process:
  - the pipeline's ms_features per launch (CUDA events around windowing + pileup) against hb_features_batch's event time for all
    targets in one call (the same kernels, one launch);
  - k_rows_out / k_lists_out kernel times (torch.profiler, CUDA activities) and their bytes/s over the algorithmic bytes (per ragged
    or collated row 2 x 32 read + 2 x 31 written; per supported entry 8 read + 12 written; per id 16) against HBM3's 3.35 TB/s;
  - the host wall time of Context.features_batch with device outputs and with host outputs (batches included);
  - corrected bases/s of `cli inference --torch` with the stand-in archive (tools/make_torchscript.py: the default model scripted)
    next to the fused pipeline (`cli inference`), both from FASTQ + *.oec.zst on one device.
The card's name and power limit are read in the same run.  Prints one JSON object.

  python tools/measure_features.py --reads 2000 --read-len 20000
"""
import argparse
import ctypes as C
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
    ap.add_argument("--skip-cli", action="store_true", help="leave out the inference --torch / inference comparison")
    args = ap.parse_args()

    import torch
    from herro_b200 import Context, api, cli, weights as hbw
    from tools import synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    synth.build()
    tmp = tempfile.mkdtemp(prefix="herro_features_")
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048)
    path = os.path.join(tmp, "default.hbw")
    hbw.save_blob(path, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
    W, b = args.window, args.batch_size
    targets = [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]]
    ovls = {t: Context.make_overlaps(rs.ovl9[int(rs.aln_off[t]):int(rs.aln_off[t + 1])], rs.cigars,
                                     rs.cig_off[int(rs.aln_off[t]):int(rs.aln_off[t + 1]) + 1]) for t in targets}
    tl = [(t, ovls[t]) for t in targets]

    # ---- the pipeline's features stage per launch
    ctx = Context(path, 0, W, b)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)

    def pipeline():
        for t in targets:
            ctx.submit_alignments(t, ovls[t])
        ctx.flush()
        ctx.drain(skip_failed=True)

    pipeline()
    pipe = []
    for _ in range(args.rounds):
        ctx.reset_stats()
        pipeline()
        s = ctx.stats()
        pipe.append(dict(launches=int(s["device_launches"]), ms_features=round(s["ms_features"], 3),
                         ms_features_per_launch=round(s["ms_features"] / max(s["device_launches"], 1), 3)))

    # ---- hb_features_batch alone (event time of its front half), and the wall time of whole calls
    L = api.load_library()
    rids = np.array(targets, np.uint32)
    n_ovl = np.array([len(ovls[t]) for t in targets], np.uint32)
    flat = np.zeros(int(n_ovl.sum()), api.OVERLAP_DTYPE)  # np.concatenate would pack the padded record layout
    o0 = 0
    for t in targets:
        flat[o0:o0 + len(ovls[t])] = ovls[t]
        o0 += len(ovls[t])
    F = ctx.features_batch(tl, batches=True)  # warm-up and sizes
    front = []
    for _ in range(args.rounds):
        ctx.reset_stats()
        sh = api.HbFeaturesShape()
        t0 = time.perf_counter()
        ctx._check(L.hb_features_batch(ctx._h, len(rids), rids.ctypes.data, n_ovl.ctypes.data, flat.ctypes.data, C.byref(sh)))
        wall = time.perf_counter() - t0
        front.append(dict(ms_features_events=round(ctx.stats()["ms_features"], 3), ms_wall=round(wall * 1e3, 2)))
    walls = dict(host=[], device=[])
    ctx.features_batch(tl, device=True, batches=True)
    for _ in range(args.rounds):
        for k, dev in (("host", False), ("device", True)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.features_batch(tl, device=dev, batches=True)
            walls[k].append(round((time.perf_counter() - t0) * 1e3, 2))

    # ---- the output kernels by name
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            ctx.features_batch(tl, device=True, batches=True)
        torch.cuda.synchronize()

    def us(name):
        e = [x for x in prof.key_averages() if name in x.key]
        if not e:
            return None, 0
        return (getattr(e[0], "device_time_total", None) or e[0].cuda_time_total) / max(e[0].count, 1), e[0].count
    rows_us, rows_n = us("k_rows_out")
    lists_us, _ = us("k_lists_out")
    N, NB, S, NI = int(F.rows.sum()), int(sum(int(x) * int(y) for x, y in zip(F.batch_B, F.batch_Lmax))), int(F.n_sup.sum()), int(F.n_ids.sum())
    rows_bytes = 126 * (N + NB) / 2  # k_rows_out runs twice per call (ragged, collated): the mean bytes per launch
    lists_bytes = 20 * S + 16 * NI

    def bw(bytes_, t):
        return None if not t else dict(us_per_call=round(t, 2), algo_bytes=int(bytes_), bytes_per_s=round(bytes_ / (t * 1e-6), 1),
                                       share_of_hbm=round(bytes_ / (t * 1e-6) / HBM_BYTES_S, 4))
    ctx.close()

    # ---- inference --torch (stand-in archive) next to the fused pipeline
    cli_res = None
    if not args.skip_cli:
        import subprocess
        fq, alns = os.path.join(tmp, "reads.fastq"), os.path.join(tmp, "alns")
        synth.write_fastq(rs, fq)
        synth.write_oec_batches(rs, alns)
        pt = os.path.join(tmp, "default.pt")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "make_torchscript.py"), path, pt], stdout=subprocess.DEVNULL)
        cli_res = {}
        for name, argv in (("fused", ["inference", "-m", path]), ("torch", ["inference", "--torch", "-m", pt, "--targets-per-launch", "512"])):
            runs = []
            for _ in range(2):
                out = os.path.join(tmp, f"{name}.fasta")
                t0 = time.perf_counter()
                r = cli.main(argv + ["--read-alns", alns, "-b", str(b), "-w", str(W), fq, out])
                s = time.perf_counter() - t0
                runs.append(dict(s=round(s, 2), corrected_bases=r["corrected_bases"], bases_per_s=round(r["corrected_bases"] / s, 1)))
            cli_res[name] = runs
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0),
                          workload=f"synthetic {args.reads} reads x {args.read_len} bp, r10, 40x, W={W}, -b {b}, default model",
                          targets=len(targets), windows=len(F.rows), rows=N, batch_rows=NB, supported=S, ids=NI, batches=len(F.batch_B),
                          pipeline=pipe, features_batch_front=front, features_batch_wall_ms=walls,
                          k_rows_out=bw(rows_bytes, rows_us), k_rows_out_launches=rows_n, k_lists_out=bw(lists_bytes, lists_us),
                          cli=cli_res)))


if __name__ == "__main__":
    main()
