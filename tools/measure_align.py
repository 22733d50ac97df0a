#!/usr/bin/env python
"""Cost of hb_align_overlaps on the GPU: the alignment `minimap2 -c` adds to overlap-only PAF, for every overlap of a read set.

A cfg3-shaped read set (2 000 targets x 20 kb, R10, 40x; the generator's overlaps with their CIGARs ignored) in one process:
  - alignments and sum of DP cells ((n + 1) x 2w per overlap) at the default w;
  - the split of that device time into k_align_fill / k_align_trace / k_align_text (torch.profiler, CUDA activities, one call);
  - cells/s of k_align_fill, and its traceback stores (one byte per cell) per second against HBM3's 3.35 TB/s;
  - the call's host wall time (Context.align: hb_align_overlaps + hb_align_fetch), and the device time of the shape (CUDA events
    around every wave's kernels) over repeated calls;
  - `herro align` (hostio.align) on the same set written as FASTQ + overlap-only PAF: each phase's wall time, formatting and
    writing the batches included;
  - the pipeline's wall time correcting the same targets from the generator's alignments (W 4096, -b 128, default model);
  - the CPU oracle's cells/s on all host cores, from a sample of overlaps;
  - the band-edge fraction at w in {32, 64, 128, 256} on R10 and R9 (a smaller set of the same shape).
The card's name and power limit are read in the same run.  Prints one JSON object.

  python tools/measure_align.py --reads 2000 --read-len 20000
"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.measure_pos_stage import card  # noqa: E402

HBM_BYTES_S = 3.35e12  # H100 SXM data sheet


def _oracle_cells(job):
    import align_oracle as ao
    T, Q, w = job
    ao.align_codes(T, Q, w)
    return (len(T) + 1) * 2 * w


def plain_overlaps(rs):
    from herro_b200 import Context
    return Context.make_overlaps(rs.ovl9, np.zeros(1, np.uint8), np.zeros(len(rs.ovl9) + 1, np.uint64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2000)
    ap.add_argument("--read-len", type=int, default=20000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--edge-reads", type=int, default=400)
    ap.add_argument("--oracle-sample", type=int, default=64)
    args = ap.parse_args()

    import torch
    import align_oracle as ao
    from herro_b200 import Context, weights as hbw
    from tools import synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = dict(card=card())
    tmp = tempfile.mkdtemp(prefix="herro_align_")
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048)
    ovl = plain_overlaps(rs)
    ctx = Context(None)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    ctx.align(ovl[:256])  # warm-up: module load, region growth
    walls, devs = [], []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        r = ctx.align(ovl)
        walls.append(time.perf_counter() - t0)
        devs.append(r["shape"]["ms_device"])
    sh = r["shape"]
    out.update(alignments=len(ovl), cells=sh["cells"], band_edge=sh["n_band_edge"], failed=sh["n_failed"], cigar_bytes=sh["cigar_bytes"],
               call_wall_s=walls, ms_device=devs)
    # ---- kernel times
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.align(ovl)
    k = {}
    for e in prof.key_averages():
        for name in ("k_align_fill", "k_align_trace", "k_align_text"):
            if name in e.key:
                k[name] = k.get(name, 0.0) + e.device_time_total / 1e3  # ms
    out["kernel_ms"] = k
    if "k_align_fill" in k:
        fill_s = k["k_align_fill"] / 1e3
        out["fill_cells_per_s"] = sh["cells"] / fill_s
        out["fill_traceback_bytes_per_s"] = sh["cells"] / fill_s
        out["fill_share_of_hbm"] = sh["cells"] / fill_s / HBM_BYTES_S
    ctx.close()
    # ---- the pipeline on the same targets
    path = os.path.join(tmp, "default.hbw")
    hbw.save_blob(path, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
    pctx = Context(path, 0, 4096, 128)
    pctx.upload_reads(rs.seqs, rs.quals, rs.off)
    t0 = time.perf_counter()
    for t in range(rs.n):
        a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
        if a1 > a0:
            pctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
    pctx.flush()
    pctx.drain(skip_failed=True)
    out["pipeline_wall_s"] = time.perf_counter() - t0
    out["pipeline_stats_ms"] = {k2: v for k2, v in pctx.stats().items() if k2 in ("ms_features", "ms_forward", "ms_consensus")}
    pctx.close()
    # ---- the oracle on all host cores
    rng = np.random.default_rng(0)
    pick = rng.choice(len(ovl), min(args.oracle_sample, len(ovl)), replace=False)
    codes = {}
    jobs = []
    for a in pick:
        q, _, qs, qe, st, t, _, ts, te = (int(x) for x in rs.ovl9[a])
        for x in (q, t):
            if x not in codes:
                codes[x] = ao.codes(rs.seq(x))
        jobs.append((codes[t][ts:te], ao.oriented_query(codes[q], qs, qe, st), 128))
    ao.lib()
    t0 = time.perf_counter()
    with ProcessPoolExecutor(os.cpu_count()) as ex:
        cells = sum(ex.map(_oracle_cells, jobs))
    out["oracle_cells_per_s"] = cells / (time.perf_counter() - t0)
    out["host_cores"] = os.cpu_count()
    # ---- band-edge fraction by w
    edge = {}
    for prof_name in ("r10", "r9"):
        es = synth.generate(args.edge_reads, args.read_len, profile=prof_name, seed=2, coverage=40.0, min_ovl=2048)
        eo = plain_overlaps(es)
        ectx = Context(None)
        ectx.upload_reads(es.seqs, es.quals, es.off)
        for w in (32, 64, 128, 256):
            rr = ectx.align(eo, w)
            edge[f"{prof_name}_w{w}"] = rr["shape"]["n_band_edge"] / max(len(eo), 1)
        ectx.close()
    out["band_edge_fraction"] = edge
    # ---- `herro align` end to end: FASTQ + overlap-only PAF -> *.oec.zst batches
    from herro_b200 import hostio
    fq, paf = os.path.join(tmp, "reads.fastq"), os.path.join(tmp, "ovl.paf")
    synth.write_fastq(rs, fq)
    with open(paf, "wb") as f:
        for ln in synth.paf_lines(rs):
            f.write(b"\t".join(ln.rstrip(b"\n").split(b"\t")[:12]) + b"\n")
    out["herro_align"] = hostio.align(fq, paf, os.path.join(tmp, "alns"), min_len=4096)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
