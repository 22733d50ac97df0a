#!/usr/bin/env python
"""Cost of hb_find_overlaps on the GPU: all-vs-all overlaps of a read set, every read a target in one call.

On the measure_align set (2 000 reads x 20 kb, R10, 40x; the generator's true overlaps with min_ovl=1):
  - index entries, query minimizers, anchors, chained groups, overlaps;
  - per-kernel device time (torch.profiler, CUDA activities, one call) and the call's device time (CUDA events, the shape) and
    host wall time over repeated calls;
  - each kernel against the bound DESIGN.md §13 gives it: the sketch's packed words read (0.25 byte per base, two passes) over
    HBM3's 3.35 TB/s; anchors chained per second;
  - recall (truth pairs sharing >= 5 000 target bases that are found) and precision (records that are truth pairs of the same
    strand) against the generator's truth.
--cfg3 also runs one call over 50 000 x 20 kb reads with all 50 000 as targets (wall and device time).  The card's name, power
limit and max SM clock are read in the same run.  Prints one JSON object.

  python tools/measure_overlap.py [--reads 2000 --read-len 20000] [--cfg3]
"""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.measure_pos_stage import card  # noqa: E402

HBM_BYTES_S = 3.35e12  # H100 SXM data sheet


def context(rs):
    from herro_b200 import Context
    ctx = Context(None)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    return ctx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=2000)
    ap.add_argument("--read-len", type=int, default=20000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cfg3", action="store_true")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from tools import synth
    out = dict(card=card())
    rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=1)
    bases = int(rs.off[-1])
    ctx = context(rs)
    targets = np.arange(rs.n, dtype=np.uint32)
    got = ctx.find_overlaps(targets)  # warm-up: regions grown, modules loaded
    walls, devs = [], []
    for _ in range(args.rounds):
        t = time.perf_counter()
        got = ctx.find_overlaps(targets)
        walls.append(time.perf_counter() - t)
        devs.append(got["shape"]["ms_device"])
    sh = got["shape"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.find_overlaps(targets)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            m = re.search(r"k_ovl_[a-z]+", e.key)
            name = m.group(0) if m else ("cub" if "cub" in e.key else e.key[:40])
            kern[name] = kern.get(name, 0.0) + e.device_time_total / 1e3
    ms_sketch = kern.get("k_ovl_sketch", float("nan"))
    ms_chain = kern.get("k_ovl_chain", float("nan"))
    sketch_bytes = 2 * 2 * bases * 0.25  # targets and queries, count and write pass
    # truth
    truth = {}
    for q, _, _, _, st, t, _, ts, te in rs.ovl9.astype(np.int64):
        truth[(int(t), int(q))] = (int(st), int(ts), int(te))
    o = got["overlaps"]
    pairs = list(zip(o["tid"].tolist(), o["qid"].tolist(), o["strand"].tolist()))
    good = sum(1 for t, q, s in pairs if (t, q) in truth and truth[(t, q)][0] == s)
    found = {(t, q) for t, q, _ in pairs}
    big = [p for p, v in truth.items() if v[2] - v[1] >= 5000]
    out.update(set=dict(reads=rs.n, bases=bases, profile="r10", coverage=40), shape={k: v for k, v in sh.items() if k != "ticket"},
               wall_s=walls, ms_device=devs, kernel_ms=kern,
               sketch_GBps=sketch_bytes / (ms_sketch / 1e3) / 1e9, sketch_share_of_hbm=sketch_bytes / (ms_sketch / 1e3) / HBM_BYTES_S,
               anchors_chained_per_s=sh["anchors"] / (ms_chain / 1e3),
               precision=good / max(len(pairs), 1), recall_ge5000=sum(p in found for p in big) / max(len(big), 1),
               truth_pairs_ge5000=len(big))
    ctx.close()
    if args.cfg3:
        c3 = synth.generate(50_000, 20_000, profile="r10", seed=3, coverage=40.0, min_ovl=2048)
        ctx = context(c3)
        t = time.perf_counter()
        g3 = ctx.find_overlaps(np.arange(c3.n, dtype=np.uint32))
        out["cfg3"] = dict(wall_s=time.perf_counter() - t, shape={k: v for k, v in g3["shape"].items() if k != "ticket"})
        ctx.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
