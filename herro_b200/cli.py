"""`python -m herro_b200.cli {inference,features} ...` — the reference's two sub-commands (src/main.rs:10-112, README.md:75-96)
as a thin argument parser over the native host pipeline (herro_b200/host/io.cpp -> the C ABI of libherro_b200):

    python -m herro_b200.cli inference --read-alns <dir> -t 4 -d 0 -m model.hbw -b 64 reads.fastq out.fasta
    python -m herro_b200.cli features  --read-alns <dir> -m model.hbw reads.fastq out_dir
    python -m herro_b200.cli predict   -m model.hbw -b 64 [-d 0] features_dir out_dir   (the model alone, on `features` output)
    python -m herro_b200.cli consensus -m model.hbw [-d 0] features_dir logits_dir reads.fastq out.fasta
                                       (consensus alone, on `features` and `predict` output)

Nothing is computed here: FASTQ parsing / 2-bit packing, `*.oec.zst` decoding and PAF parsing, the feature / consumer threads
and the FASTA writer are C++ threads (hbh_inference); `features` drives hb_dump_features launch by launch.  In deployment this
role is played by the unchanged Rust binary (INTEGRATION.md); the flags keep the reference's meaning: reads shorter than `-w`
are not loaded (src/haec_io.rs:48), unknown names / self overlaps / repeated (query,target) pairs are skipped
(src/overlaps.rs:137-185), `-c` cluster files restrict targets to core reads (:154-159).
"""
from __future__ import annotations

import argparse
import os
import sys

from . import api, hostio


def read_cluster(path):
    """src/lib.rs:208-239: `0\\t<id>` core, `1\\t<id>` neighbour."""
    core, neigh = [], []
    for line in open(path, "rb"):
        f = line.rstrip(b"\n").split(b"\t")
        if f[0] == b"0":
            core.append(f[1])
        elif f[0] == b"1":
            neigh.append(f[1])
        else:
            raise SystemExit("Invalid cluster file")
    return core, neigh


def inference(args):
    core = neigh = None
    if args.cluster:
        core, neigh = read_cluster(args.cluster)
    devices = [int(d) for d in str(args.devices).split(",")]
    r = hostio.inference(args.reads, args.read_alns, args.model, args.output, args.window_size, args.batch_size,
                         args.feat_gen_threads, devices, core, neigh)
    print(f"Processed {r['targets']} reads, wrote {r['records']} records ({r['corrected_bases']} bases); "
          f"fastq {r['fastq_load_s'] + r['pack_s']:.2f}s, alignments {r['alignment_ingest_s']:.2f}s, upload {r['read_store_upload_s']:.2f}s, "
          f"correction {r['correction_s']:.2f}s" + (f"; skipped {r['failed_targets']} reads" if r["failed_targets"] else ""), file=sys.stderr)
    return r


def features(args):
    """`herro features` (src/lib.rs:50-111): the per-window feature files of every target, from the device path."""
    R = hostio.Reads(args.reads, min_len=args.window_size)
    A = hostio.Alignments(args.read_alns, R)
    ctx = api.Context(args.model, 0, args.window_size, 64, launch_targets=1 << 20, keep_debug=True)
    R.upload(ctx)
    n = 0
    step = max(1, args.targets_per_launch)
    for k0 in range(0, A.n_targets, step):  # the debug taps keep one launch: dump launch by launch
        group = range(k0, min(k0 + step, A.n_targets))
        for k in group:
            rid, ov = A.target(k)
            ctx.submit_alignments(rid, ov)
        ctx.flush()
        ctx.drain(skip_failed=True)
        for k in group:
            ctx.dump_features(int(A.target_rids[k]), args.output, R.ids)
            n += 1
    print(f"Wrote the feature files of {n} reads under {args.output}.", file=sys.stderr)


def predict(args):
    """The model alone on `herro features` output: every read's reference batches (hostio.read_feature_batches) through
    hb_forward_batch; per window with supported positions, <out>/<read>/<wid>.info_logits.npy (f32 [n]) and
    <wid>.bases_logits.npy (f32 [n, 5])."""
    import numpy as np
    ctx = api.Context(args.model, args.device, batch_size=args.batch_size)
    n_win = n_pos = 0
    for read_dir in hostio.feature_reads(args.features):
        for fb in hostio.read_feature_batches(read_dir, args.batch_size):
            info, bl = ctx.forward_batch(fb.bases, fb.quals, fb.lens, fb.indices)
            out = os.path.join(args.output, fb.read)
            os.makedirs(out, exist_ok=True)
            for wid, i, b in zip(fb.wids, info, bl):
                np.save(os.path.join(out, f"{wid}.info_logits.npy"), i)
                np.save(os.path.join(out, f"{wid}.bases_logits.npy"), b)
                n_win += 1
                n_pos += len(i)
    ctx.close()
    print(f"Wrote the logits of {n_pos} supported positions in {n_win} windows under {args.output}.", file=sys.stderr)


def consensus(args):
    """consensus() alone on `features` and `predict` output: every read's ConsensusWindows (hostio.read_consensus_windows) through
    hb_consensus_batch, many reads per call, written as correction_writer writes them.  The FASTQ gives only ids and descriptions."""
    R = hostio.Reads(args.reads, min_len=0)
    desc = dict(zip(R.ids, R.descriptions))
    R.close()
    ctx = api.Context(args.model, args.device)
    out = hostio.FastaWriter(args.output)
    pending, rows = [], 0

    def run():
        names = [n for n, _ in pending]
        for name, segs in zip(names, ctx.consensus_batch(*hostio.consensus_args([w for _, w in pending]))):
            if segs:
                out.write(name, desc.get(name), segs)
        pending.clear()

    for read_dir in hostio.feature_reads(args.features):
        name = os.path.basename(read_dir)
        wins = hostio.read_consensus_windows(read_dir, os.path.join(args.logits, name))
        if name.encode() not in desc:
            raise SystemExit(f"read {name} of {args.features} is not in {args.reads}")
        pending.append((name.encode(), wins))
        rows += sum(w.bases.shape[0] for w in wins)
        if rows >= args.rows_per_call:
            run()
            rows = 0
    if pending:
        run()
    records, bases = out.close()
    ctx.close()
    print(f"Wrote {records} records ({bases} bases) to {args.output}.", file=sys.stderr)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="herro_b200")
    sub = ap.add_subparsers(dest="cmd", required=True)
    inf = sub.add_parser("inference")
    inf.add_argument("--read-alns", required=True, help="directory with *.oec.zst alignment batches")
    inf.add_argument("-w", dest="window_size", type=int, default=4096)
    inf.add_argument("-t", dest="feat_gen_threads", type=int, default=1)
    inf.add_argument("-m", dest="model", required=True)
    inf.add_argument("-d", dest="devices", default="0")
    inf.add_argument("-b", dest="batch_size", type=int, required=True)
    inf.add_argument("-c", dest="cluster", default="")
    inf.add_argument("reads")
    inf.add_argument("output")
    ft = sub.add_parser("features")
    ft.add_argument("--read-alns", required=True)
    ft.add_argument("-w", dest="window_size", type=int, default=4096)
    ft.add_argument("-m", dest="model", required=True, help="weights (a context needs them; the feature files do not depend on them)")
    ft.add_argument("--targets-per-launch", type=int, default=256)
    ft.add_argument("reads")
    ft.add_argument("output")
    pr = sub.add_parser("predict", help="the model alone on a `features` output directory")
    pr.add_argument("-m", dest="model", required=True)
    pr.add_argument("-b", dest="batch_size", type=int, required=True, help="windows per model batch, as `-b` of the features run")
    pr.add_argument("-d", dest="device", type=int, default=0)
    pr.add_argument("features")
    pr.add_argument("output")
    cs = sub.add_parser("consensus", help="consensus alone on `features` and `predict` output directories")
    cs.add_argument("-m", dest="model", required=True, help="weights (a context needs them; consensus does not use them)")
    cs.add_argument("-d", dest="device", type=int, default=0)
    cs.add_argument("--rows-per-call", type=int, default=1 << 22, help="window rows gathered before each library call")
    cs.add_argument("features")
    cs.add_argument("logits")
    cs.add_argument("reads")
    cs.add_argument("output")
    args = ap.parse_args(argv)
    if args.cmd == "inference":
        return inference(args)
    if args.cmd == "predict":
        return predict(args)
    if args.cmd == "consensus":
        return consensus(args)
    return features(args)


if __name__ == "__main__":
    main()
