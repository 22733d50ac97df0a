"""`python -m herro_b200.cli {inference,features} ...` — the reference's two sub-commands (src/main.rs:10-112, README.md:75-96)
as a thin argument parser over the native host pipeline (herro_b200/host/io.cpp -> the C ABI of libherro_b200):

    python -m herro_b200.cli inference --read-alns <dir> -t 4 -d 0 -m model.hbw -b 64 reads.fastq out.fasta
    python -m herro_b200.cli inference --torch --read-alns <dir> -d 0 -m model.pt -b 64 reads.fastq out.fasta
                                       (any TorchScript graph with the reference's forward signature, run by torch.jit)
    python -m herro_b200.cli features  --read-alns <dir> reads.fastq out_dir
    python -m herro_b200.cli predict   -m model.hbw -b 64 [-d 0] features_dir out_dir   (the model alone, on `features` output)
    python -m herro_b200.cli consensus -m model.hbw [-d 0] features_dir logits_dir reads.fastq out.fasta
                                       (consensus alone, on `features` and `predict` output)

Nothing is computed here: FASTQ parsing / 2-bit packing, `*.oec.zst` decoding and PAF parsing, the feature / consumer threads
and the FASTA writer are C++ threads (hbh_inference); `features` and `inference --torch` call hb_features_batch.  Each command keeps
the reads in pinned host memory instead of device memory when they take more than half of the smallest selected GPU's memory
(hostio.host_store_above).  In deployment this
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


def write_features(F, k, out_dir, names):
    """The feature files of target k of a Features result (Context.features_batch) under out_dir/<read name>/."""
    d = os.path.join(out_dir, os.fsdecode(names[F.rids[k]]))
    for wid in range(int(F.n_windows[k])):
        w = F.window(int(F.win_off[k]) + wid)
        hostio.write_feature_window(d, wid, w["bases"], w["quals"], w["supported"], [names[int(q)] for q in w["ids"]])


def features(args):
    """`herro features` (src/lib.rs:50-111): the per-window feature files of every target, from hb_features_batch on a context
    without weights, `--targets-per-launch` targets per call."""
    R = hostio.Reads(args.reads, min_len=args.window_size)
    A = hostio.Alignments(args.read_alns, R)
    ctx = api.Context(None, 0, args.window_size, 64)
    R.load_into(ctx, hostio.device_bytes([0]))
    n = 0
    step = max(1, args.targets_per_launch)
    for k0 in range(0, A.n_targets, step):
        F = ctx.features_batch([A.target(k) for k in range(k0, min(k0 + step, A.n_targets))])
        for k in range(len(F.rids)):
            if F.status[k]:  # the reference would have panicked on this read's alignments
                print(f"skipped read {os.fsdecode(R.ids[F.rids[k]])}: error {int(F.status[k])}", file=sys.stderr)
                continue
            write_features(F, k, args.output, R.ids)
            n += 1
    ctx.close()
    print(f"Wrote the feature files of {n} reads under {args.output}.", file=sys.stderr)


def quals_normalised(quals):
    """inference()'s quality transform (src/inference.rs:19-21,152-153): fp32, multiply then subtract."""
    import torch
    return (2.0 / 93.0) * quals.to(torch.float32) - (2.0 * 33.0 / 93.0 + 1.0)


def inference_torch(args):
    """`inference --torch`: the features stage and consensus on the device through the library (a context without weights), the
    model call by torch.jit on a TorchScript archive the library does not parse, as src/inference.rs:147-175 calls it: int tokens,
    normalised qualities, lens and the indices list.  One device; `--targets-per-launch` targets per features call."""
    import numpy as np
    import torch
    dev = int(str(args.devices).split(",")[0])
    if "," in str(args.devices):
        raise SystemExit("--torch runs on one device (-d)")
    R = hostio.Reads(args.reads, min_len=args.window_size)
    A = hostio.Alignments(args.read_alns, R)
    ctx = api.Context(None, dev, args.window_size, args.batch_size)
    R.load_into(ctx, hostio.device_bytes([dev]))
    cuda = torch.device("cuda", dev)
    module = torch.jit.load(args.model, map_location=cuda).eval()
    out = hostio.FastaWriter(args.output)
    step = max(1, args.targets_per_launch)
    failed = 0
    with torch.no_grad(), torch.cuda.device(cuda):
        for k0 in range(0, A.n_targets, step):
            F = ctx.features_batch([A.target(k) for k in range(k0, min(k0 + step, A.n_targets))], device=True, batches=True)
            logits = []
            for _, bases, quals, lens, indices in F.batches():
                idx = [torch.from_numpy(np.ascontiguousarray(i)).to(cuda) for i in indices]
                _, bl = module(bases.to(torch.int32), quals_normalised(quals), torch.from_numpy(lens).to(cuda), idx)
                logits.append(bl.float())
            for k, segs in enumerate(ctx.consensus_batch(*F.consensus_args(logits))):
                rid = F.rids[k]
                if F.status[k]:
                    failed += 1
                elif segs:
                    out.write(R.ids[rid], R.descriptions[rid], segs)
    records, bases = out.close()
    ctx.close()
    print(f"Processed {A.n_targets} reads, wrote {records} records ({bases} bases)" + (f"; skipped {failed} reads" if failed else ""),
          file=sys.stderr)
    return dict(targets=A.n_targets, records=records, corrected_bases=bases, failed_targets=failed)


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
    inf.add_argument("--torch", action="store_true",
                     help="-m is a TorchScript archive that torch.jit runs (any graph with the reference's forward signature); features "
                          "and consensus run in the library")
    inf.add_argument("--targets-per-launch", type=int, default=256, help="with --torch: targets per features call")
    inf.add_argument("reads")
    inf.add_argument("output")
    ft = sub.add_parser("features")
    ft.add_argument("--read-alns", required=True)
    ft.add_argument("-w", dest="window_size", type=int, default=4096)
    ft.add_argument("-m", dest="model", default=None, help="accepted and ignored: the feature files do not depend on the model")
    ft.add_argument("--targets-per-launch", type=int, default=256, help="targets per features call")
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
        if args.torch:
            if args.cluster:
                raise SystemExit("-c is not supported with --torch")
            return inference_torch(args)
        return inference(args)
    if args.cmd == "predict":
        return predict(args)
    if args.cmd == "consensus":
        return consensus(args)
    return features(args)


if __name__ == "__main__":
    main()
