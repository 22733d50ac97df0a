#!/usr/bin/env python
"""End-to-end `inference` from files with the streaming alignment reader against a build of the parent commit (which parses every
file before correcting), on the cfg3 read set of bench.py (50 000 reads x 20 kb, R10, 40x, W 4096, -b 128) written as FASTQ and
`--files` *.oec.zst batches.  Every run is its own process (so its peak RSS, VmHWM or else ru_maxrss, is its own); the two trees alternate for
`--rounds` rounds, then this tree runs `--rounds` more times with a budget of one file (the largest file's text).  Reports per run:
corrected bases/s, first_submit_s, alignment_ingest_s, total_s, peak RSS and alignment_peak_bytes; the card's name and power limit and
the host's core count are read in the same run.  Prints one JSON object.

  python tools/measure_streaming_ingest.py --parent <tree of the parent commit, built>
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.measure_pos_stage import card  # noqa: E402

CHILD = r"""
import json, sys
tree, args, kw = sys.argv[1], json.loads(sys.argv[2]), json.loads(sys.argv[3])
sys.path.insert(0, tree)
from herro_b200 import hostio
r = hostio.inference(*args, **kw)
hwm = [int(l.split()[1]) * 1024 for l in open("/proc/self/status") if l.startswith("VmHWM:")]
import resource  # where /proc does not report VmHWM, the kernel's maximum resident set of this process
hwm = hwm[0] if hwm else resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
print(json.dumps(dict({k: float(v) for k, v in r.items()}, peak_rss_bytes=hwm)))
"""


def run(tree, args, kw):
    tree = os.path.abspath(tree)
    out = subprocess.run([sys.executable, "-c", CHILD, tree, json.dumps(args), json.dumps(kw)], cwd=tree, capture_output=True,
                         text=True)
    if out.returncode != 0:
        raise RuntimeError(f"inference in {tree} failed ({out.returncode}): {out.stderr[-2000:]}")
    r = json.loads(out.stdout.strip().splitlines()[-1])
    r["bases_per_s"] = r["corrected_bases"] / r["total_s"]
    with open(args[3], "rb") as f:  # the record set, whatever order the consumers wrote it in
        r["records_sha256"] = hashlib.sha256(b">".join(sorted(f.read().split(b">")[1:]))).hexdigest()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="a tree of the parent commit on which build() has run")
    ap.add_argument("--reads", type=int, default=50000)
    ap.add_argument("--read-len", type=int, default=20000)
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--threads", type=int, default=8, help="feature threads (-t)")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()

    import pyarrow as pa
    from herro_b200 import weights as hbw
    from tools import synth
    synth.build()
    work = tempfile.mkdtemp(prefix="herro_stream_ingest_")
    try:
        t0 = time.time()
        rs = synth.generate(args.reads, args.read_len, profile="r10", seed=1, coverage=40.0, min_ovl=2048)
        fq, alns = os.path.join(work, "reads.fastq"), os.path.join(work, "alns")
        synth.write_fastq(rs, fq)
        os.makedirs(alns)
        per = (rs.n + args.files - 1) // args.files
        codec = pa.Codec("zstd")
        text, comp = [], []
        for bi, s in enumerate(range(0, rs.n, per)):
            tg = range(s, min(s + per, rs.n))
            body = f"{len(tg)}\n".encode() + b"".join((rs.ids[t] + "\n").encode() for t in tg) + b"".join(synth.paf_lines(rs, tg))
            z = codec.compress(body, asbytes=True)
            with open(os.path.join(alns, f"{bi}.oec.zst"), "wb") as f:
                f.write(z)
            text.append(len(body))
            comp.append(len(z))
            del body, z
        bases = rs.total_bases
        del rs
        t_write = time.time() - t0
        model = os.path.join(work, "model.hbw")
        hbw.save_blob(model, hbw.NetConfig(), hbw.random_weights(hbw.NetConfig(), seed=7))
        pos = [fq, alns, model, os.path.join(work, "out.fasta"), 4096, args.batch_size, args.threads]
        runs = []
        for rnd in range(args.rounds):
            for name, tree, kw in (("parent", args.parent, {}), ("stream_default", ROOT, {})):
                r = run(tree, pos, kw)
                runs.append(dict(round=rnd, tree=name, **r))
        for rnd in range(args.rounds):
            r = run(ROOT, pos, dict(aln_buffer_bytes=max(text)))
            runs.append(dict(round=rnd, tree="stream_one_file", **r))
        checks = {}
        for name in ("parent", "stream_default", "stream_one_file"):
            rr = [r for r in runs if r["tree"] == name]
            checks[name] = sorted({r["records_sha256"] for r in rr})
        res = dict(card=card(), host_cores=os.cpu_count(), reads=args.reads, read_len=args.read_len, read_bases=bases,
                   files=len(text), text_bytes=text, compressed_bytes=comp, input_write_s=t_write, threads=args.threads,
                   batch_size=args.batch_size, runs=runs, record_sets=checks,
                   identical=len({h for v in checks.values() for h in v}) == 1)
    finally:
        shutil.rmtree(work, ignore_errors=True)
    s = json.dumps(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s)
    print(s)


if __name__ == "__main__":
    main()
