"""The host side of `herro align` without a GPU: the overlap-only PAF reader (admission, gzip, chunks) and the batch writer (routing,
header layout, columns), with CIGARs from the alignment oracle; the written batches read back through hostio.Alignments."""
import gzip
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import align_oracle as ao  # noqa: E402
from herro_b200 import api, hostio  # noqa: E402
from tools import synth  # noqa: E402



@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("align_batches")
    rs = synth.generate(30, 5000, profile="r10", seed=9, coverage=12.0, min_len=3000)
    fq = str(d / "reads.fastq")
    synth.write_fastq(rs, fq)
    lines = []
    for k, ln in enumerate(synth.paf_lines(rs)):
        cols = ln.rstrip(b"\n").split(b"\t")[:12]
        if k % 5 == 0:
            cols += [b"tp:A:P", b"cg:Z:1M"]   # a tag and a CIGAR that must be ignored
        lines.append(b"\t".join(cols) + b"\n")
    c0 = lines[0].split(b"\t")
    lines.append(lines[3])                                                            # a repeated pair: written as it comes
    lines.append(b"\t".join([c0[0], c0[1], c0[2], c0[3], c0[4], c0[0], c0[1]] + c0[7:]))  # a self overlap
    lines.append(b"\t".join([b"no_such_read"] + c0[1:]))                             # an unknown name
    paf = str(d / "ovl.paf")
    open(paf, "wb").write(b"".join(lines))
    with gzip.open(paf + ".gz", "wb") as f:
        f.write(b"".join(lines))
    min_len = int(np.sort(np.diff(rs.off))[4]) + 1  # the five shortest reads are not loaded: their lines are skipped
    return rs, fq, paf, lines, d, min_len


def expected_admitted(rs, lines, reads):
    names = {n.decode(): i for i, n in enumerate(reads.ids)}
    out = []
    for ln in lines:
        c = ln.rstrip(b"\n").split(b"\t")
        q, t = c[0].decode(), c[5].decode()
        if q in names and t in names and q != t:
            out.append((names[q], int(c[2]), int(c[3]), int(c[4] == b"-"), names[t], int(c[7]), int(c[8]), c[11]))
    return out


def read_all(paf, reads, chunk):
    r = hostio.PafReader(paf, reads)
    got = []
    while (o := r.next(chunk)) is not None:
        got.append(o)
    st = r.stats()
    r.close()
    return (np.concatenate(got) if got else np.zeros(0, api.OVERLAP_DTYPE)), st


def test_paf_admission_gzip_and_chunks(data):
    rs, fq, paf, lines, _, min_len = data
    reads = hostio.Reads(fq, min_len=min_len)
    assert reads.n == rs.n - 5
    want = expected_admitted(rs, lines, reads)
    a, st = read_all(paf, reads, 1 << 20)
    b, _ = read_all(paf + ".gz", reads, 1 << 20)
    c, _ = read_all(paf, reads, 7)
    assert st["lines"] == len(lines) and st["skipped"] == len(lines) - len(want)
    for x in (b, c):
        assert x.tobytes() == a.tobytes()
    got = [(int(o["qid"]), int(o["qstart"]), int(o["qend"]), int(o["strand"]), int(o["tid"]), int(o["tstart"]), int(o["tend"]))
           for o in a]
    assert got == [w[:7] for w in want]
    assert (a["cigar_len"] == 0).all() and (a["cigar"] == 0).all()


def oracle_align(reads, seqs, ovl, w=128):
    codes = {}
    out = ovl.copy()
    status = np.zeros(len(ovl), np.int32)
    matches = np.zeros(len(ovl), np.uint32)
    cigs = []
    for k, o in enumerate(ovl):
        for x in (int(o["qid"]), int(o["tid"])):
            if x not in codes:
                codes[x] = ao.codes(seqs[reads.ids[x].decode()])
        st, (qs, qe, ts, te), cig, mt = ao.align_overlap(codes[int(o["tid"])], codes[int(o["qid"])], int(o["qstart"]), int(o["qend"]),
                                                         int(o["strand"]), int(o["tstart"]), int(o["tend"]), w)
        status[k], matches[k] = st, mt
        out[k]["qstart"], out[k]["qend"], out[k]["tstart"], out[k]["tend"] = qs, qe, ts, te
        cigs.append(cig)
    buf = np.frombuffer(b"".join(cigs) or b"\0", np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(c) for c in cigs])]).astype(np.uint64)
    out["cigar"] = buf.ctypes.data + off[:-1]
    out["cigar_len"] = np.diff(off).astype(np.uint32)
    return out, status, matches, cigs, buf


def decompress(path):
    import pyarrow as pa
    with pa.CompressedInputStream(pa.OSFile(path), "zstd") as f:
        return f.read()


def test_batches_routing_header_and_read_back(data):
    rs, fq, paf, _, d, min_len = data
    reads = hostio.Reads(fq, min_len=min_len)
    seqs = {rs.ids[i]: rs.seq(i) for i in range(rs.n)}
    out_dir = str(d / "alns")
    bs = 8
    r = hostio.PafReader(paf + ".gz", reads)
    wr = hostio.BatchWriter(out_dir, reads, batch_size=bs)
    written = []
    keep = []
    while (ovl := r.next(11)) is not None:
        al, status, matches, cigs, buf = oracle_align(reads, seqs, ovl)
        keep.append(buf)
        wr.write(r, al, status, matches)
        written += [(al[k], cigs[k], int(matches[k])) for k in range(len(al)) if status[k] >= 0]
    per_batch = wr.close()
    r.close()
    nb = (reads.n + bs - 1) // bs
    assert sorted(os.listdir(out_dir)) == sorted(f"{k}.oec.zst" for k in range(nb))
    assert per_batch == [sum(1 for o, _, _ in written if int(o["tid"]) // bs == k) for k in range(nb)]
    for k in range(nb):
        text = decompress(os.path.join(out_dir, f"{k}.oec.zst")).split(b"\n")
        ids = reads.ids[k * bs:(k + 1) * bs]
        assert text[0] == str(len(ids)).encode() and text[1:1 + len(ids)] == list(ids)
        body = [ln for ln in text[1 + len(ids):] if ln]
        mine = [(o, c, m) for o, c, m in written if int(o["tid"]) // bs == k]
        assert len(body) == len(mine)
        for ln, (o, c, m) in zip(body, mine):
            f = ln.split(b"\t")
            assert len(f) == 13 and f[12] == b"cg:Z:" + c
            assert f[0] == reads.ids[int(o["qid"])] and f[5] == reads.ids[int(o["tid"])]
            assert [int(x) for x in f[2:4] + f[7:9]] == [int(o["qstart"]), int(o["qend"]), int(o["tstart"]), int(o["tend"])]
            assert int(f[9]) == m and int(f[10]) == sum(int(n) for n in __import__("re").findall(rb"(\d+)[MID]", c))
    # read back: the reader's first-wins rule drops the repeated pair; everything else comes back as written
    A = hostio.Alignments(out_dir, reads)
    back = {}
    for t in range(A.n_targets):
        rid, ov = A.target(t)
        for o in ov:
            back.setdefault((int(o["qid"]), rid), []).append(
                (int(o["qstart"]), int(o["qend"]), int(o["tstart"]), int(o["tend"]), C_string(o)))
    first = {}
    for o, c, _ in written:
        first.setdefault((int(o["qid"]), int(o["tid"])), (int(o["qstart"]), int(o["qend"]), int(o["tstart"]), int(o["tend"]), c))
    assert {k: v[0] for k, v in back.items()} == first and all(len(v) == 1 for v in back.values())
    A.close()


def C_string(o):
    import ctypes
    return ctypes.string_at(int(o["cigar"]), int(o["cigar_len"]))
