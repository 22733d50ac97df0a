"""hb_align_overlaps on the device against the alignment oracle (tests/align_oracle.cpp): every output of hb_align_fetch
(coordinates, CIGAR text, status, matches) byte for byte, on synthetic R10 / R9 sets and on chosen edge cases."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import align_oracle as ao  # noqa: E402
import helpers  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu

BASES = np.frombuffer(b"ACGT", np.uint8)


def overlaps(rows):
    """hb_overlap[] from (qid, qlen, qstart, qend, strand, tid, tlen, tstart, tend) rows, without CIGARs."""
    from herro_b200 import Context
    rows = np.asarray(rows, np.uint32).reshape(-1, 9)
    cig = np.zeros(1, np.uint8)
    return Context.make_overlaps(rows, cig, np.zeros(len(rows) + 1, np.uint64))


def oracle(seqs, ovl, w):
    codes = [ao.codes(s) for s in seqs]
    out = []
    for o in ovl:
        q, t = int(o["qid"]), int(o["tid"])
        out.append(ao.align_overlap(codes[t], codes[q], int(o["qstart"]), int(o["qend"]), int(o["strand"]), int(o["tstart"]),
                                    int(o["tend"]), w))
    return out


def check(got, want, ovl):
    assert len(got["status"]) == len(want)
    for k, (st, (qs, qe, ts, te), cig, mt) in enumerate(want):
        o = got["overlaps"][k]
        assert int(got["status"][k]) == st, k
        assert (int(o["qstart"]), int(o["qend"]), int(o["tstart"]), int(o["tend"])) == (qs, qe, ts, te), k
        assert got["cigars"][k] == cig, k
        assert int(got["matches"][k]) == mt, k
        for f in ("qid", "qlen", "strand", "tid", "tlen"):
            assert o[f] == ovl[k][f]


def readset_context(rs, store=False):
    from herro_b200.api import Context, ReadStore
    ctx = Context(None)
    if store:
        st = ReadStore(rs.seqs, rs.quals, rs.off)
        ctx.attach_read_store(st)
    else:
        ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    return ctx


def synth_overlaps(rs, limit):
    return overlaps(rs.ovl9[:limit])


@pytest.fixture(scope="module", params=["r10", "r9"])
def synth_set(request):
    rs = synth.generate(40, 6000, profile=request.param, seed=7, coverage=15.0)
    return rs, [rs.seq(i) for i in range(rs.n)]


@pytest.mark.parametrize("w", [16, 64, 0])
def test_synthetic_sets_match_the_oracle(synth_set, w):
    rs, seqs = synth_set
    ovl = synth_overlaps(rs, 160)
    assert set(ovl["strand"].tolist()) == {0, 1}
    ctx = readset_context(rs)
    got = ctx.align(ovl, band_w=w)
    want = oracle(seqs, ovl, w or 128)
    check(got, want, ovl)
    edge = sum(1 for x in want if x[0] == ao.HB_ALN_BAND_EDGE)
    if w == 16:
        assert edge > 0  # a band this narrow cannot hold every path
    assert got["shape"]["n_band_edge"] == edge and got["shape"]["n_failed"] == 0
    assert got["shape"]["cells"] == sum((int(o["tend"]) - int(o["tstart"]) + 1) * 2 * (w or 128) for o in ovl)
    assert got["shape"]["cigar_bytes"] == sum(len(c) for c in got["cigars"])


def test_host_store_equals_uploaded_store(synth_set):
    rs, _ = synth_set
    ovl = synth_overlaps(rs, 80)
    a = readset_context(rs).align(ovl, 64)
    b = readset_context(rs, store=True).align(ovl, 64)
    for k in ("status", "matches"):
        assert np.array_equal(a[k], b[k])
    assert a["cigars"] == b["cigars"]
    for f in ("qstart", "qend", "tstart", "tend"):
        assert np.array_equal(a["overlaps"][f], b["overlaps"][f])


def mutate(rng, s, rate):
    b = np.frombuffer(s, np.uint8)
    keep = rng.random(len(b)) >= rate
    sub = rng.random(len(b)) < rate
    b = np.where(sub, BASES[rng.integers(0, 4, len(b))], b)
    return b[keep].tobytes()


def revcomp(s):
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


class Custom:
    """Hand-made reads: the store's first and last reads take part, next to long deletions and homopolymer indels."""

    def __init__(self, seed=3):
        rng = np.random.default_rng(seed)
        r0 = BASES[rng.integers(0, 4, 6000)].tobytes()
        # homopolymer runs in r0, one base shorter in r2
        hp = bytearray(r0)
        for p in range(300, 5600, 400):
            hp[p:p + 8] = b"A" * 8
        r0 = bytes(hp)
        r1 = r0[:2000] + r0[2070:]                      # a 70 bp deletion: the long gap piece wins
        r2 = bytearray(r0)
        for p in range(5500, 300, -400):
            del r2[p]                                   # one base of every homopolymer run (fix_cigar shifts the gap left)
        r3 = revcomp(mutate(rng, r0, 0.01))             # strand 1
        r4 = mutate(rng, r0[:3000], 0.02) + r0[3000:3055] + mutate(rng, r0[3055:], 0.02)
        self.seqs = [r0, r1, bytes(r2), r3, r4, BASES[rng.integers(0, 4, 40)].tobytes(), mutate(rng, r0[-4000:], 0.01)]
        self.quals = [b"+" * len(s) for s in self.seqs]

    def upload(self, ctx):
        off = np.zeros(len(self.seqs) + 1, np.uint64)
        off[1:] = np.cumsum([len(s) for s in self.seqs])
        ctx.upload_reads(np.frombuffer(b"".join(self.seqs), np.uint8), np.frombuffer(b"".join(self.quals), np.uint8), off)

    def row(self, q, qs, qe, st, t, ts, te):
        return (q, len(self.seqs[q]), qs, qe, st, t, len(self.seqs[t]), ts, te)


def test_edge_cases_match_the_oracle():
    from herro_b200 import Context
    c = Custom()
    L = [len(s) for s in c.seqs]
    last = len(c.seqs) - 1
    rows = [
        c.row(1, 0, L[1], 0, 0, 0, L[0]),                  # 70 bp deletion
        c.row(2, 0, L[2], 0, 0, 0, L[0]),                  # homopolymer deletions
        c.row(3, 0, L[3], 1, 0, 0, L[0]),                  # reverse strand
        c.row(0, 0, L[0], 0, 4, 0, L[4]),
        c.row(0, 10, 11, 0, 1, 10, 11),                    # 1-base spans
        c.row(0, 10, 12, 1, 1, 10, 11),                    # m / n exactly 2
        c.row(0, 10, 13, 0, 1, 10, 11),                    # just beyond: HB_ERR_INPUT
        c.row(0, 0, 2000, 0, 1, 0, 1000),                  # m / n exactly 2, long
        c.row(0, 0, 1000, 0, 1, 0, 2001),                  # n / m just beyond 2: HB_ERR_INPUT
        c.row(0, 5, 5, 0, 1, 5, 9),                        # empty span: HB_ERR_INPUT
        c.row(0, 0, L[0] + 1, 0, 1, 0, 100),               # outside its read: HB_ERR_INPUT
        c.row(last, 0, L[last], 0, 0, L[0] - 4000, L[0]),  # the store's last read, at the end of the first
        c.row(0, L[0] - 4000, L[0], 1, last, 0, L[last]),  # ... and the other way, on strand 1
        c.row(5, 0, 40, 0, 0, 100, 140),                   # unrelated short sequences
    ]
    ovl = overlaps(rows)
    for w in (16, 64, 128, 256):
        ctx = Context(None)
        c.upload(ctx)
        got = ctx.align(ovl, band_w=w)
        want = oracle(c.seqs, ovl, w)
        check(got, want, ovl)
        assert [int(x) for x in got["status"][[6, 8, 9, 10]]] == [ao.HB_ERR_INPUT] * 4
        assert got["shape"]["n_failed"] == 4
        if w >= 64:
            assert b"70D" in got["cigars"][0]


def test_call_errors():
    from herro_b200 import Context
    from herro_b200.api import HerroError
    c = Custom()
    ctx = Context(None)
    ok = overlaps([c.row(1, 0, 100, 0, 0, 0, 100)])
    with pytest.raises(HerroError) as e:
        ctx.align(ok)
    assert e.value.code == -6  # no reads yet
    c.upload(ctx)
    for bad_w in (8, 24, 272, 512):
        with pytest.raises(HerroError) as e:
            ctx.align(ok, band_w=bad_w)
        assert e.value.code == -1
    for r in ([c.row(1, 0, 100, 2, 0, 0, 100)], [(99, 100, 0, 100, 0, 0, 6000, 0, 100)], [(0, 100, 0, 100, 0, 99, 6000, 0, 100)]):
        with pytest.raises(HerroError) as e:
            ctx.align(overlaps(r))
        assert e.value.code == -1
    assert ctx.align(ok)["shape"]["n_overlaps"] == 1
    assert ctx.align(overlaps(np.zeros((0, 9))))["shape"]["n_overlaps"] == 0


def test_long_overlaps_over_several_waves(monkeypatch):
    from herro_b200 import Context
    rng = np.random.default_rng(11)
    r0 = BASES[rng.integers(0, 4, 100_000)].tobytes()
    seqs = [r0, mutate(rng, r0, 0.01), revcomp(mutate(rng, r0, 0.02)), mutate(rng, r0[:60_000], 0.01)]
    off = np.zeros(len(seqs) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    L = [len(s) for s in seqs]
    rows = [(1, L[1], 0, L[1], 0, 0, L[0], 0, L[0]), (2, L[2], 0, L[2], 1, 0, L[0], 0, L[0]),
            (0, L[0], 0, L[0], 0, 1, L[1], 0, L[1]), (3, L[3], 0, L[3], 0, 0, L[0], 0, 60_000)]
    ovl = overlaps(rows)
    monkeypatch.setenv("HERRO_B200_ALN_WAVE_BYTES", str(30 << 20))  # one 100 kb overlap per wave at w = 128
    ctx = Context(None)
    ctx.upload_reads(np.frombuffer(b"".join(seqs), np.uint8), np.full(int(off[-1]), 43, np.uint8), off)
    got = ctx.align(ovl)
    check(got, oracle(seqs, ovl, 128), ovl)
    assert (got["status"] >= 0).all()


def test_beside_the_pipeline_and_into_it():
    """An alignment call running beside hb_submit_alignments leaves the pipeline's output unchanged, and its output overlaps,
    submitted as they come back, correct the reads as the oracle's alignments do."""
    from herro_b200 import Context
    rs = helpers.small_readset(n_reads=30, mean_len=8000, seed=4)
    seqs = [rs.seq(i) for i in range(rs.n)]
    model = helpers.model_path(seed=3)
    plain = overlaps(rs.ovl9)
    want = oracle(seqs, plain, 128)

    def oracle_overlaps():
        cigs = [c for _, _, c, _ in want]
        buf = np.frombuffer(b"".join(cigs) or b"\0", np.uint8)
        off = np.zeros(len(cigs) + 1, np.uint64)
        off[1:] = np.cumsum([len(c) for c in cigs])
        o = Context.make_overlaps(rs.ovl9, buf, off)
        for k, (_, (qs, qe, ts, te), _, _) in enumerate(want):
            o[k]["qstart"], o[k]["qend"], o[k]["tstart"], o[k]["tend"] = qs, qe, ts, te
        return o, buf

    def run(ovl, beside=False):
        ctx = Context(model, 0, 4096, 64)
        ctx.upload_reads(rs.seqs, rs.quals, rs.off)
        stop = threading.Event()
        side = []

        def aligner():
            while not stop.is_set():
                side.append(ctx.align(plain[:40]))

        th = threading.Thread(target=aligner) if beside else None
        if th:
            th.start()
        for t in range(rs.n):
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            if a1 > a0:
                ctx.submit_alignments(t, ovl[a0:a1])
        ctx.flush()
        out = {r.rid: r.segments for r in ctx.drain()}
        if th:
            stop.set()
            th.join()
            assert side
            for s in side:
                assert s["cigars"] == [x[2] for x in want[:40]]
        return out

    ora, _buf = oracle_overlaps()
    base = run(ora)
    assert base and any(base.values())
    assert run(ora, beside=True) == base
    dev = readset_context(rs).align(plain)
    keep = dev["cigar_text"]  # noqa: F841  (the overlaps point into it)
    assert run(dev["overlaps"]) == base


@pytest.fixture(scope="module")
def overlap_only_set(tmp_path_factory):
    """A synthetic FASTQ and the generator's PAF with its cg:Z: fields stripped, as minimap2 without -c writes it."""
    d = tmp_path_factory.mktemp("align_e2e")
    rs = helpers.small_readset(n_reads=30, mean_len=8000, seed=6)
    fq = str(d / "reads.fastq")
    synth.write_fastq(rs, fq)
    paf = str(d / "ovl.paf")
    with open(paf, "wb") as f:
        for ln in synth.paf_lines(rs):
            f.write(b"\t".join(ln.rstrip(b"\n").split(b"\t")[:12]) + b"\n")
    return rs, fq, paf, d


def fasta_records(path):
    """-> sorted (record name, sequence) pairs of a FASTA file"""
    text = open(path, "rb").read()
    out = []
    for rec in text.split(b">")[1:]:
        head, _, seq = rec.partition(b"\n")
        out.append((head.split()[0], seq.replace(b"\n", b"")))
    return sorted(out)


def test_cli_align_then_inference_equals_the_oracle_alignments(overlap_only_set):
    from herro_b200 import Context, api, cli
    rs, fq, paf, d = overlap_only_set
    model = helpers.model_path(seed=3)
    alns = str(d / "alns")
    r = cli.main(["align", "-d", "0", "--batch-size", "7", fq, paf, alns])
    assert r["lines"] == len(rs.ovl9) and r["skipped"] == 0 and r["failed"] == 0 and r["aligned"] == len(rs.ovl9)
    assert sorted(os.listdir(alns)) == sorted(f"{k}.oec.zst" for k in range((rs.n + 6) // 7))
    out = str(d / "out.fasta")
    cli.main(["inference", "--read-alns", alns, "-m", model, "-b", "64", fq, out])
    # the oracle's alignments submitted directly
    seqs = [rs.seq(i) for i in range(rs.n)]
    want = oracle(seqs, overlaps(rs.ovl9), 128)
    cigs = [c for _, _, c, _ in want]
    buf = np.frombuffer(b"".join(cigs), np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(c) for c in cigs])]).astype(np.uint64)
    ovl = Context.make_overlaps(rs.ovl9, buf, off)
    for k, (_, (qs, qe, ts, te), _, _) in enumerate(want):
        ovl[k]["qstart"], ovl[k]["qend"], ovl[k]["tstart"], ovl[k]["tend"] = qs, qe, ts, te
    ctx = Context(model, 0, 4096, 64)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    for t in range(rs.n):
        a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
        if a1 > a0:
            ctx.submit_alignments(t, ovl[a0:a1])
    ctx.flush()
    direct = str(d / "direct.fasta")
    with open(direct, "wb") as f:
        for res in ctx.drain():
            if res.segments:
                f.write(api.fasta_records(rs.ids[res.rid].encode(), None, res.segments))
    got, ref = fasta_records(out), fasta_records(direct)
    assert ref and got == ref
