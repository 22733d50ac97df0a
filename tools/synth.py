"""Python front-end of the synthetic read-set generator (tools/synth.cpp) + writers for the
reference's on-disk inputs: FASTQ and `--read-alns` `*.oec.zst` batches
(scripts/batch.py:24-44, src/overlaps.rs:288-323).  Bench/test input generation only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libsynth.so")

PROFILES = {
    # sub, ins, del, hp_boost  (SURVEY.md §8d)
    "r10": (0.004, 0.003, 0.005, 0.6),
    "r9": (0.015, 0.015, 0.025, 0.6),
    # low-error reads: long CIGAR ops and tied rankings.  The haplotype SNPs / indels (het_snp, het_indel) and the long
    # deletions stay, so supported positions still appear at het sites.
    "exact": (0.0, 0.0, 0.0, 0.0),
    "q30": (1e-3, 1e-4, 1e-4, 0.6),
}


def build(force=False):
    src = os.path.join(_HERE, "synth.cpp")
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(src):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", _LIB, src])
    return _LIB


@dataclass
class ReadSet:
    ids: list            # list[str]
    seqs: np.ndarray     # concatenated ASCII u8
    quals: np.ndarray    # concatenated Phred+33 u8
    off: np.ndarray      # [n+1] u64
    aln_off: np.ndarray  # [n+1] u64 — alignments of target t are [aln_off[t], aln_off[t+1])
    ovl9: np.ndarray     # [n_aln, 9] u32: qid qlen qstart qend strand tid tlen tstart tend
    cig_off: np.ndarray  # [n_aln+1] u64
    cigars: np.ndarray   # concatenated ASCII u8
    strand: np.ndarray
    hap: np.ndarray

    @property
    def n(self):
        return len(self.ids)

    def seq(self, i) -> bytes:
        return self.seqs[int(self.off[i]):int(self.off[i + 1])].tobytes()

    def qual(self, i) -> bytes:
        return self.quals[int(self.off[i]):int(self.off[i + 1])].tobytes()

    def cigar(self, a) -> bytes:
        return self.cigars[int(self.cig_off[a]):int(self.cig_off[a + 1])].tobytes()

    def target_alns(self, t):
        a0, a1 = int(self.aln_off[t]), int(self.aln_off[t + 1])
        return self.ovl9[a0:a1], [self.cigar(a) for a in range(a0, a1)]

    @property
    def total_bases(self):
        return int(self.off[-1])


def _lib():
    build()
    L = C.CDLL(_LIB)
    L.synth_generate.restype = C.c_void_p
    L.synth_generate.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                 C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    L.synth_free.argtypes = [C.c_void_p]
    L.synth_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    vp = C.c_void_p
    L.synth_get_reads.argtypes = [vp] + [vp] * 6
    L.synth_get_alns.argtypes = [vp] + [vp] * 4
    L.synth_make_alns.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    L.synth_make_alns.restype = None
    L.synth_read_lens.argtypes = [vp, vp]
    L.synth_read_lens.restype = None
    return L


class Generator:
    """Two-phase use of the generator: reads first (their lengths decide the sharding), then the alignments of a chosen
    target subset.  `generate()` below is the one-shot form."""

    def __init__(self, n_reads: int, mean_len: int, *, profile="r10", seed=1, coverage=40.0, sd_frac=0.10, min_len=None,
                 max_len=None, het_snp=1e-3, het_indel=1e-4, long_del=2e-6, min_ovl=2048, genome_len=None, threads=None):
        self.L = _lib()
        sub, ins, dele, hpb = PROFILES[profile]
        if genome_len is None:
            genome_len = max(int(n_reads * mean_len / coverage), mean_len * 2)
        min_len = min_len if min_len is not None else max(int(mean_len * 0.5), 1)
        max_len = max_len if max_len is not None else int(mean_len * 2)
        self.threads = threads or os.cpu_count() or 1
        self.n = n_reads
        self.h = self.L.synth_generate(seed, genome_len, n_reads, mean_len, int(mean_len * sd_frac), min_len, max_len, sub, ins,
                                       dele, hpb, het_snp, het_indel, long_del, min_ovl, self.threads, 0, 0, 1, 0)

    def read_lens(self) -> np.ndarray:
        out = np.zeros(self.n, np.uint32)
        self.L.synth_read_lens(self.h, out.ctypes.data)
        return out

    def readset(self, targets=None, target_stride=(1, 0)) -> ReadSet:
        """All reads + the alignments of targets [begin, end) with t % stride == phase (default: every target)."""
        L, h = self.L, self.h
        tb, te = targets if targets is not None else (0, self.n)
        L.synth_make_alns(h, tb, te, target_stride[0], target_stride[1], self.threads)
        sz = (C.c_uint64 * 4)()
        L.synth_sizes(h, sz)
        n, nb, na, cb = (int(x) for x in sz)
        seqs = np.zeros(nb, np.uint8); quals = np.zeros(nb, np.uint8); off = np.zeros(n + 1, np.uint64)
        strand = np.zeros(n, np.uint8); hap = np.zeros(n, np.uint8); gs = np.zeros(n, np.uint64)
        L.synth_get_reads(h, seqs.ctypes.data, quals.ctypes.data, off.ctypes.data, strand.ctypes.data,
                          hap.ctypes.data, gs.ctypes.data)
        aln_off = np.zeros(n + 1, np.uint64); ovl9 = np.zeros((max(na, 1), 9), np.uint32)
        cig_off = np.zeros(na + 1, np.uint64); cig = np.zeros(max(cb, 1), np.uint8)
        L.synth_get_alns(h, aln_off.ctypes.data, ovl9.ctypes.data, cig_off.ctypes.data, cig.ctypes.data)
        ids = [f"read_{i:06d}" for i in range(n)]
        return ReadSet(ids, seqs, quals, off, aln_off, ovl9[:na], cig_off, cig[:cb], strand, hap)

    def close(self):
        if self.h:
            self.L.synth_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def generate(n_reads: int, mean_len: int, *, targets=None, target_stride=(1, 0), **kw) -> ReadSet:
    """targets=(begin, end) / target_stride=(stride, phase): build alignments only for those target reads (all reads are
    always generated, so the read store and every query are those of the full set)."""
    g = Generator(n_reads, mean_len, **kw)
    try:
        return g.readset(targets, target_stride)
    finally:
        g.close()


def write_fastq(rs: ReadSet, path: str, descriptions=None):
    with open(path, "wb") as f:
        for i in range(rs.n):
            hdr = rs.ids[i] + ((" " + descriptions[i]) if descriptions and descriptions[i] is not None else "")
            f.write(b"@" + hdr.encode() + b"\n" + rs.seq(i) + b"\n+\n" + rs.qual(i) + b"\n")


def paf_lines(rs: ReadSet, targets=None):
    targets = range(rs.n) if targets is None else targets
    for t in targets:
        for a in range(int(rs.aln_off[t]), int(rs.aln_off[t + 1])):
            q, ql, qs, qe, st, tt, tl, ts, te = (int(x) for x in rs.ovl9[a])
            yield (f"{rs.ids[q]}\t{ql}\t{qs}\t{qe}\t{'-' if st else '+'}\t{rs.ids[tt]}\t{tl}\t{ts}\t{te}\t0\t0\t60\t"
                   f"cg:Z:").encode() + rs.cigar(a) + b"\n"


def write_oec_batches(rs: ReadSet, outdir: str, batch_size: int = 50_000):
    """`<N>\\n<read_id>\\n x N<PAF line>...` zstd-compressed per batch of targets (App. C)."""
    import pyarrow as pa
    os.makedirs(outdir, exist_ok=True)
    codec = pa.Codec("zstd")
    for bi, s in enumerate(range(0, rs.n, batch_size)):
        tg = range(s, min(s + batch_size, rs.n))
        body = f"{len(tg)}\n".encode() + b"".join((rs.ids[t] + "\n").encode() for t in tg)
        body += b"".join(paf_lines(rs, tg))
        with open(os.path.join(outdir, f"{bi}.oec.zst"), "wb") as f:
            f.write(codec.compress(body, asbytes=True))
