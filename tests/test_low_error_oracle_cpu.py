"""The oracle against answers derived by hand on read sets built by hand: a seeded random target and queries that are exact
copies of it (or of a sub-span of it), CIGARs `{n}M`.  A reverse copy is the reverse complement with its qualities reversed,
so in target orientation every copy shows the target's bases and its own qualities.  These sets reach what noisy reads almost
never do: one CIGAR op per overlap-window, windows whose rankings tie everywhere, windows with no supported position.  The GPU
tests of the same sets (test_gpu_low_error_reads.py) rest on these answers, not on the oracle alone."""
import hashlib
import math
import re

import numpy as np
import pytest

import helpers
from herro_b200 import api
from oracle import pyoracle as po
from tools import synth

W = 1024
TLEN = 5 * W + 300          # six windows, the last one 300 bases long
N_COPIES = 35               # more than the 30 columns the model takes
SNP_POS = 2 * W + 517       # in window 2
SNP_QIDS = [3, 6, 9, 12, 15, 18, 21, 24, 27, 30]   # copies carrying the substitution, interleaved with the exact ones
TOKEN = {c: i for i, c in enumerate(b"ACGT*acgt#.")}  # BASES_MAP (src/inference.rs:23-31)
_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def revcomp(s: bytes) -> bytes:
    return s.translate(_COMP)[::-1]


def random_bases(rng, n) -> bytes:
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def random_quals(rng, n) -> bytes:
    return (33 + rng.integers(2, 45, n)).astype(np.uint8).tobytes()


def build_readset(target: bytes, tqual: bytes, copies) -> synth.ReadSet:
    """Read 0 is the target; read k (k >= 1) is copies[k - 1] = (seq, qual, reverse, tstart, tend, cigar) with seq / qual in target
    orientation.  One alignment per copy, all with target 0, in copy order."""
    return build_groups([(target, tqual, copies)])


def build_groups(groups) -> synth.ReadSet:
    """build_readset for several targets: each group (target, tqual, copies) appends its target, then its copies."""
    seqs, quals, ovl9, cigs, aln_off = [], [], [], [], [0]
    for target, tqual, copies in groups:
        t = len(seqs)
        seqs.append(target)
        quals.append(tqual)
        for k, (s, q, rev, ts, te, cig) in enumerate(copies, start=t + 1):
            seqs.append(revcomp(s) if rev else s)
            quals.append(q[::-1] if rev else q)
            ovl9.append([k, len(s), 0, len(s), int(rev), t, len(target), ts, te])
            cigs.append(cig)
        aln_off += [len(ovl9)] * (len(copies) + 1)  # the target's alignments, then none for each copy
    n = len(seqs)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    cig_off = np.zeros(len(cigs) + 1, np.uint64)
    cig_off[1:] = np.cumsum([len(c) for c in cigs])
    return synth.ReadSet([f"read_{i:06d}" for i in range(n)], np.frombuffer(b"".join(seqs), np.uint8).copy(),
                         np.frombuffer(b"".join(quals), np.uint8).copy(), off, np.array(aln_off, np.uint64),
                         np.array(ovl9, np.uint32).reshape(-1, 9), cig_off, np.frombuffer(b"".join(cigs), np.uint8).copy(),
                         np.zeros(n, np.uint8), np.zeros(n, np.uint8))


def full_copies(tlen=TLEN, n=N_COPIES, seed=11, snp_qids=(), snp_pos=None):
    """A random target and n full-length copies, forward and reverse alternately (qid 1 forward).  The copies whose qid is in
    snp_qids carry one substitution at snp_pos.  -> (ReadSet, copy sequences and qualities in target orientation)."""
    rng = np.random.default_rng(seed)
    target, tqual = random_bases(rng, tlen), random_quals(rng, tlen)
    copies, oriented = [], []
    for k in range(1, n + 1):
        s = bytearray(target)
        if k in snp_qids:
            s[snp_pos] = b"ACGT"[(b"ACGT".index(s[snp_pos]) + 1) % 4]
        q = random_quals(rng, tlen)
        copies.append((bytes(s), q, k % 2 == 0, 0, tlen, f"{tlen}M".encode()))
        oriented.append((bytes(s), q))
    return build_readset(target, tqual, copies), oriented


def window_bounds(wid, tlen=TLEN, w=W):
    return wid * w, min((wid + 1) * w, tlen)


def check_copy_columns(win, wid, rs, oriented, kept_qids):
    """Column 0 is the target; column j >= 1 is copy kept_qids[j - 1], its bases lowercase when reverse, its own qualities."""
    a, b = window_bounds(wid)
    t = rs.seq(0)[a:b]
    assert win.bases.shape == (b - a, 31)
    assert bytes(win.bases[:, 0]) == bytes(TOKEN[c] for c in t)
    assert win.quals[:, 0].tobytes() == rs.qual(0)[a:b]
    for j, q in enumerate(kept_qids, start=1):
        s, ql = oriented[q - 1]
        rev = q % 2 == 0
        assert bytes(win.bases[:, j]) == bytes(TOKEN[c + 32 if rev else c] for c in s[a:b]), (wid, j, q)
        assert win.quals[:, j].tobytes() == ql[a:b], (wid, j, q)


# ------------------------------------------------------------------------------------------ 1. exact copies
def test_exact_copies_tie_everywhere_and_support_nothing():
    """35 exact full-length copies, W 1024.  Every accuracy is 1.0 and no position is supported, so no copy has an agreement
    ratio and every ln-weighted score is 0: both stable sorts keep the input order.  Every window holds all 35 copies, keeps the
    first 30, has no supported position, and the consensus of a read without supported positions is the read itself."""
    rs, oriented = full_copies()
    T = po.Target(po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)]), 0, *rs.target_alns(0), W, 4)
    wins = T.windows()
    assert [w.wid for w in wins] == list(range(6))
    for w in wins:
        assert w.n_total_wins == 6 and w.n_alns == 30
        assert list(w.qids) == list(range(1, 36))
        assert len(w.supported) == 0 and len(w.sup_rows) == 0
        check_copy_columns(w, w.wid, rs, oriented, list(range(1, 31)))
    assert T.n_batches == 0
    assert T.consensus() == [rs.seq(0)]


# ------------------------------------------------------------------------------------------ 2. one substitution in ten copies
def test_one_substitution_ranks_the_exact_copies_first():
    """25 exact copies and 10 (qids 3, 6, ..., 30) with one substitution at SNP_POS.  The 36-column pileup of window 2 has 26
    target alleles and 10 others at SNP_POS (get_supported's threshold: int(36 * 0.1) = 3), so it is the one supported
    position, and after ranking still one in the 31 kept columns (25 + 1 target alleles, 5 others, threshold int(3.1) = 3).
    The agreement ratio of each copy is counted there alone: an exact copy has n = 1, d = 0, score 1 / 1 * ln 2; a SNP copy n = 0,
    d = 1, score 0.  So in every window the exact copies come first, then the SNP copies, each group in input order, and the
    kept SNP copies are the first five."""
    rs, oriented = full_copies(snp_qids=SNP_QIDS, snp_pos=SNP_POS)
    score = {q: 0.0 if q in SNP_QIDS else 1 / (1 + 0) * math.log(1 + 0 + 1) for q in range(1, 36)}  # n / (n + d) * ln(n + d + 1)
    want_ids = sorted(range(1, 36), key=lambda q: -score[q])  # stable, as sort_by_key(Reverse(score)) is
    assert want_ids == [q for q in range(1, 36) if q not in SNP_QIDS] + SNP_QIDS
    T = po.Target(po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)]), 0, *rs.target_alns(0), W, 4)
    for w in T.windows():
        assert w.n_alns == 30
        assert list(w.qids) == want_ids, w.wid
        check_copy_columns(w, w.wid, rs, oriented, want_ids[:30])
        if w.wid == SNP_POS // W:
            assert w.supported.tolist() == [[SNP_POS % W, 0]]
            assert w.sup_rows.tolist() == [SNP_POS % W]
        else:
            assert len(w.supported) == 0
    assert T.n_batches == 1


# ------------------------------------------------------------------------------------------ 3. window membership at the edges
# Copies of the target span [ts, te) on a TLEN = 5 * 1024 + 300 = 5420 target at W 1024, derived from src/windowing.rs:53-100:
#   zeroth_window_thresh z = (0.1 * 1024) as u32 = 102, nth_window_thresh = 5420 - 102 = 5318;
#   first = 0 if ts < z else ceil(ts / W); last = (te - 1) / W + 1 if te > 5318 else te / W; nothing if the target or query span
#   is shorter than W or last - first < 1.
EDGE_CASES = [
    # name,                     ts,     te,    windows
    ("start-at-2W",             2048,   5420,  [2, 3, 4, 5]),
    ("start-at-2W+1",           2049,   5420,  [3, 4, 5]),
    ("start-below-z",           50,     5420,  [0, 1, 2, 3, 4, 5]),
    ("start-at-z-1",            101,    5420,  [0, 1, 2, 3, 4, 5]),
    ("start-at-z",              102,    5420,  [1, 2, 3, 4, 5]),
    ("end-at-3W",               0,      3072,  [0, 1, 2]),
    ("end-at-3W+1",             0,      3073,  [0, 1, 2]),
    ("end-at-nth+1",            0,      5319,  [0, 1, 2, 3, 4, 5]),
    ("end-at-nth",              0,      5318,  [0, 1, 2, 3, 4]),
    ("end-at-nth-1",            0,      5317,  [0, 1, 2, 3, 4]),
    ("span-W-on-a-window",      3072,   4096,  [3]),
    ("span-W-across-a-boundary", 3000,  4024,  []),
    ("span-W-1",                3072,   4095,  []),
    ("interior-span-W+1",       1023,   2048,  [1]),
]


def edge_readset():
    rng = np.random.default_rng(23)
    target, tqual = random_bases(rng, TLEN), random_quals(rng, TLEN)
    copies = [(target[ts:te], random_quals(rng, te - ts), k % 2 == 1, ts, te, f"{te - ts}M".encode())
              for k, (_, ts, te, _) in enumerate(EDGE_CASES)]
    return build_readset(target, tqual, copies)


def hand_windows(ts, te, wins, cig_len):
    """One `{n}M` op: window k covers target [max(ts, kW), min(te, (k+1)W)); its query range and the op offsets are that range
    relative to ts (src/windowing.rs:149-194 cuts the op at each boundary it crosses)."""
    out = []
    for k in wins:
        a, b = max(ts, k * W), min(te, (k + 1) * W)
        out.append((k, a, a - ts, b - ts, 0, a - ts, cig_len, b - ts))
    return out


@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_window_membership_at_the_edges(case):
    name, ts, te, wins = case
    rs = edge_readset()
    k = [c[0] for c in EDGE_CASES].index(name)
    nw = (TLEN + W - 1) // W
    cig = rs.cigar(k)
    want = hand_windows(ts, te, wins, len(cig))
    assert po.extract_windows(rs.ovl9[k], cig, W, nw) == want
    ovl = api.Context.make_overlaps(rs.ovl9, rs.cigars, rs.cig_off)
    ows = api.extract_windows(ovl[k:k + 1], W, nw)
    got = [(int(o["window_idx"]), int(o["tstart"]), int(o["qstart"]), int(o["qend"]), int(o["cigar_start_idx"]),
            int(o["cigar_start_offset"]), int(o["cigar_end_idx"]), int(o["cigar_end_offset"])) for o in ows]
    assert got == want
    first, end = api.window_range(ovl[k:k + 1], W, nw)
    assert list(range(first, end)) == wins


def test_edge_copies_join_the_windows_derived_by_hand():
    """All the edge copies as one target: every window's ids are the copies that join it, in input order (all accuracies 1.0, no
    supported position), and its n_alns is their count."""
    rs = edge_readset()
    T = po.Target(po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)]), 0, *rs.target_alns(0), W, 4)
    for w in T.windows():
        members = [k + 1 for k, c in enumerate(EDGE_CASES) if w.wid in c[3]]
        assert list(w.qids) == members, w.wid
        assert w.n_alns == len(members) and len(w.supported) == 0
    assert [len([c for c in EDGE_CASES if k in c[3]]) for k in range(6)] == [7, 9, 9, 9, 8, 6]


# ------------------------------------------------------------------------------------------ 4. the synthetic profiles
def op_lengths(rs) -> np.ndarray:
    return np.array([int(n) for n in re.findall(rb"(\d+)[MID]", rs.cigars.tobytes())], np.int64)


def test_low_error_profiles_make_long_ops():
    """The `exact` and `q30` profiles of tools/synth: errors only at haplotype differences and long deletions (exact), or at
    ~1.2e-3 per base (q30), so their CIGARs carry ops thousands of bases long, where r10's median op is a few dozen bases."""
    ops = {p: op_lengths(helpers.small_readset(n_reads=30, mean_len=12000, seed=4, profile=p)) for p in ("exact", "q30", "r10")}
    assert (ops["exact"] >= 10000).any() and (ops["q30"] >= 1024).sum() > 10
    assert np.median(ops["exact"]) > 10 * np.median(ops["r10"]) and np.median(ops["q30"]) > 4 * np.median(ops["r10"])


# sha256 of (seqs, quals, off, ovl9, cigars) of synth.generate(60, 8000, profile=p, seed=s, coverage=20.0): the sets every
# existing test draws from must not change when a profile is added.
PINNED = {
    ("r10", 1): "153e669c23215fc56dc91539ca7c5ec7a9496ef6099faafcf5e43d9eb7e1bf68",
    ("r10", 7): "22030e32578a7c3b8cc52fb56fa2105cb954f46c4d53ad1dee80e2c731ec2c15",
    ("r9", 2): "ec6bf254f8e2383002910d7c13c31b9b4ebd111a4d74e2a53724b2e89451845b",
    ("r9", 5): "945f4d809a09dabcee323dfb9bf1914fa1431db44fe53de87aa714aa8d9dd395",
}


def readset_digest(rs) -> str:
    h = hashlib.sha256()
    for a in (rs.seqs, rs.quals, rs.off, rs.ovl9, rs.cig_off, rs.cigars):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("profile,seed", list(PINNED))
def test_existing_profiles_generate_the_same_sets(profile, seed):
    assert readset_digest(synth.generate(60, 8000, profile=profile, seed=seed, coverage=20.0)) == PINNED[(profile, seed)]
