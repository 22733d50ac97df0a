"""The overlap oracle (tests/overlap_oracle.cpp), which the device must equal, checked on its own: hash64 against an independent
numpy restatement, minimizer selection and chaining on hand-made inputs, the occurrence threshold, and the whole definition against
the synthetic generator's true overlaps."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import overlap_oracle as oo  # noqa: E402
from tools import synth  # noqa: E402

BASES = np.frombuffer(b"ACGT", np.uint8)


def np_hash64(key, mask):
    """Thomas Wang's 64-bit integer hash, masked to 2k bits, in numpy's wrapping uint64 arithmetic."""
    with np.errstate(over="ignore"):
        key, m = np.uint64(key), np.uint64(mask)
        key = (~key + (key << np.uint64(21))) & m
        key = key ^ (key >> np.uint64(24))
        key = (key + (key << np.uint64(3)) + (key << np.uint64(8))) & m
        key = key ^ (key >> np.uint64(14))
        key = (key + (key << np.uint64(2)) + (key << np.uint64(4))) & m
        key = key ^ (key >> np.uint64(28))
        key = (key + (key << np.uint64(31))) & m
    return int(key)


def py_minimizers(seq: bytes, k: int, w: int):
    """The sketch of DESIGN.md §13, written from the definition: [(h, i, z)]"""
    c = [b"ACGT".index(x) for x in seq]
    mask = (1 << 2 * k) - 1
    kms = []
    for i in range(k - 1, len(c)):
        f = r = 0
        for u in range(k):
            f = f << 2 | c[i - k + 1 + u]
            r = r << 2 | (c[i - u] ^ 3)
        if f != r:
            kms.append((np_hash64(min(f, r), mask), i, int(r < f)))
    sel = []
    for e in range(w - 1, len(kms)):
        best = min(kms[e - w + 1:e + 1], key=lambda t: (t[0], t[1]))
        if not sel or sel[-1][1] != best[1]:
            sel.append(best)
    return sel


def rnd(rng, n) -> bytes:
    return BASES[rng.integers(0, 4, n)].tobytes()


def revcomp(s: bytes) -> bytes:
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


# ---- hash and sketch
@pytest.mark.parametrize("k", [12, 15, 25, 28])
def test_hash64_known_answers(k):
    mask = (1 << 2 * k) - 1
    rng = np.random.default_rng(k)
    keys = [0, 1, 2, 3, mask, mask - 1, 0x123456789 & mask] + [int(x) & mask for x in rng.integers(0, 1 << 62, 40, dtype=np.int64)]
    for key in keys:
        assert oo.hash64(key, mask) == np_hash64(key, mask), key
    assert oo.hash64(0, (1 << 50) - 1) == np_hash64(0, (1 << 50) - 1)


@pytest.mark.parametrize("k,key,h", [(25, 0x0, 0x1df3e729bc06f), (25, 0x1, 0x27c69b794f8ce), (25, 0x123456789abc, 0x20879929c98b8),
                                       (15, 0x2aaaaaaa, 0x304a3cb6), (28, (1 << 56) - 1, 0xfa4d157df516b7)])
def test_hash64_fixed_values(k, key, h):
    # values of np_hash64, kept so that a change to both restatements at once is seen
    assert oo.hash64(key, (1 << 2 * k) - 1) == h == np_hash64(key, (1 << 2 * k) - 1)


def test_hash64_is_a_bijection_on_the_masked_domain():
    mask = (1 << 24) - 1
    assert len({oo.hash64(x, mask) for x in range(4096)}) == 4096


@pytest.mark.parametrize("k,w", [(25, 17), (15, 10), (12, 2), (28, 32), (16, 5)])
def test_sketch_matches_the_definition_on_random_reads(k, w):
    rng = np.random.default_rng(k * 100 + w)
    for n in (k + w - 2, k + w - 1, k + w, 300, 701):
        s = rnd(rng, n)
        h, pos, z = oo.sketch(s, k, w)
        assert list(zip(h.tolist(), pos.tolist(), z.tolist())) == py_minimizers(s, k, w), n


def test_read_lengths_at_the_first_window():
    rng = np.random.default_rng(2)
    k, w = 25, 17
    s = rnd(rng, k + w - 1)
    assert len(oo.sketch(s, k, w)[0]) == 1
    assert len(oo.sketch(s[:-1], k, w)[0]) == 0
    assert len(oo.sketch(s[:k - 1], k, w)[0]) == 0


def test_ties_inside_a_window_take_the_leftmost():
    # every k-mer of a homopolymer is the same: each window ties throughout and selects its leftmost k-mer
    k, w = 15, 10
    h, pos, z = oo.sketch(b"A" * 60, k, w)
    assert pos.tolist() == list(range(k - 1, 60 - w + 1))
    assert len(set(h.tolist())) == 1 and not np.any(z)
    rng = np.random.default_rng(5)
    km = rnd(rng, k)
    s = rnd(rng, 20) + km + rnd(rng, 3) + km + rnd(rng, 40)
    h, pos, z = oo.sketch(s, k, w)
    assert list(zip(h.tolist(), pos.tolist(), z.tolist())) == py_minimizers(s, k, w)


def test_palindromic_kmer_is_skipped_at_even_k():
    k, w = 16, 2
    half = b"ACGTTGCAACGG"[:8]
    pal = half + revcomp(half)  # its own reverse complement
    assert pal == revcomp(pal)
    s = b"A" * 3 + pal + b"C" * 3
    mini = py_minimizers(s, k, w)
    assert all(i != 3 + k - 1 for _, i, _ in mini)
    h, pos, z = oo.sketch(s, k, w)
    assert 3 + k - 1 not in pos.tolist()
    assert list(zip(h.tolist(), pos.tolist(), z.tolist())) == mini


# ---- chaining
K = 15


def ch(x, y, **kw):
    kw.setdefault("k", K)
    return oo.chain(x, y, **kw)


def test_chain_on_a_diagonal():
    c = ch([100, 120, 140, 160], [10, 30, 50, 70])
    assert c["n_anchors"] == 4 and c["first"] == 0 and c["last"] == 3
    assert c["score"] == K + 3 * K
    assert c["covered"] == 4 * K  # spacing 20 > k: disjoint k-mers
    c = ch([100, 105, 110], [10, 15, 20])
    assert c["score"] == K + 5 + 5 and c["covered"] == 10 + K  # overlapping k-mers: their union


def test_chain_needs_positive_dx_and_dy():
    assert ch([100, 100], [10, 30])["n_anchors"] == 1  # dx == 0
    assert ch([100, 120], [30, 30])["n_anchors"] == 1  # dy == 0
    assert ch([100, 120], [40, 30])["n_anchors"] == 1  # dy < 0


def test_chain_gap_and_band_limits():
    assert ch([0, 5000], [0, 5000])["n_anchors"] == 2
    assert ch([0, 5001], [0, 5001])["n_anchors"] == 1  # dx > max_gap stops the scan
    assert ch([0, 4900], [0, 5001], bandwidth=200)["n_anchors"] == 1  # dy > max_gap
    assert ch([0, 100], [0, 110], bandwidth=10)["n_anchors"] == 2  # |dx - dy| == bandwidth
    assert ch([0, 100], [0, 111], bandwidth=10)["n_anchors"] == 1
    # gap cost g(l) = floor(k l / 100) + floor(floor(log2 l) / 2): g(10) = 1 + 1
    assert ch([0, 100], [0, 110], bandwidth=10)["score"] == K + K - 2


def test_chain_max_iter():
    x, y = [0, 10, 11, 30], [0, 10, 900, 30]
    c1 = ch(x, y, max_iter=1)  # anchor 3 sees only anchor 2, which it cannot follow
    c2 = ch(x, y, max_iter=2)
    assert c1["n_anchors"] == 2 and c1["last"] == 1
    assert c2["n_anchors"] == 3 and c2["last"] == 3


def test_chain_ties_strict_and_closest():
    # anchor 2 follows anchor 0 or anchor 1 for the same score: the closest predecessor, 1, wins
    c = ch([0, 50, 100], [50, 0, 100])
    assert c["n_anchors"] == 2 and c["first"] == 1 and c["score"] == K + K - (K * 50 // 100 + 5 // 2)
    # a candidate scoring exactly k does not replace the start value: g(85) = 12 + 3 = k
    c = ch([0, 100], [0, 185])
    assert c["n_anchors"] == 1 and c["last"] == 0 and c["score"] == K
    c = ch([0, 100], [0, 179])  # g(79) = 11 + 3
    assert c["n_anchors"] == 2 and c["score"] == K + 1
    # the end is the first anchor of the largest score
    c = ch([0, 1000], [0, 3000])
    assert c["last"] == 0 and c["score"] == K


def test_min_score_and_min_anchors_at_their_boundaries():
    rng = np.random.default_rng(7)
    g = rnd(rng, 9000)
    seqs = [g[:6000], g[2000:9000]]
    r = oo.find(seqs, [0, 1], min_score=100)["records"]
    assert len(r) == 2
    score, na = int(r[0][9]), int(r[0][10])
    assert len(oo.find(seqs, [0], min_score=score)["records"]) == 1
    assert len(oo.find(seqs, [0], min_score=score + 1)["records"]) == 0
    assert len(oo.find(seqs, [0], min_score=100, min_anchors=na)["records"]) == 1
    assert len(oo.find(seqs, [0], min_score=100, min_anchors=na + 1)["records"]) == 0


@pytest.mark.parametrize("fwd,rev,strand", [(4000, 2000, 0), (2000, 4000, 1)])
def test_the_better_strand_of_a_pair(fwd, rev, strand):
    rng = np.random.default_rng(11)
    t = rnd(rng, 12000)
    q = t[:fwd] + rnd(rng, 500) + revcomp(t[6000:6000 + rev])
    r = oo.find([t, q], [0], min_score=500)["records"]
    assert len(r) == 1 and int(r[0][4]) == strand


# ---- occurrence threshold
def test_occurrence_threshold():
    occ = np.array([1] * 990 + [50] * 10, np.uint32)
    # 1000 distinct hashes; rank floor(0.995 * 1000) = 995 -> occ 50
    assert oo.max_occ(occ, 5000, 10) == 50
    assert oo.max_occ(occ, 20000, 10) == 10  # rank 980 -> occ 1, below the floor
    assert oo.max_occ(occ, 20000, 1) == 1
    occ2 = np.arange(1, 201, dtype=np.uint32)
    assert oo.max_occ(occ2, 5000, 10) == 200  # rank floor(0.995 * 200) = 199: the last
    assert oo.max_occ(occ2, 100000, 10) == 181
    assert oo.max_occ(np.zeros(0, np.uint32), 5000, 10) == 10


# ---- against the generator's truth
def test_oracle_against_synthetic_truth():
    rs = synth.generate(120, 12000, profile="r10", seed=5, coverage=20.0, min_ovl=1)
    seqs = [rs.seq(i) for i in range(rs.n)]
    got = oo.find(seqs, list(range(rs.n)))["records"]
    truth = {}
    for q, _, _, _, st, t, _, ts, te in rs.ovl9.astype(np.int64):
        truth[(int(t), int(q))] = (int(st), int(ts), int(te))
    assert len(got) > 1000
    for r in got:
        q, t, s, ts, te = int(r[0]), int(r[5]), int(r[4]), int(r[7]), int(r[8])
        assert (t, q) in truth, (t, q)
        st, a, b = truth[(t, q)]
        assert s == st and a <= ts and te <= b
    found = {(int(r[5]), int(r[0])) for r in got}
    big = [p for p, v in truth.items() if v[2] - v[1] >= 5000]
    assert len(big) > 1000
    assert sum(p in found for p in big) >= 0.99 * len(big)
