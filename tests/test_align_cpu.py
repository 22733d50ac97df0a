"""The alignment oracle of hb_align_overlaps (tests/align_oracle.cpp) against the reference's fix_cigar known answers, an independent
full-matrix two-piece Gotoh, and the generator's true alignments."""
import json
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import align_oracle as ao  # noqa: E402
from tools import synth  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fix_cigar_known_answers.json")
NEG = -(10 ** 9)


def gap(l):
    return min(4 + 2 * l, 24 + l) if l else 0


def ops(cigar: bytes):
    return [(int(n), k) for n, k in re.findall(rb"(\d+)([MID])", cigar)]


def rescore(T, Q, cigar: bytes, t0=0, q0=0):
    """Score of a CIGAR over T[t0:] / Q[q0:]; also returns the target and query bases it spans."""
    s, t, q = 0, t0, q0
    for n, k in ops(cigar):
        if k == b"M"[0:1]:
            s += int(np.sum(np.where(T[t:t + n] == Q[q:q + n], 2, -4)))
            t += n
            q += n
        elif k == b"I":
            s -= gap(n)
            q += n
        else:
            s -= gap(n)
            t += n
    return s, t - t0, q - q0


def gotoh(T, Q):
    """Full-matrix two-piece affine global alignment score (match 2, mismatch -4, gap min(4 + 2l, 24 + l)), row by row in numpy."""
    n, m = len(T), len(Q)
    H = np.full(m + 1, NEG, np.int64)
    H[0] = 0
    j = np.arange(m + 1)
    H[1:] = -np.minimum(4 + 2 * j[1:], 24 + j[1:])
    F1 = np.full(m + 1, NEG, np.int64)
    F2 = np.full(m + 1, NEG, np.int64)
    for i in range(1, n + 1):
        F1 = np.maximum(H - 6, F1 - 2)
        F2 = np.maximum(H - 25, F2 - 1)
        Hn = np.full(m + 1, NEG, np.int64)
        Hn[1:] = H[:-1] + np.where(Q == T[i - 1], 2, -4)
        Hn = np.maximum(Hn, np.maximum(F1, F2))
        E1 = np.full(m + 1, NEG, np.int64)
        E2 = np.full(m + 1, NEG, np.int64)
        for x in range(1, m + 1):
            E1[x] = max(Hn[x - 1] - 6, E1[x - 1] - 2)
            E2[x] = max(Hn[x - 1] - 25, E2[x - 1] - 1)
            Hn[x] = max(Hn[x], E1[x], E2[x])
        H = Hn
    return int(H[m])


def test_fix_cigar_known_answers():
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) == 3
    for c in cases:
        got, ts, qs = ao.fix_cigar(c["target"].encode(), c["query"].encode(), c["cigar_in"].encode())
        assert got.decode() == c["cigar_out"] and (ts, qs) == (0, 0)


def test_fix_cigar_drops_a_leading_gap():
    assert ao.fix_cigar(b"AACGT", b"ACGT", b"1D4M") == (b"4M", 1, 0)
    assert ao.fix_cigar(b"ACGT", b"TTACGT", b"0M2I4M") == (b"4M", 0, 2)


def mutate(rng, s, rate):
    out = []
    for b in s:
        r = rng.random()
        if r < rate:
            out.append(int(rng.integers(4)))
        elif r < 2 * rate:
            continue
        elif r < 3 * rate:
            out += [int(b), int(rng.integers(4))]
        else:
            out.append(int(b))
    return np.array(out or [0], np.uint8)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_full_matrix_gotoh(seed):
    rng = np.random.default_rng(seed)
    done = 0
    while done < 25:
        n = int(rng.integers(1, 41))
        T = rng.integers(0, 4, n).astype(np.uint8)
        Q = mutate(rng, T, 0.1) if rng.random() < 0.7 else rng.integers(0, 4, int(rng.integers(1, 41))).astype(np.uint8)
        m = len(Q)
        if m > 2 * n or n > 2 * m:
            continue
        r = ao.align_codes(T, Q, 64)
        assert r["score"] == gotoh(T, Q)
        assert not r["edge"]
        c = r["cigar"]
        assert c[-1:] == b"M" and re.fullmatch(rb"(\d+M)(\d+[ID]\d+M)*", c)
        s, tl, ql = rescore(T, Q, c, r["lead_d"], r["lead_i"])
        assert (tl, ql) == (n - r["lead_d"] - r["trail_d"], m - r["lead_i"] - r["trail_i"])
        ends = gap(r["lead_d"]) + gap(r["lead_i"]) + gap(r["trail_d"]) + gap(r["trail_i"])
        assert s - ends == r["score"]
        want_matches = sum(int(np.sum(T[t:t + k] == Q[q:q + k])) for t, q, k in _m_blocks(c, r["lead_d"], r["lead_i"]))
        assert r["matches"] == want_matches
        done += 1


def _m_blocks(cigar, t, q):
    for n, k in ops(cigar):
        if k == b"M":
            yield t, q, n
            t += n
            q += n
        elif k == b"I":
            q += n
        else:
            t += n


def path_offset(cigar: bytes, n, m):
    """Largest |j - c(i)| over the cells of a CIGAR's path (c(i) = floor(i m / n))."""
    i = j = 0
    worst = 0
    for k, op in ops(cigar):
        for _ in range(k):
            if op == b"M":
                i += 1
                j += 1
            elif op == b"I":
                j += 1
            else:
                i += 1
            worst = max(worst, abs(j - (i * m) // n))
    return worst


@pytest.mark.parametrize("profile", ["r10", "r9"])
def test_oracle_at_least_the_true_alignment(profile):
    rs = synth.generate(24, 3000, profile=profile, seed=5, coverage=12.0)
    w = 128
    checked = 0
    for a in range(min(len(rs.ovl9), 60)):
        q, ql, qs, qe, st, t, tl, ts, te = (int(x) for x in rs.ovl9[a])
        cig = rs.cigar(a)
        n, m = te - ts, qe - qs
        if m > 2 * n or n > 2 * m or path_offset(cig, n, m) >= w - 1:
            continue
        T = ao.codes(rs.seq(t))[ts:te]
        Q = ao.oriented_query(ao.codes(rs.seq(q)), qs, qe, st)
        true_score, tl_, ql_ = rescore(T, Q, cig)
        assert (tl_, ql_) == (n, m)
        r = ao.align_codes(T, Q, w)
        assert r["score"] >= true_score
        checked += 1
    assert checked >= 20
