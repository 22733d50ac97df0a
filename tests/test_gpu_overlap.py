"""hb_find_overlaps on the device against the overlap oracle (tests/overlap_oracle.cpp): every record of hb_find_fetch (all
hb_overlap fields, score, n_anchors, covered) byte for byte and in order, and the shape's counts, on synthetic R10 / R9 sets and
on chosen edge cases."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import overlap_oracle as oo  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu

BASES = np.frombuffer(b"ACGT", np.uint8)
LOW = dict(k=15, w=10, min_score=500)


def arrays(seqs):
    """(seqs, quals, off) of a read list, as Context.upload_reads takes them."""
    off = np.zeros(len(seqs) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    cat = np.frombuffer(b"".join(seqs), np.uint8).copy()
    return cat, np.full(len(cat), ord("5"), np.uint8), off


def context(seqs, store=False, chunk_bases=None, monkeypatch=None):
    from herro_b200.api import Context, ReadStore
    if chunk_bases is not None:
        monkeypatch.setenv("HERRO_B200_OVL_CHUNK_BASES", str(chunk_bases))
    ctx = Context(None)
    if chunk_bases is not None:
        monkeypatch.delenv("HERRO_B200_OVL_CHUNK_BASES")
    if store:
        st = ReadStore(*arrays(seqs))
        ctx.attach_read_store(st)
        ctx._test_store = st
    else:
        ctx.upload_reads(*arrays(seqs))
    return ctx


def records(got):
    o = got["overlaps"]
    cols = [o[f].astype(np.uint32) for f in oo.RECORD_FIELDS[:9]] + [got["score"], got["n_anchors"], got["covered"]]
    return np.stack(cols, 1) if len(o) else np.zeros((0, 12), np.uint32)


def check(ctx, seqs, targets, **kw):
    got = ctx.find_overlaps(targets, **kw)
    want = oo.find(seqs, targets, **kw)
    assert np.array_equal(records(got), want["records"])
    assert not np.any(got["overlaps"]["cigar"]) and not np.any(got["overlaps"]["cigar_len"])
    sh = got["shape"]
    for f in ("max_occ", "n_filtered_hashes", "index_entries", "query_minimizers", "anchors"):
        assert sh[f] == want[f], f
    assert sh["n_targets"] == len(targets) and sh["n_overlaps"] == len(want["records"])
    return got, want


@pytest.fixture(scope="module", params=["r10", "r9"])
def synth_set(request):
    rs = synth.generate(60, 9000, profile=request.param, seed=9, coverage=12.0)
    return rs, [rs.seq(i) for i in range(rs.n)], request.param


@pytest.mark.parametrize("kw", [{}, LOW], ids=["defaults", "k15w10"])
def test_synthetic_sets_match_the_oracle(synth_set, kw):
    rs, seqs, profile = synth_set
    ctx = context(seqs)
    got, want = check(ctx, seqs, list(range(rs.n)), **kw)
    if kw or profile == "r10":  # at k = 25, R9's error rate leaves too few exact 25-mers on 9 kb reads for a chain of 2 500
        assert len(want["records"]) > 50
        assert set(want["records"][:, 4].tolist()) == {0, 1}


def test_target_subsets_match_the_oracle(synth_set):
    rs, seqs, _ = synth_set
    ctx = context(seqs)
    rng = np.random.default_rng(3)
    perm = rng.permutation(rs.n)
    for part in (perm[:7], perm[7:30], perm[30:]):
        check(ctx, seqs, [int(t) for t in part])


def test_frequency_filter_decides():
    rs = synth.generate(50, 8000, profile="r10", seed=4, coverage=10.0)
    seqs = [rs.seq(i) for i in range(rs.n)]
    rng = np.random.default_rng(1)
    planted = BASES[rng.integers(0, 4, 600)].tobytes()
    seqs = [s[:3000] + planted + s[3000:] if i % 2 == 0 else s for i, s in enumerate(seqs)]
    ctx = context(seqs)
    got, want = check(ctx, seqs, list(range(len(seqs))))
    assert want["n_filtered_hashes"] > 0 and want["max_occ"] < 25


def test_chunks_and_host_store_change_nothing(synth_set, monkeypatch):
    rs, seqs, _ = synth_set
    targets = list(range(0, rs.n, 2))
    base = records(context(seqs).find_overlaps(targets, **LOW))
    assert len(base)
    for store, chunk in ((False, 20000), (True, None), (True, 1)):
        got = context(seqs, store=store, chunk_bases=chunk, monkeypatch=monkeypatch).find_overlaps(targets, **LOW)
        assert np.array_equal(records(got), base), (store, chunk)


def revcomp(s: bytes) -> bytes:
    return s[::-1].translate(bytes.maketrans(b"ACGT", b"TGCA"))


def test_edge_cases():
    rng = np.random.default_rng(8)
    rnd = lambda n: BASES[rng.integers(0, 4, n)].tobytes()  # noqa: E731
    g = rnd(40000)
    seqs = [g[0:12000],             # 0: first read of the store
            rnd(9000),              # 1: shares nothing: a target with no overlaps
            revcomp(g[4000:15000]),  # 2: the reverse complement of part of read 0
            g[2000:2030],           # 3: fewer than w k-mers: no minimizer
            g[18000:38000],         # 4, 5: two identical 20 kb reads
            g[18000:38000],
            g[8000:20000]]          # 6: last read of the store
    ctx = context(seqs)
    got, want = check(ctx, seqs, list(range(len(seqs))))
    rec = {(int(r[5]), int(r[0])): r for r in want["records"]}
    assert not any(t == 1 or q == 1 for t, q in rec)
    assert not any(t == 3 or q == 3 for t, q in rec)
    assert int(rec[(0, 2)][4]) == 1 and int(rec[(2, 0)][4]) == 1
    assert int(rec[(4, 5)][10]) > 1000  # one group of many warp steps
    assert (0, 6) in rec and (6, 0) in rec
    for targets in ([0], [6], [1], [3, 4]):
        check(ctx, seqs, targets)


def test_found_overlaps_align(synth_set):
    rs, seqs, _ = synth_set
    ctx = context(seqs)
    got = ctx.find_overlaps(list(range(rs.n)), **LOW)
    aln = ctx.align(got["overlaps"])
    assert len(aln["status"]) == len(got["overlaps"]) > 0
    assert not np.any(aln["status"] < 0)


def test_bad_arguments_run_nothing(synth_set):
    from herro_b200.api import HerroError
    rs, seqs, _ = synth_set
    ctx = context(seqs)
    for targets, kw, code in (([rs.n], {}, -4), ([1, 1], {}, -4), ([0], dict(k=11), -1), ([0], dict(k=29), -1),
                              ([0], dict(w=33), -1), ([0], dict(top_frac_ppm=1000000), -1), ([], {}, -1)):
        with pytest.raises(HerroError) as e:
            ctx.find_overlaps(targets, **kw)
        assert e.value.code == code, (targets, kw)


def test_counters_are_the_calls_own(synth_set):
    rs, seqs, _ = synth_set
    ctx = context(seqs, store=True)
    targets = list(range(rs.n))
    ctx.reset_stats()
    ctx.find_overlaps(targets)
    s1 = {k: v for k, v in ctx.stats().items() if not isinstance(v, (dict, list))}
    nonzero = {k for k, v in s1.items() if v}
    assert {"kernel_launches", "h2d_bytes", "d2h_bytes"} <= nonzero <= {"kernel_launches", "h2d_bytes", "d2h_bytes", "host_allocs",
                                                                         "ms_host_alloc"}
    ctx.find_overlaps(targets)
    s2 = {k: v for k, v in ctx.stats().items() if not isinstance(v, (dict, list))}
    for f in ("kernel_launches", "h2d_bytes", "d2h_bytes"):
        assert s2[f] == 2 * s1[f], f
