"""No-GPU checks of hb_consensus_batch's ground: the oracle's consensus() on caller-supplied windows equals its consensus() of the
fixture's targets, hand-derived windows pin each rule the header states (the GPU test runs the same cases through the library), the
`herro features` + `predict` reader rebuilds the oracle's ConsensusWindows, and the entry point is declared, exported and guarded."""
import os
import re
import shutil

import numpy as np
import pytest

import consensus_oracle
import helpers  # noqa: F401  (puts the repository root on sys.path)
from herro_b200 import api, hostio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP = os.path.join(ROOT, "tests", "golden", "features_dump")
A, C, G, T, GAP, a_, c_, g_, t_, HASH, DOT = range(11)
NAN = float("nan")


def win(rows, n_alns, sup=(), logits=()):
    """A window from token rows (each padded to 31 columns with '.'), its supported (pos, ins) list and their logits."""
    b = np.full((len(rows), 31), DOT, np.uint8)
    for r, row in enumerate(rows):
        b[r, :len(row)] = row
    return (b, n_alns, np.array(sup, np.uint32).reshape(-1, 2), np.array(logits, np.float32).reshape(-1, 5))


def onehot(k):
    x = [0.0] * 5
    x[k] = 9.0
    return x


PLAIN = win([[A, A, C], [C, A, A], [G, T, T], [A, C, G], [GAP, GAP, GAP], [G, C, C, A, A], [c_, c_, A]], 2)
# HAND[name] = (reads, expected segments per read); a read is a list of windows in wid order.  "panic" = HB_ERR_INPUT at the
# (read, window, row, column) given.
HAND = {
    # vote: majority, target column below 2, '*' emits nothing, the tie rule with the target column, lower-case folded;
    # columns past n_alns are not counted ([G, C, C, A, A] at n_alns 2 counts G, C, C)
    "vote": ([[PLAIN]], [[b"AAT" + b"A" + b"C" + b"C"]]),
    "vote-ties": ([[win([[A, C, C, A], [G, C, C, A, A], [T, A, A, C, C]], 4)]], [[b"A" + b"A" + b"A"]]),
    # argmax: last max wins, NaN greatest (last NaN wins), -0 == +0, class 4 emits nothing
    "argmax": ([[win([[A, A, A]] * 5, 2, [(0, 0), (1, 0), (2, 0), (3, 0), (4, 0)],
                     [[1, 3, 3, 0, 0], [NAN, 5, 0, 0, 0], [0, NAN, 1, NAN, 0], [-0.0, 0.0, -1, -1, -1], [0, 0, 0, 0, 1]])]],
               [[b"GATC"]]),
    # duplicate entry: the later one wins; an entry that matches no row is ignored
    "duplicate": ([[win([[A, A, A], [A, A, A]], 2, [(0, 0), (7, 0), (0, 0)], [onehot(G), onehot(T), onehot(C)])]], [[b"CA"]]),
    # unsorted entries
    "unsorted": ([[win([[A, A, A], [GAP, A, A], [A, A, A]], 2, [(1, 0), (0, 1), (0, 0)], [onehot(T), onehot(G), onehot(C)])]],
                 [[b"CGT"]]),
    # leading '*' rows have pos 65535
    "leading-gaps": ([[win([[GAP, GAP, GAP], [GAP, GAP, GAP], [A, A, A]], 2, [(65535, 2)], [onehot(G)])]], [[b"GA"]]),
    # a run of 256 '*' rows: ins wraps to 0, so the 256th '*' row shares the key (0, 0) with row 0
    "ins-wrap": ([[win([[A, A, A]] + [[GAP, GAP, GAP]] * 256, 2, [(0, 0), (0, 5)], [onehot(T), onehot(C)])]], [[b"TCT"]]),
    # tokens >= 11 past n_alns are never read
    "ignored-columns": ([[win([[A, A, C, 200, 11, 255]], 2)]], [[b"A"]]),
    # a window with n_alns < 2 inside the kept range ends the segment; the ones outside it are trimmed and never read (their
    # bytes would panic)
    "split-trim": ([[win([[DOT, 200]], 0), win([[C, C, C]], 2), win([[200, 200, 200]], 1), win([[G, G, G], [T, T, T]], 3),
                     win([[DOT]], 1)]], [[b"C", b"GT"]]),
    # None (no window with n_alns > 1) and Some(empty) both give no record; reads are independent
    "none-and-empty": ([[win([[A, A, A]], 1), win([[A]], 0)], [win([[GAP, GAP, GAP]], 2)], [], [win([[T, T, T]], 30)]],
                       [[], [], [], [b"T"]]),
    # n_alns 30 reads all 31 columns
    "n_alns-30": ([[win([[A] + [C] * 30], 30)]], [[b"C"]]),
    # panics: '.' in column 0 of a voting row; a token >= 11 in a counted column.  The first in row-major order is named.
    "panic-dot": ([[win([[A, A, A]], 2)], [win([[A, A, A], [DOT, A, A]], 2)]], ("panic", (1, 0, 1, 0))),
    "panic-11": ([[win([[A, A, 11]], 2)]], ("panic", (0, 0, 0, 2))),
    "panic-first": ([[win([[A, A, A], [DOT, A, 12], [A, 13, A]], 2)]], ("panic", (0, 0, 1, 0))),
    # the same bytes at a supported row, or in an n_alns < 2 window, are fine
    "no-panic-supported": ([[win([[A, A, A], [DOT, A, 12]], 2, [(1, 0)], [onehot(T)])]], [[b"AT"]]),
    "no-panic-skipped": ([[win([[A, A, A]], 2), win([[DOT, 12, 12]], 1), win([[C, C, C]], 2)]], [[b"A", b"C"]]),
}


def oracle_segments(reads):
    return consensus_oracle.consensus_windows(reads)


@pytest.mark.parametrize("name", list(HAND))
def test_hand_derived_windows_pin_the_rules(name):
    reads, want = HAND[name]
    if isinstance(want, tuple):
        with pytest.raises(consensus_oracle.OraclePanic):
            oracle_segments(reads)
        return
    assert oracle_segments(reads) == want


def test_oracle_on_caller_windows_equals_its_consensus():
    """The oracle's consensus() on its own windows and logits, passed as caller arrays (consensus_oracle), gives ho_consensus for every
    target of the golden dump."""
    from oracle import pyoracle as po
    from tools import make_feature_fixture as mf
    rs = mf.readset()
    reads = po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)])
    rng = np.random.default_rng(12)
    n_seg = 0
    for t in mf.TARGETS:
        ovl, cigs = rs.target_alns(t)
        Tg = po.Target(reads, t, ovl, cigs, mf.W, 4)
        wins = Tg.windows()
        for trial in range(3):
            mine = []
            for i, w in enumerate(wins):
                n = len(w.supported)
                bl = rng.normal(size=(n, 5)).astype(np.float32)
                if trial == 2 and n:
                    bl[:, 4] = bl.max(axis=1) + 1  # every supported row emits nothing
                Tg.set_logits(i, np.zeros(n, np.float32), bl)
                mine.append((w.wid, (w.bases, w.n_alns, w.supported, bl)))
            want = Tg.consensus()
            got = consensus_oracle.consensus_windows([[x for _, x in sorted(mine, key=lambda p: p[0])]])[0]
            assert got == (want or []), (t, trial)
            n_seg += len(got)
    assert n_seg >= 3


def write_logits(tmp, rng):
    """Random logits for every window with supported positions of the dump, as `predict` lays them out."""
    out = {}
    for d in hostio.feature_reads(DUMP):
        read = os.path.basename(d)
        os.makedirs(os.path.join(tmp, read), exist_ok=True)
        for f in os.listdir(d):
            if f.endswith(".supported.npy"):
                n = len(np.load(os.path.join(d, f)))
                if n:
                    wid = int(f.split(".")[0])
                    bl = rng.normal(size=(n, 5)).astype(np.float32)
                    np.save(os.path.join(tmp, read, f"{wid}.bases_logits.npy"), bl)
                    out[(read, wid)] = bl
    return out


def test_reader_rebuilds_the_oracle_windows(tmp_path):
    from oracle import pyoracle as po
    from tools import make_feature_fixture as mf
    rs = mf.readset()
    reads = po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)])
    logits = write_logits(str(tmp_path), np.random.default_rng(3))
    n_win = 0
    for t in mf.TARGETS:
        ovl, cigs = rs.target_alns(t)
        want = sorted(po.Target(reads, t, ovl, cigs, mf.W, 4).windows(), key=lambda w: w.wid)
        got = hostio.read_consensus_windows(os.path.join(DUMP, rs.ids[t]), str(tmp_path / rs.ids[t]))
        assert [g.wid for g in got] == [w.wid for w in want] == list(range(len(want)))
        for g, w in zip(got, want):
            assert g.bases.dtype == np.uint8 and np.array_equal(g.bases, w.bases)
            assert g.n_alns == w.n_alns
            assert np.array_equal(g.supported, w.supported.reshape(-1, 2))
            assert g.bases_logits.shape == (len(w.supported), 5)
            if len(w.supported):
                assert np.array_equal(g.bases_logits, logits[(rs.ids[t], w.wid)])
            n_win += 1
    assert n_win >= 9


def test_reader_refuses_gaps_and_missing_logits(tmp_path):
    logits = str(tmp_path / "logits")
    write_logits(logits, np.random.default_rng(1))
    src = hostio.feature_reads(DUMP)[0]
    read = os.path.basename(src)
    d = str(tmp_path / "features" / read)
    shutil.copytree(src, d)
    assert len(hostio.read_consensus_windows(d, os.path.join(logits, read))) == 4
    for f in os.listdir(d):
        if f.startswith("1."):
            os.remove(os.path.join(d, f))
    with pytest.raises(ValueError, match="window 1 is missing"):
        hostio.read_consensus_windows(d, os.path.join(logits, read))
    shutil.rmtree(d)
    shutil.copytree(src, d)
    victim = sorted(f for f in os.listdir(os.path.join(logits, read)))[0]
    os.remove(os.path.join(logits, read, victim))
    with pytest.raises(ValueError, match="bases_logits.npy is missing"):
        hostio.read_consensus_windows(d, os.path.join(logits, read))


def test_consensus_batch_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "herro_b200.h")).read()
    assert re.search(r"\bint hb_consensus_batch\s*\(", hdr)
    assert re.search(r"#define HB_CONS_DEVICE_PTRS 1u", hdr)
    assert "hb_consensus_batch" in api.EXPORTED_SYMBOLS
    assert api.HB_CONS_DEVICE_PTRS == 1


def test_consensus_batch_rejects_bad_arguments_before_the_library():
    """Shapes, dtypes, layouts and counts are checked in Python; no context is needed to see them refused."""
    ctx = api.Context.__new__(api.Context)  # no device here: only the argument checks run
    b = np.zeros((5, 31), np.uint8)
    bl = np.zeros((2, 5), np.float32)
    sup = [np.zeros((2, 2), np.uint32), np.zeros((0, 2), np.uint32)]
    good = ([2], [3, 2], [2, 2], b, sup, bl)
    cases = [
        ([2], [3, 2], [2, 2], b.astype(np.int32), sup, bl),           # bases dtype
        ([2], [3, 2], [2, 2], b, sup, bl.astype(np.float64)),         # logits dtype
        ([2], [3, 2], [2, 2], b[:, :30], sup, bl),                    # bases not [N, 31]
        ([2], [3, 2], [2, 2], np.zeros((10, 31), np.uint8)[::2], sup, bl),  # not contiguous
        ([2], [3, 3], [2, 2], b, sup, bl),                            # N does not match rows
        ([2], [3, 2], [2, 2], b, sup, bl[:1]),                        # S does not match supported
        ([2], [3, 2], [2, 2], b, [np.zeros((2, 3), np.uint32), sup[1]], bl),  # supported not [n, 2]
        ([3], [3, 2], [2, 2], b, sup, bl),                            # W does not match
        ([2], [3, 2], [2, 256], b, sup, bl),                          # n_alns beyond a u8
        ([2], [3, -2], [2, 2], b, sup, bl),                           # negative rows
        ([2], [3, 2], [2.5, 2], b, sup, bl),                          # not integers
        ([2], [3, 2], [2, 2], b, sup, list(bl)),                      # a list, not an array
    ]
    for args in cases:
        with pytest.raises((TypeError, ValueError)):
            ctx.consensus_batch(*args)
    with pytest.raises(AttributeError):  # the good arguments get as far as the library call, which needs a context
        ctx.consensus_batch(*good)
