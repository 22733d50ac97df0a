"""No-GPU checks of hb_forward_batch's host side: the `herro features` reader builds exactly the model batches the reference's
collate would (compared with the oracle's batches of the targets the golden dump was written from), and the new entry point is
declared and exported."""
import os
import re

import numpy as np

import helpers  # noqa: F401  (puts the repository root on sys.path)
from herro_b200 import api, hostio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP = os.path.join(ROOT, "tests", "golden", "features_dump")


def test_feature_reader_batches_equal_the_reference_batches():
    from oracle import pyoracle as po
    from tools import make_feature_fixture as mf
    rs = mf.readset()
    reads = po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)])
    dirs = hostio.feature_reads(DUMP)
    assert [os.path.basename(d) for d in dirs] == [rs.ids[t] for t in mf.TARGETS]
    n_batches = n_gap_rows = 0
    for t, d in zip(mf.TARGETS, dirs):
        ovl, cigs = rs.target_alns(t)
        T = po.Target(reads, t, ovl, cigs, mf.W, 4)
        wins = T.windows()
        got = hostio.read_feature_batches(d, 4)
        assert len(got) == T.n_batches
        for i, g in enumerate(got):
            B = T.batch(i)
            assert g.read == rs.ids[t]
            assert g.wids == [wins[int(k)].wid for k in B.win_index]
            assert g.bases.dtype == np.uint8 and np.array_equal(g.bases, B.bases)
            assert g.quals.dtype == np.uint8 and np.array_equal(g.quals, B.quals)
            assert np.array_equal(g.lens, B.lens)
            assert len(g.indices) == len(B.indices)
            for a, b in zip(g.indices, B.indices):
                assert a.dtype == np.int32 and np.array_equal(a, b)
            n_gap_rows += int((g.bases[:, :, 0] == hostio.TOK_GAP).sum())
            n_batches += 1
    assert n_batches >= 3
    assert n_gap_rows > 0  # insertion rows exist, so target_rows[pos] + ins is exercised


def test_forward_batch_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "herro_b200.h")).read()
    assert re.search(r"\bint hb_forward_batch\s*\(", hdr)
    assert re.search(r"#define HB_FWD_DEVICE_PTRS 1u", hdr)
    assert "hb_forward_batch" in api.EXPORTED_SYMBOLS
    assert api.HB_FWD_DEVICE_PTRS == 1


def test_forward_batch_rejects_bad_arguments_before_the_library():
    """Shapes, dtypes, layouts and index lists are checked in Python; no context is needed to see them refused."""
    ctx = api.Context.__new__(api.Context)  # no device here: only the argument checks run
    ok = np.zeros((2, 5, 31), np.uint8)
    cases = [
        (ok.astype(np.int32), ok, [1, 1], [[0], [0]]),
        (ok[:, :, :30], ok[:, :, :30], [1, 1], [[0], [0]]),
        (ok[:, ::2], ok[:, ::2], [1, 1], [[0], [0]]),
        (ok, ok[:1], [1, 1], [[0], [0]]),
        (ok, ok, [1], [[0]]),
        (ok, ok, [1, 2], [[0], [0]]),
    ]
    for bases, quals, lens, idx in cases:
        try:
            ctx.forward_batch(bases, quals, lens, idx)
        except (TypeError, ValueError):
            continue
        raise AssertionError("accepted a bad argument")
