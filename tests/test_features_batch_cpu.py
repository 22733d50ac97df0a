"""hb_features_batch / hb_features_fetch without a GPU: the declarations, exports and struct layouts, the NULL-argument errors, a
context without weights getting as far as the device check, the Python-side argument checks, and the `cli features` file writer
reproducing tests/golden/features_dump from the oracle's windows."""
import ctypes as C
import glob
import os
import re
import subprocess

import numpy as np
import pytest

import helpers
from herro_b200 import api, hostio

ROOT = helpers.ROOT
HB_OK, HB_ERR_ARG, HB_ERR_CUDA = 0, -1, -2
DUMP = os.path.join(ROOT, "tests", "golden", "features_dump")


def test_features_batch_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "herro_b200.h")).read()
    assert re.search(r"\bint hb_features_batch\s*\(", hdr)
    assert re.search(r"\bint hb_features_fetch\s*\(", hdr)
    assert re.search(r"#define HB_FEAT_DEVICE_PTRS 1u", hdr)
    assert re.search(r"#define HB_FLAG_NO_MODEL +2u", hdr)
    assert {"hb_features_batch", "hb_features_fetch"} <= set(api.EXPORTED_SYMBOLS)
    lib = C.CDLL(api.LIB_PATH)
    lib.hb_features_batch, lib.hb_features_fetch
    assert api.HB_FEAT_DEVICE_PTRS == 1 and api.HB_FLAG_NO_MODEL == 2


def test_ctypes_structs_match_the_header(tmp_path):
    """sizeof / offsetof of hb_features_shape and hb_features_out as a C compiler lays them out, against the ctypes mirrors."""
    fields = {"hb_features_shape": [n for n, _ in api.HbFeaturesShape._fields_],
              "hb_features_out": [n for n, _ in api.HbFeaturesOut._fields_]}
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "herro_b200.h"', "int main(void) {"]
    for s, names in fields.items():
        src.append(f'printf("%zu\\n", sizeof({s}));')
        src += [f'printf("%zu\\n", offsetof({s}, {n}));' for n in names]
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(c)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = []
    for cls in (api.HbFeaturesShape, api.HbFeaturesOut):
        want.append(C.sizeof(cls))
        want += [getattr(cls, n).offset for n, _ in cls._fields_]
    assert got == want


def test_null_arguments_are_errors_not_crashes():
    L = api.load_library()
    sh = api.HbFeaturesShape()
    out = api.HbFeaturesOut(C.sizeof(api.HbFeaturesOut))
    assert L.hb_features_batch(None, 0, None, None, None, C.byref(sh)) == HB_ERR_ARG
    assert L.hb_features_batch(None, 0, None, None, None, None) == HB_ERR_ARG
    assert L.hb_features_fetch(None, C.byref(sh), C.byref(out), 0, None) == HB_ERR_ARG
    assert L.hb_features_fetch(None, None, None, 0, None) == HB_ERR_ARG


def test_no_model_context_accepts_a_null_model_path():
    """With HB_FLAG_NO_MODEL a NULL model_path passes the argument check and hb_create goes on to the device (HB_ERR_CUDA without
    one); without the flag a NULL path is still HB_ERR_ARG."""
    L = api.load_library()
    h = C.c_void_p()
    opt = api.HbOptions(C.sizeof(api.HbOptions), 4096, 64, 0, 0)
    assert L.hb_create(C.byref(h), 0, None, C.byref(opt)) == HB_ERR_ARG
    assert L.hb_create(C.byref(h), 0, None, None) == HB_ERR_ARG
    opt.flags = api.HB_FLAG_NO_MODEL
    rc = L.hb_create(C.byref(h), 0, None, C.byref(opt))
    assert rc in (HB_OK, HB_ERR_CUDA), rc  # HB_OK where a device is present
    if rc == HB_OK:
        L.hb_destroy(h)
    else:
        assert b"no CUDA device" in L.hb_last_error(None)


def test_features_batch_rejects_bad_arguments_before_the_library():
    ctx = api.Context.__new__(api.Context)  # no device here: only the argument checks run
    ov = np.zeros(2, api.OVERLAP_DTYPE)
    cases = [
        ([(0, ov)], dict(device=1)),                              # device not a bool
        ([(0, ov)], dict(batches="yes")),                         # batches not a bool
        ([0], {}),                                                # not a pair
        ([(0, ov, 1)], {}),                                       # not a pair
        ([(-1, ov)], {}),                                         # rid negative
        ([(2 ** 32, ov)], {}),                                    # rid past u32
        ([(1.0, ov)], {}),                                        # rid not an integer
        ([(True, ov)], {}),                                       # rid a bool
        ([(0, np.zeros((2, 9), np.uint32))], {}),                 # overlaps not hb_overlap records
        ([(0, np.zeros((2, 1), api.OVERLAP_DTYPE))], {}),         # overlaps not 1-D
        ([(0, list(ov))], {}),                                    # overlaps not an array
    ]
    for targets, kw in cases:
        with pytest.raises((TypeError, ValueError)):
            ctx.features_batch(targets, **kw)


def oracle_targets():
    from oracle import pyoracle as po
    from tools import make_feature_fixture as mff
    rs = mff.readset()
    reads = po.Reads(rs.ids, [rs.seq(i) for i in range(rs.n)], [rs.qual(i) for i in range(rs.n)])
    out = []
    for t in mff.TARGETS:
        ovl, cigs = rs.target_alns(t)
        if len(ovl):
            out.append((t, po.Target(reads, t, ovl, cigs, mff.W, 4)))
    return rs, out


def test_cli_writer_reproduces_the_golden_dump_from_the_oracle_windows(tmp_path):
    """The files `cli features` writes from a Features result, fed here with the oracle's windows laid out as hb_features_fetch lays
    them out (window after window), are byte-identical to the fixture."""
    from herro_b200 import cli
    rs, targets = oracle_targets()
    names = [i.encode() for i in rs.ids]
    wins = [w for _, T in targets for w in T.windows()]
    cat = lambda xs, shape, dt: np.concatenate(xs).reshape(shape).astype(dt) if xs else np.zeros(shape, dt)  # noqa: E731
    arrays = dict(
        status=np.zeros(len(targets), np.int32), n_windows=np.array([T.n_windows for _, T in targets], np.uint32),
        rows=np.array([w.bases.shape[0] for w in wins], np.uint32), n_alns=np.array([w.n_alns for w in wins], np.uint8),
        n_sup=np.array([len(w.sup_rows) for w in wins], np.uint32), n_ids=np.array([len(w.qids) for w in wins], np.uint32),
        bases=cat([w.bases for w in wins], (-1, 31), np.uint8), quals=cat([w.quals for w in wins], (-1, 31), np.uint8),
        supported=cat([w.supported.reshape(-1, 2) for w in wins], (-1, 2), np.uint32),
        indices=cat([w.sup_rows for w in wins], (-1,), np.int32), ids=cat([w.qids for w in wins], (-1,), np.uint32))
    F = api.Features([t for t, _ in targets], arrays, 4)
    out = str(tmp_path / "feats")
    for k in range(len(targets)):
        cli.write_features(F, k, out, names)
    n = 0
    for d in sorted(glob.glob(os.path.join(DUMP, "read_*"))):
        for a in sorted(glob.glob(os.path.join(d, "*"))):
            b = os.path.join(out, os.path.basename(d), os.path.basename(a))
            assert open(a, "rb").read() == open(b, "rb").read(), b
            n += 1
    assert n == 3 * len(wins) and n >= 30


def test_features_helpers_give_the_oracle_batches_and_consensus_args():
    """Features.batches() over collated arrays laid out as hb_features_fetch lays them out gives the oracle's T.batch(b), and
    consensus_args splits the supported list per window."""
    rs, targets = oracle_targets()
    wins = [w for _, T in targets for w in T.windows()]
    rows = np.array([w.bases.shape[0] for w in wins], np.uint32)
    n_sup = np.array([len(w.sup_rows) for w in wins], np.uint32)
    batch_B, batch_Lmax, batch_win, bb, bq, want = [], [], [], [], [], []
    w0 = 0
    for _, T in targets:
        for b in range(T.n_batches):
            B = T.batch(b)
            want.append(B)
            batch_B.append(B.bases.shape[0])
            batch_Lmax.append(B.bases.shape[1])
            batch_win += [w0 + int(i) for i in B.win_index]
            bb.append(B.bases.reshape(-1, 31))
            bq.append(B.quals.reshape(-1, 31))
        w0 += T.n_windows
    arrays = dict(status=np.zeros(len(targets), np.int32), n_windows=np.array([T.n_windows for _, T in targets], np.uint32), rows=rows,
                  n_alns=np.array([w.n_alns for w in wins], np.uint8), n_sup=n_sup, n_ids=np.array([len(w.qids) for w in wins], np.uint32),
                  bases=np.concatenate([w.bases for w in wins]), quals=np.concatenate([w.quals for w in wins]),
                  supported=np.concatenate([w.supported.reshape(-1, 2) for w in wins]).astype(np.uint32),
                  indices=np.concatenate([w.sup_rows for w in wins]).astype(np.int32), ids=np.concatenate([w.qids for w in wins]),
                  batch_B=np.array(batch_B, np.uint32), batch_Lmax=np.array(batch_Lmax, np.uint32), batch_win=np.array(batch_win, np.uint32),
                  batch_bases=np.concatenate(bb), batch_quals=np.concatenate(bq))
    F = api.Features([t for t, _ in targets], arrays, 4)
    got = list(F.batches())
    assert len(got) == len(want) >= 3
    for (ws, bases, quals, lens, idx), B in zip(got, want):
        assert np.array_equal(bases, B.bases) and np.array_equal(quals, B.quals) and np.array_equal(lens, B.lens)
        assert len(idx) == len(B.indices) and all(np.array_equal(a, b) for a, b in zip(idx, B.indices))
    logits = [np.full((int(n), 5), w, np.float32) for w, n in enumerate(n_sup)]
    nw, r, na, b, sup, bl = F.consensus_args([logits])
    assert np.array_equal(r, rows) and len(sup) == len(wins) and np.array_equal(bl, np.concatenate(logits))
    assert all(np.array_equal(s, w.supported.reshape(-1, 2)) for s, w in zip(sup, wins))
