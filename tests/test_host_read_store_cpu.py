"""The read store in host memory without a GPU: the declarations are exported, bad arguments are refused before any CUDA call, the
packed-store size the harness compares is the layout's, and the rule that chooses the store for `inference` / `features`."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import helpers
from herro_b200 import api, hostio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HB_ERR_ARG = -1
NEW = ("hb_read_store_create", "hb_read_store_destroy", "hb_attach_read_store")


def test_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "herro_b200.h")).read()
    assert "typedef struct hb_read_store hb_read_store;" in hdr
    lib = C.CDLL(api.LIB_PATH)
    for sym in NEW:
        assert re.search(r"\bint " + sym + r"\(", hdr) and sym in api.EXPORTED_SYMBOLS and hasattr(lib, sym)


def test_bad_arguments_before_any_cuda_call():
    L = api.load_library()
    words = np.zeros(4, np.uint64)
    qual = np.zeros(100, np.uint8)
    lens = np.array([100], np.uint32)
    wp = np.array([words.ctypes.data], np.uint64)
    qp = np.array([qual.ctypes.data], np.uint64)
    null = np.array([0], np.uint64)
    h = C.c_void_p()
    assert L.hb_read_store_create(None, 1, wp.ctypes.data, lens.ctypes.data, qp.ctypes.data) == HB_ERR_ARG
    assert L.hb_read_store_create(C.byref(h), 0, wp.ctypes.data, lens.ctypes.data, qp.ctypes.data) == HB_ERR_ARG
    for a, b, c in ((None, lens.ctypes.data, qp.ctypes.data), (wp.ctypes.data, None, qp.ctypes.data), (wp.ctypes.data, lens.ctypes.data, None),
                    (null.ctypes.data, lens.ctypes.data, qp.ctypes.data), (wp.ctypes.data, lens.ctypes.data, null.ctypes.data)):
        assert L.hb_read_store_create(C.byref(h), 1, a, b, c) == HB_ERR_ARG
        assert L.hb_last_error(None)
    assert h.value is None
    assert L.hb_read_store_destroy(None) == HB_ERR_ARG
    assert L.hb_attach_read_store(None, None) == HB_ERR_ARG
    with pytest.raises(api.HerroError) as e:
        api.ReadStore(np.zeros(0, np.uint8), np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert e.value.code == HB_ERR_ARG


def test_store_bytes_of_the_harness(tmp_path):
    from tools import synth
    rs = helpers.small_readset(n_reads=12, mean_len=5000, seed=3)
    fq = str(tmp_path / "r.fastq")
    synth.write_fastq(rs, fq)
    R = hostio.Reads(fq, min_len=1)
    lens = R.lens.astype(np.int64)
    assert R.store_bytes() == int(((lens + 31) // 32 * 8 + lens).sum())


def test_selection_rule():
    GB = 10 ** 9
    above = hostio.host_store_above([80 * GB, 40 * GB])
    assert above == 20 * GB                                  # half the smallest selected device
    assert not 20 * GB > above and 20 * GB + 1 > above       # device store up to it, host store past it
    assert hostio.host_store_above([80 * GB]) == 40 * GB
    assert hostio.host_store_above(None, "host") == 0        # any non-empty store is larger
    assert not (2 ** 63) > hostio.host_store_above(None, "device")
    with pytest.raises(ValueError):
        hostio.host_store_above([80 * GB], "gpu")
