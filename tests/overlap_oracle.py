"""Test infrastructure: the CPU oracle of hb_find_overlaps (tests/overlap_oracle.cpp), built with g++ into tests/_tmp on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "overlap_oracle.cpp")
LIB = os.path.join(ROOT, "tests", "_tmp", "liboverlap_oracle.so")

PARAM_NAMES = ("k", "w", "min_score", "min_anchors", "max_gap", "bandwidth", "max_iter", "top_frac_ppm", "min_occ")
DEFAULTS = dict(k=25, w=17, min_score=2500, min_anchors=3, max_gap=5000, bandwidth=150, max_iter=5000, top_frac_ppm=5000,
                min_occ=10)
RECORD_FIELDS = ("qid", "qlen", "qstart", "qend", "strand", "tid", "tlen", "tstart", "tend", "score", "n_anchors", "covered")

_CODE = np.full(256, 255, np.uint8)
for _k, _c in enumerate(b"ACGT"):
    _CODE[_c] = _k

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            tmp = f"{LIB}.{os.getpid()}"
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", tmp, SRC])
            os.replace(tmp, LIB)
        L = C.CDLL(LIB)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.oo_hash64.argtypes = [u64, u64]
        L.oo_hash64.restype = u64
        L.oo_sketch.argtypes = [vp, u32, u32, u32, vp, vp, vp, u32]
        L.oo_sketch.restype = u32
        L.oo_max_occ.argtypes = [vp, u32, u32, u32]
        L.oo_max_occ.restype = u32
        L.oo_chain.argtypes = [vp, vp, u32, vp, vp]
        L.oo_find.argtypes = [vp, vp, u32, vp, u32, vp, vp, u64, vp]
        L.oo_find.restype = u64
        _lib = L
    return _lib


def params(**kw) -> np.ndarray:
    p = dict(DEFAULTS)
    p.update({k: v for k, v in kw.items() if v})
    return np.array([p[n] for n in PARAM_NAMES], np.uint32)


def codes(seq: bytes) -> np.ndarray:
    """ASCII ACGT -> 2-bit codes (A 0, C 1, G 2, T 3)."""
    return _CODE[np.frombuffer(seq, np.uint8)]


def hash64(key: int, mask: int) -> int:
    return int(lib().oo_hash64(key, mask))


def sketch(seq: bytes, k: int, w: int):
    """-> (h u64[], pos u32[], z u32[]) of one read's minimizers"""
    c = np.ascontiguousarray(codes(seq))
    cap = max(len(c), 1)
    h, pos, z = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    n = lib().oo_sketch(c.ctypes.data, len(c), k, w, h.ctypes.data, pos.ctypes.data, z.ctypes.data, cap)
    return h[:n], pos[:n], z[:n]


def max_occ(occ, top_frac_ppm=5000, min_occ=10) -> int:
    occ = np.ascontiguousarray(occ, np.uint32)
    return int(lib().oo_max_occ(occ.ctypes.data, len(occ), top_frac_ppm, min_occ))


def chain(x, y, **kw) -> dict:
    """The chain of one group of anchors (sorted by (x, y)) -> dict(score, n_anchors, first, last, covered)."""
    x, y = np.ascontiguousarray(x, np.uint32), np.ascontiguousarray(y, np.uint32)
    p, out = params(**kw), np.zeros(5, np.int64)
    lib().oo_chain(x.ctypes.data, y.ctypes.data, len(x), p.ctypes.data, out.ctypes.data)
    return dict(zip(("score", "n_anchors", "first", "last", "covered"), (int(v) for v in out)))


def find(seqs, targets, **kw) -> dict:
    """hb_find_overlaps restated: seqs are the store's reads (bytes), targets the call's read ids.
    -> dict(records: u32[n, 12] in RECORD_FIELDS order, max_occ, n_filtered_hashes, index_entries, query_minimizers, anchors)"""
    cs = [codes(s) for s in seqs]
    off = np.zeros(len(cs) + 1, np.uint64)
    off[1:] = np.cumsum([len(c) for c in cs])
    allc = np.ascontiguousarray(np.concatenate(cs) if cs else np.zeros(1, np.uint8))
    tg = np.ascontiguousarray(targets, np.uint32)
    p = params(**kw)
    stats = np.zeros(5, np.uint64)
    cap = 1 << 16
    while True:
        out = np.zeros((cap, 12), np.uint32)
        n = int(lib().oo_find(allc.ctypes.data, off.ctypes.data, len(cs), tg.ctypes.data, len(tg), p.ctypes.data, out.ctypes.data,
                              cap, stats.ctypes.data))
        if n <= cap:
            break
        cap = n
    return dict(records=out[:n], max_occ=int(stats[0]), n_filtered_hashes=int(stats[1]), index_entries=int(stats[2]),
                query_minimizers=int(stats[3]), anchors=int(stats[4]))
