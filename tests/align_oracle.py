"""Test infrastructure: the CPU oracle of hb_align_overlaps (tests/align_oracle.cpp), built with g++ into tests/_tmp on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "align_oracle.cpp")
LIB = os.path.join(ROOT, "tests", "_tmp", "libalign_oracle.so")

HB_OK, HB_ALN_BAND_EDGE, HB_ERR_INPUT = 0, 1, -4
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
        vp = C.c_void_p
        L.ao_fix_cigar.argtypes = [vp, vp, C.c_char_p, vp, C.c_uint32, vp]
        L.ao_align.argtypes = [vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp, vp, C.c_uint32]
        _lib = L
    return _lib


def codes(seq: bytes) -> np.ndarray:
    """ASCII ACGT -> 2-bit codes (A 0, C 1, G 2, T 3; the complement is code ^ 3)."""
    return _CODE[np.frombuffer(seq, np.uint8)]


def fix_cigar(target: bytes, query: bytes, cigar: bytes):
    """-> (fixed CIGAR, tshift, qshift)"""
    out = C.create_string_buffer(len(cigar) + 16)
    sh = np.zeros(2, np.uint32)
    t, q = np.frombuffer(target, np.uint8).copy(), np.frombuffer(query, np.uint8).copy()
    if lib().ao_fix_cigar(t.ctypes.data, q.ctypes.data, cigar, out, len(out), sh.ctypes.data) != 0:
        raise ValueError("malformed CIGAR")
    return out.value, int(sh[0]), int(sh[1])


def align_codes(T: np.ndarray, Q: np.ndarray, w: int) -> dict:
    """The banded alignment of code arrays T (target) and Q (oriented query): score, lead/trail shifts, edge, matches, cigar."""
    T = np.ascontiguousarray(T, np.uint8)
    Q = np.ascontiguousarray(Q, np.uint8)
    res = np.zeros(7, np.int32)
    cap = 4 * (len(T) + len(Q)) + 64
    buf = C.create_string_buffer(cap)
    rc = lib().ao_align(T.ctypes.data, len(T), Q.ctypes.data, len(Q), w, res.ctypes.data, buf, cap)
    if rc != 0:
        raise RuntimeError(f"ao_align failed ({rc})")
    return dict(score=int(res[0]), lead_d=int(res[1]), lead_i=int(res[2]), trail_d=int(res[3]), trail_i=int(res[4]),
                edge=bool(res[5]), matches=int(res[6]), cigar=buf.value)


def oriented_query(q: np.ndarray, qstart: int, qend: int, strand: int) -> np.ndarray:
    s = q[qstart:qend]
    return (s[::-1] ^ 3).astype(np.uint8) if strand else s


def align_overlap(t_codes: np.ndarray, q_codes: np.ndarray, qstart, qend, strand, tstart, tend, w):
    """One overlap as hb_align_overlaps defines it -> (status, (qstart, qend, tstart, tend), cigar bytes, matches).  A failed
    overlap keeps its coordinates and has an empty CIGAR."""
    n, m = tend - tstart, qend - qstart
    if (qstart > qend or qend > len(q_codes) or tstart > tend or tend > len(t_codes) or n == 0 or m == 0 or m > 2 * n
            or n > 2 * m):
        return HB_ERR_INPUT, (qstart, qend, tstart, tend), b"", 0
    r = align_codes(t_codes[tstart:tend], oriented_query(q_codes, qstart, qend, strand), w)
    ts, te = tstart + r["lead_d"], tend - r["trail_d"]
    if strand:
        qs, qe = qstart + r["trail_i"], qend - r["lead_i"]
    else:
        qs, qe = qstart + r["lead_i"], qend - r["trail_i"]
    return (HB_ALN_BAND_EDGE if r["edge"] else HB_OK), (qs, qe, ts, te), r["cigar"], r["matches"]
