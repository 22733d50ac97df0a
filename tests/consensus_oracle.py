"""Test infrastructure: the CPU oracle's consensus() on caller-supplied windows (tests/consensus_oracle.cpp, which includes
oracle/herro_oracle.cpp as it is), built with g++ into tests/_tmp on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "consensus_oracle.cpp")
ORACLE = os.path.join(ROOT, "oracle", "herro_oracle.cpp")
LIB = os.path.join(ROOT, "tests", "_tmp", "libconsensus_oracle.so")


class OraclePanic(RuntimeError):
    """The oracle's consensus() hit one of the reference's panic sites."""


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(ORACLE)):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            tmp = f"{LIB}.{os.getpid()}"
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", tmp, SRC])
            os.replace(tmp, LIB)
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.ho_last_error.restype = C.c_char_p
        L.ho_consensus_windows.argtypes = [C.c_uint32] + [vp] * 10
        _lib = L
    return _lib


def consensus_windows(reads):
    """consensus() on caller-supplied windows.  reads: per read, its windows in wid order as (bases [L, 31] u8 tokens, n_alns,
    supported [n, 2] (pos, ins), bases_logits [n, 5] f32).  -> per read, list[bytes] (empty: no record, None included).
    Raises OraclePanic where the reference would panic."""
    wins = [w for r in reads for w in r]
    n_windows = np.array([len(r) for r in reads] or [0], dtype=np.uint32)
    rows = np.array([len(w[0]) for w in wins] or [0], dtype=np.uint32)
    n_alns = np.array([w[1] for w in wins] or [0], dtype=np.uint8)
    n_sup = np.array([len(w[2]) for w in wins] or [0], dtype=np.uint32)
    bases = np.ascontiguousarray(np.concatenate([np.asarray(w[0], np.uint8).reshape(-1, 31) for w in wins] + [np.zeros((1, 31), np.uint8)]))
    sup = np.ascontiguousarray(np.concatenate([np.asarray(w[2], np.uint32).reshape(-1, 2) for w in wins] + [np.zeros((1, 2), np.uint32)]))
    bl = np.ascontiguousarray(np.concatenate([np.asarray(w[3], np.float32).reshape(-1, 5) for w in wins] + [np.zeros((1, 5), np.float32)]))
    seqs = np.zeros(max(int(rows.sum()), 1), np.uint8)
    seg_len = np.zeros(max(len(wins), 1), np.uint32)
    n_segs = np.zeros(max(len(reads), 1), np.uint32)
    L = lib()
    if L.ho_consensus_windows(len(reads), *(a.ctypes.data for a in (n_windows, rows, n_alns, bases, n_sup, sup, bl, seqs, seg_len, n_segs))) != 0:
        raise OraclePanic(L.ho_last_error().decode())
    out, s, o = [], 0, 0
    for i in range(len(reads)):
        segs = []
        for _ in range(int(n_segs[i])):
            segs.append(seqs[o:o + int(seg_len[s])].tobytes())
            o += int(seg_len[s])
            s += 1
        out.append(segs)
    return out
