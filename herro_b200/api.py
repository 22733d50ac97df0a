"""Host-side mirror of the reference's hot-path interface over the C ABI (include/herro_b200.h).

The deployed host is the reference's Rust binary (INTEGRATION.md); there is no Rust toolchain
offline, so this ctypes layer is the harness that plays `lib.rs::error_correction`
(src/lib.rs:113-206) for tests and benchmarks: it keeps the reference's vocabulary — reads,
alignments grouped by target (`(tid, Vec<Alignment>)`, src/overlaps.rs:371-373), windows,
corrected segments — and calls exactly the entry points the Rust `mod ffi` would bind.

Everything compute-related happens inside libherro_b200.so (CUDA, sm_90a).  There is no CPU
fallback: constructing a Context without a CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libherro_b200.so")

HB_FLAG_KEEP_DEBUG = 1
HB_FLAG_NO_MODEL = 2

OVERLAP_DTYPE = np.dtype(
    {"names": ["qid", "qlen", "qstart", "qend", "strand", "tid", "tlen", "tstart", "tend", "cigar", "cigar_len"],
     "formats": ["<u4"] * 9 + ["<u8", "<u4"],
     "offsets": [0, 4, 8, 12, 16, 20, 24, 28, 32, 40, 48],
     "itemsize": 56})
OVERLAP_WINDOW_DTYPE = np.dtype([(n, "<u4") for n in (
    "overlap_idx", "window_idx", "tstart", "qstart", "qend", "cigar_start_idx", "cigar_start_offset", "cigar_end_idx",
    "cigar_end_offset")])


class HbOptions(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("window_size", C.c_uint32), ("batch_size", C.c_uint32),
                ("launch_targets", C.c_uint32), ("flags", C.c_uint32)]


KERNEL_CLASSES = ["tokenize", "pass1", "scores", "pass2a", "scan", "pileup", "lists", "stem", "layernorm", "gemm",
                  "attention", "heads", "consensus", "ffn", "qkv_attn", "pos_attn"]


class HbStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("targets", "windows", "overlap_windows", "rows", "supported",
                                          "corrected_bases", "h2d_bytes", "d2h_bytes", "kernel_launches",
                                          "device_launches", "pileup_algo_bytes", "gemm_flops", "forward_flops")] + \
               [(n, C.c_double) for n in ("ms_features", "ms_forward", "ms_consensus")] + \
               [("ms_kernel", C.c_double * 16), ("n_kernel", C.c_uint64 * 16)] + \
               [(n, C.c_uint64) for n in ("last_launch_targets", "last_launch_windows", "last_launch_bases")] + \
               [("ms_worker_busy", C.c_double), ("ms_worker_gpu_wait", C.c_double)] + \
               [("host_allocs", C.c_uint64), ("ms_host_alloc", C.c_double), ("ms_submit_wait", C.c_double),
                ("class_flops", C.c_uint64 * 16), ("ms_worker_phase", C.c_double * 8)]


class HbFeaturesShape(C.Structure):
    _fields_ = [("ticket", C.c_uint64)] + [(n, C.c_uint32) for n in ("n_targets", "n_windows", "n_batches", "n_failed")] + \
               [(n, C.c_uint64) for n in ("n_rows", "n_sup", "n_ids", "n_batch_rows")]


FEATURES_OUT_FIELDS = ("status", "n_windows", "rows", "n_alns", "n_sup", "n_ids", "bases", "quals", "supported", "indices", "ids",
                       "batch_B", "batch_Lmax", "batch_win", "batch_bases", "batch_quals")


class HbFeaturesOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32)] + [(n, C.c_void_p) for n in FEATURES_OUT_FIELDS]


HOST_LIB_PATH = os.path.join(_HERE, "libherro_host.so")


class HerroError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"herro_b200 error {code}: {msg}")
        self.code = code


_lib = None


def load_library():
    """dlopen the in-tree CUDA library; fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise HerroError(-2, f"{LIB_PATH} not built - run `python -c 'import __graft_entry__ as g; g.build()'` "
                             "(herro_b200 has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, u32, u32p = C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)
    L.hb_last_error.restype = C.c_char_p
    L.hb_last_error.argtypes = [vp]
    L.hb_create.argtypes = [C.POINTER(vp), C.c_int, C.c_char_p, C.POINTER(HbOptions)]
    L.hb_destroy.argtypes = [vp]
    L.hb_destroy.restype = None
    L.hb_upload_reads.argtypes = [vp, u32, vp, vp, vp]
    L.hb_read_store_create.argtypes = [C.POINTER(vp), u32, vp, vp, vp]
    L.hb_read_store_destroy.argtypes = [vp]
    L.hb_attach_read_store.argtypes = [vp, vp]
    L.hb_submit_target.argtypes = [vp, u32, u32, vp, u32, vp, u32]
    L.hb_submit_alignments.argtypes = [vp, u32, vp, u32]
    L.hb_extract_windows.argtypes = [vp, u32, u32, u32, vp, u32, u32p]
    L.hb_window_range.argtypes = [vp, u32, u32, u32p, u32p]
    L.hb_flush.argtypes = [vp]
    L.hb_set_launch_targets.argtypes = [vp, u32]
    L.hb_set_kernel_timing.argtypes = [vp, C.c_int]
    L.hb_poll_corrected.argtypes = [vp, u32p, C.POINTER(vp), C.POINTER(vp), u32p]
    L.hb_release_result.argtypes = [vp, vp]
    L.hb_release_result.restype = None
    L.hb_bind_calling_thread.argtypes = [vp]
    L.hb_get_stats.argtypes = [vp, C.POINTER(HbStats)]
    L.hb_reset_stats.argtypes = [vp]
    L.hb_debug_window_shape.argtypes = [vp, u32, u32, u32p]
    L.hb_debug_dump_window.argtypes = [vp, u32, u32, vp, vp, vp, vp, vp, vp]
    L.hb_replay_last_launch.argtypes = [vp, u32, C.POINTER(C.c_float)]
    L.hb_dump_features.argtypes = [vp, u32, C.c_char_p, vp]
    L.hb_inspect_model.argtypes = [C.c_char_p, u32p, C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.hb_inspect_model_ex.argtypes = [C.c_char_p, u32p, C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    fp = C.POINTER(C.c_float)
    L.hb_selftest_gemm.argtypes = [C.c_int, u32, u32, u32, C.c_int, C.c_int, u32, fp, fp, fp, fp]
    L.hb_selftest_pos_attention.argtypes = [C.c_int, u32p, u32, u32, u32, fp, fp, fp]
    L.hb_forward_batch.argtypes = [vp, u32, u32, vp, vp, vp, vp, vp, vp, u32, vp]
    L.hb_consensus_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u32, vp]
    L.hb_features_batch.argtypes = [vp, u32, vp, vp, vp, C.POINTER(HbFeaturesShape)]
    L.hb_features_fetch.argtypes = [vp, C.POINTER(HbFeaturesShape), C.POINTER(HbFeaturesOut), u32, vp]
    _lib = L
    return L


EXPORTED_SYMBOLS = ["hb_inspect_model", "hb_dump_features", "hb_window_range", "hb_bind_calling_thread", "hb_set_launch_targets", "hb_set_kernel_timing", "hb_extract_windows", "hb_create", "hb_destroy", "hb_upload_reads", "hb_submit_target", "hb_submit_alignments", "hb_flush",
                    "hb_poll_corrected", "hb_release_result", "hb_last_error", "hb_get_stats", "hb_reset_stats",
                    "hb_debug_window_shape", "hb_debug_dump_window", "hb_replay_last_launch", "hb_selftest_gemm",
                    "hb_inspect_model_ex", "hb_selftest_pos_attention", "hb_forward_batch", "hb_consensus_batch",
                    "hb_features_batch", "hb_features_fetch", "hb_read_store_create", "hb_read_store_destroy", "hb_attach_read_store"]
HB_FWD_DEVICE_PTRS = 1
HB_CONS_DEVICE_PTRS = 1
HB_FEAT_DEVICE_PTRS = 1


def selftest_gemm(M, N, K, act=0, res=0, lda_extra=0, device=0):
    """-> dict(max_abs_err, max_abs_ref, ms_tc, ms_simt): wgmma bf16x3 contraction vs fp32 SIMT."""
    L = load_library()
    v = [C.c_float() for _ in range(4)]
    rc = L.hb_selftest_gemm(device, M, N, K, act, res, lda_extra, *[C.byref(x) for x in v])
    if rc != 0:
        raise HerroError(rc, L.hb_last_error(None).decode())
    return dict(max_abs_err=v[0].value, max_abs_ref=v[1].value, ms_tc=v[2].value, ms_simt=v[3].value)


def selftest_pos_attention(lens, heads: int, head_dim: int, qkv: np.ndarray, device=0):
    """The position-axis stage's masked attention kernel on sequences of `lens` rows stored back to back in `qkv`
    ([sum lens, 3 * heads * head_dim] fp32, q | k | v) -> (output [sum lens, heads * head_dim] fp32, kernel ms)."""
    L = load_library()
    lens = np.ascontiguousarray(lens, dtype=np.uint32)
    D = heads * head_dim
    qkv = np.ascontiguousarray(qkv, dtype=np.float32)
    if qkv.shape != (int(lens.sum()), 3 * D):
        raise ValueError(f"qkv must be [{int(lens.sum())}, {3 * D}], got {qkv.shape}")
    out = np.zeros((int(lens.sum()), D), dtype=np.float32)
    ms = C.c_float()
    fp = C.POINTER(C.c_float)
    rc = L.hb_selftest_pos_attention(device, lens.ctypes.data_as(C.POINTER(C.c_uint32)), len(lens), heads, head_dim,
                                     qkv.ctypes.data_as(fp), out.ctypes.data_as(fp), C.byref(ms))
    if rc != 0:
        raise HerroError(rc, L.hb_last_error(None).decode())
    return out, ms.value


# ------------------------------------------------------------------------------------------
# haec_io.rs host side: 2-bit packing (src/haec_io.rs:121-136).  Host data plane — stays in the
# Rust binary in deployment; needed here only because the harness replaces that binary.
# ------------------------------------------------------------------------------------------
_ENC = np.full(256, 255, dtype=np.uint64)
for _i, _ch in enumerate(b"ACGT"):
    _ENC[_ch] = _i
    _ENC[_ch + 32] = _i


def pack_2bit(seq: np.ndarray) -> np.ndarray:
    """ASCII u8 array -> u64 words, 32 bases per word, A0 C1 G2 T3, little-endian in the word."""
    n = int(seq.shape[0])
    codes = _ENC[seq]
    if n and int(codes.max()) > 3:
        raise ValueError("non-ACGT base: the reference's 2-bit packing is undefined for it (SURVEY.md H12)")
    nw = (n + 31) // 32
    pad = np.zeros(nw * 32, dtype=np.uint64)
    pad[:n] = codes
    shifts = (np.arange(32, dtype=np.uint64) * np.uint64(2))[None, :]
    return np.bitwise_or.reduce(pad.reshape(nw, 32) << shifts, axis=1)


def extract_windows(overlaps: np.ndarray, window_size: int, n_windows: int) -> np.ndarray:
    """Host-only windowing of all alignments of one target (hb_extract_windows) -> OVERLAP_WINDOW_DTYPE array."""
    L = load_library()
    cap = len(overlaps) * (n_windows + 1) + 1
    out = np.zeros(cap, dtype=OVERLAP_WINDOW_DTYPE)
    n = C.c_uint32()
    rc = L.hb_extract_windows(overlaps.ctypes.data, len(overlaps), window_size, n_windows, out.ctypes.data, cap,
                              C.byref(n))
    if rc != 0:
        raise HerroError(rc, "alignment on which the reference would panic")
    return out[:n.value]


def inspect_model(path: str):
    """Architecture and parameter hash of a model file (HB200W1 blob or TorchScript archive), host only (hb_inspect_model_ex)."""
    L = load_library()
    dims = (C.c_uint32 * 9)()
    h = C.c_uint64()
    err = C.create_string_buffer(512)
    rc = L.hb_inspect_model_ex(path.encode(), dims, C.byref(h), err, len(err))
    if rc != 0:
        raise HerroError(rc, err.value.decode(errors="replace"))
    keys = ("stem_k", "channels", "heads", "layers", "ffn", "collapse", "pos_layers", "pos_heads", "pos_ffn")
    return dict(zip(keys, [int(x) for x in dims])), int(h.value)


def window_range(overlap: np.ndarray, window_size: int, n_windows: int):
    """(first, end) of the windows one alignment (a 1-element OVERLAP_DTYPE array) contributes to (hb_window_range)."""
    L = load_library()
    a, b = C.c_uint32(), C.c_uint32()
    rc = L.hb_window_range(overlap.ctypes.data, window_size, n_windows, C.byref(a), C.byref(b))
    if rc != 0:
        raise HerroError(rc, "alignment on which the reference would panic")
    return a.value, b.value


@dataclass
class Corrected:
    rid: int
    segments: list  # list[bytes]; empty = read omitted from the output (consensus() returned None)


def _split(a, counts):
    """a split into consecutive pieces of counts[i] entries (numpy arrays or torch tensors)."""
    counts = [int(c) for c in counts]
    if type(a).__module__.split(".")[0] == "torch":
        import torch
        return list(torch.split(a[:sum(counts)], counts)) if counts else []
    return np.split(a[:sum(counts)], np.cumsum(counts)[:-1]) if counts else []


class Features:
    """What one Context.features_batch produced (hb_features_batch): the targets in the order given, each with all of its windows
    in wid order.  Per target: rids, status (0, or the HB_ERR_* code of a target that failed alone), n_windows.  Per window:
    rows (L'), n_alns, n_sup, n_ids.  Flat, window after window: bases / quals [sum rows, 31] u8, supported [sum n_sup, 2] u32
    (pos, ins), indices [sum n_sup] i32 (the row of each supported entry), ids [sum n_ids] u32 (query read ids in final rank
    order).  With batches: batch_B, batch_Lmax, batch_win (the window of each batch slot) and batch_bases / batch_quals
    [sum B * Lmax, 31] u8, the reference batches padded with 11 / 126.  The bulk arrays are torch CUDA tensors with device=True."""

    def __init__(self, rids, arrays: dict, batch_size: int):
        self.rids = rids
        self.batch_size = batch_size
        self.__dict__.update(arrays)
        self.win_off = np.zeros(len(self.rids) + 1, np.int64)
        self.win_off[1:] = np.cumsum(self.n_windows)
        self.row_off = np.zeros(len(self.rows) + 1, np.int64)
        self.row_off[1:] = np.cumsum(self.rows)
        self.sup_off = np.zeros(len(self.rows) + 1, np.int64)
        self.sup_off[1:] = np.cumsum(self.n_sup)
        self.id_off = np.zeros(len(self.rows) + 1, np.int64)
        self.id_off[1:] = np.cumsum(self.n_ids)

    def window(self, w: int) -> dict:
        """Window w of the window order: L, n_alns, bases, quals, supported, sup_rows and ids, the fields of debug_window."""
        r0, r1, s0, s1 = self.row_off[w], self.row_off[w + 1], self.sup_off[w], self.sup_off[w + 1]
        return dict(L=int(self.rows[w]), n_alns=int(self.n_alns[w]), bases=self.bases[r0:r1], quals=self.quals[r0:r1],
                    supported=self.supported[s0:s1], sup_rows=self.indices[s0:s1], ids=self.ids[self.id_off[w]:self.id_off[w + 1]])

    def batches(self):
        """Yields the reference batches in order as (windows, bases [B, Lmax, 31], quals [B, Lmax, 31], lens [B] i32, indices: B arrays
        of i32 rows): the arguments of Context.forward_batch, or of a TorchScript module after the conversion inference() makes.
        `windows` are the batch's windows as indices into the window order."""
        if not hasattr(self, "batch_B"):
            raise ValueError("features_batch(..., batches=True) collates the reference batches")
        r = s = 0
        for B, lmax in zip(self.batch_B, self.batch_Lmax):
            B, lmax = int(B), int(lmax)
            wins = [int(w) for w in self.batch_win[s:s + B]]
            n = B * lmax
            bases = self.batch_bases[r:r + n].reshape(B, lmax, 31)
            quals = self.batch_quals[r:r + n].reshape(B, lmax, 31)
            lens = np.array([int(self.n_sup[w]) for w in wins], np.int32)
            yield wins, bases, quals, lens, [self.indices[self.sup_off[w]:self.sup_off[w + 1]] for w in wins]
            r += n
            s += B

    def consensus_args(self, bases_logits):
        """The arguments of Context.consensus_batch for these targets.  bases_logits: one [n_sup, 5] row per supported entry in the
        window order - an [S, 5] array or tensor, or, as the model returns them, a list with the logits of each batch of batches()
        (each [sum lens, 5], or a list of B per-window pieces): the batches hold every window with supported positions once, in the
        window order."""
        if isinstance(bases_logits, (list, tuple)):
            flat = []
            for x in bases_logits:
                flat.extend(x if isinstance(x, (list, tuple)) else [x])
            if type(flat[0] if flat else self.bases).__module__.split(".")[0] == "torch":
                import torch
                bases_logits = (torch.cat([x.reshape(-1, 5) for x in flat]).float().contiguous() if flat else
                                torch.zeros((0, 5), dtype=torch.float32, device=self.bases.device))
            else:
                bases_logits = np.ascontiguousarray(np.concatenate([np.asarray(x).reshape(-1, 5) for x in flat]) if flat else
                                                    np.zeros((0, 5)), dtype=np.float32)
        return (self.n_windows, self.rows, self.n_alns, self.bases, _split(self.supported, self.n_sup), bases_logits)


@dataclass
class _Packed:
    n: int
    lens: np.ndarray   # u32 [n]
    words: np.ndarray  # u64, all reads
    woff: np.ndarray   # u64 [n+1]
    quals: np.ndarray  # u8, all reads
    wp: np.ndarray     # u64 [n]: address of each read's words
    qp: np.ndarray     # u64 [n]: address of each read's qualities


def _pack_reads(seqs, quals, off) -> _Packed:
    """Concatenated ASCII / Phred+33 bytes with off[n+1] -> the HAECSeq layout (as get_reads packs it, src/haec_io.rs:56) and the
    per-read pointer arrays hb_upload_reads and hb_read_store_create take."""
    n = len(off) - 1
    lens = np.diff(off).astype(np.uint32)
    woff = np.zeros(n + 1, dtype=np.uint64)
    woff[1:] = np.cumsum((lens.astype(np.uint64) + 31) // 32)
    words = np.zeros(int(woff[-1]) + 1, dtype=np.uint64)
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    off64 = np.ascontiguousarray(off, dtype=np.uint64)
    if _host_lib().hbh_pack_2bit(seqs.ctypes.data, off64.ctypes.data, n, words.ctypes.data, woff.ctypes.data,
                                 min(os.cpu_count() or 1, 32)) != 0:
        raise ValueError("non-ACGT base: the reference's 2-bit packing is undefined for it (SURVEY.md H12)")
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    wp = (words.ctypes.data + woff[:-1] * 8).astype(np.uint64)
    qp = (quals.ctypes.data + off64[:-1]).astype(np.uint64)
    return _Packed(n, lens, words, woff, quals, wp, qp)


class ReadStore:
    """The reads in pinned, device-mapped host memory (hb_read_store_create), for read sets larger than a GPU's memory: attach it to
    any number of contexts on any devices (Context.attach_read_store) instead of uploading a copy to each.  Arguments as
    Context.upload_reads.  close() frees it; it fails (HerroError, HB_ERR_STATE) while a context is still attached."""

    def __init__(self, seqs: np.ndarray, quals: np.ndarray, off: np.ndarray):
        p = _pack_reads(seqs, quals, off)
        self._init(p.n, p.wp.ctypes.data, p.lens, p.qp.ctypes.data)

    @classmethod
    def _create(cls, n, word_ptrs, lens_ptr, qual_ptrs):
        """From the per-read pointer arrays of a packed store (hostio.Reads.host_store)."""
        self = cls.__new__(cls)
        lens = np.ctypeslib.as_array(C.cast(lens_ptr, C.POINTER(C.c_uint32)), (n,)).copy() if n else np.zeros(0, np.uint32)
        self._init(n, word_ptrs, lens, qual_ptrs, lens_ptr)
        return self

    def _init(self, n, word_ptrs, lens, qual_ptrs, lens_ptr=None):
        self._L = load_library()
        self._h = C.c_void_p()
        self.n = n
        self.lens = lens
        rc = self._L.hb_read_store_create(C.byref(self._h), n, word_ptrs, lens_ptr if lens_ptr is not None else lens.ctypes.data,
                                          qual_ptrs)
        if rc != 0:
            raise HerroError(rc, self._L.hb_last_error(None).decode())

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            rc = self._L.hb_read_store_destroy(self._h)
            if rc != 0:
                raise HerroError(rc, self._L.hb_last_error(None).decode())
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context:
    """One per GPU — the per-device worker group of src/lib.rs:154-200."""

    def __init__(self, model_path, device: int = 0, window_size: int = 4096, batch_size: int = 64,
                 launch_targets: int = 0, keep_debug: bool = False):
        """model_path None: a context without weights (HB_FLAG_NO_MODEL), for features_batch and consensus_batch around a model
        the caller runs itself."""
        self._L = load_library()
        self._h = C.c_void_p()
        opt = HbOptions(C.sizeof(HbOptions), window_size, batch_size, launch_targets,
                        (HB_FLAG_KEEP_DEBUG if keep_debug else 0) | (HB_FLAG_NO_MODEL if model_path is None else 0))
        rc = self._L.hb_create(C.byref(self._h), device, None if model_path is None else model_path.encode(), C.byref(opt))
        if rc != 0:
            raise HerroError(rc, self._L.hb_last_error(None).decode())
        self.window_size = window_size
        self.batch_size = batch_size
        self.device = device
        self._keep = []
        self.read_len = None
        self.failed = []
        self._store = None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.hb_destroy(self._h)
            self._h = C.c_void_p()
        self._store = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise HerroError(rc, self._L.hb_last_error(self._h).decode())
        return rc

    # -- read store ---------------------------------------------------------------------
    def upload_reads(self, seqs: np.ndarray, quals: np.ndarray, off: np.ndarray):
        """seqs/quals: concatenated ASCII / Phred+33 bytes, off[n+1].  Packs to the HAECSeq
        layout on the host (as get_reads does, src/haec_io.rs:56) and replicates it on the GPU."""
        p = _pack_reads(seqs, quals, off)
        self._check(self._L.hb_upload_reads(self._h, p.n, p.wp.ctypes.data, p.lens.ctypes.data, p.qp.ctypes.data))
        self.read_len = p.lens
        self.packed_words, self.packed_word_off = p.words, p.woff
        self._store = None

    def attach_read_store(self, store: "ReadStore"):
        """Use a read store in pinned host memory instead of an uploaded copy (hb_attach_read_store): each launch gathers only its
        own reads over PCIe.  The context keeps a reference to the store, so the store outlives it."""
        if not isinstance(store, ReadStore) or not store._h.value:
            raise TypeError("store must be an open ReadStore")
        self._check(self._L.hb_attach_read_store(self._h, store._h))
        self._store = store
        self.read_len = store.lens

    # -- submission ---------------------------------------------------------------------
    @staticmethod
    def make_overlaps(ovl9: np.ndarray, cigars: np.ndarray, cig_off: np.ndarray) -> np.ndarray:
        """hb_overlap[] whose cigar pointers reference `cigars` (must stay alive until submit returns)."""
        ovl9 = np.asarray(ovl9, dtype=np.uint32).reshape(-1, 9)
        n = ovl9.shape[0]
        o = np.zeros(n, dtype=OVERLAP_DTYPE)
        for k, name in enumerate(OVERLAP_DTYPE.names[:9]):
            o[name] = ovl9[:, k]
        cig_off = np.asarray(cig_off, dtype=np.uint64)
        o["cigar"] = cigars.ctypes.data + cig_off[:-1]
        o["cigar_len"] = (cig_off[1:] - cig_off[:-1]).astype(np.uint32)
        return o

    def submit_alignments(self, rid: int, overlaps: np.ndarray):
        """`(tid, Vec<Alignment>)` as alignment_reader sends it (src/overlaps.rs:371-373)."""
        self._check(self._L.hb_submit_alignments(self._h, rid, overlaps.ctypes.data, len(overlaps)))

    def submit_target(self, rid: int, n_windows: int, overlaps: np.ndarray, windows: np.ndarray):
        """Target with host-computed OverlapWindows (the Rust host keeps extract_windows)."""
        windows = np.ascontiguousarray(windows, dtype=OVERLAP_WINDOW_DTYPE)
        self._check(self._L.hb_submit_target(self._h, rid, n_windows, overlaps.ctypes.data, len(overlaps),
                                             windows.ctypes.data, len(windows)))

    def flush(self):
        self._check(self._L.hb_flush(self._h))

    # -- the model call alone -----------------------------------------------------------
    def forward_batch(self, bases, quals, lens, indices):
        """The reference's inference() (src/inference.rs:147-175) on one collated batch (hb_forward_batch), with the arguments of
        oracle/forward_ref.run_batch: bases / quals [B, Lmax, 31] u8 (tokens / raw quality bytes), lens [B], indices: B sequences
        of rows.  numpy arrays are read from host memory; torch.uint8 CUDA tensors on the context's device are read in place,
        after the work already queued on torch's current stream.  -> (info logits, bases logits), each a list of B arrays split
        by lens: numpy float32 arrays, or CUDA tensors for CUDA inputs."""
        on_device = type(bases).__module__.split(".")[0] == "torch"
        if on_device:
            import torch
            for name, t in (("bases", bases), ("quals", quals)):
                if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or not t.is_cuda:
                    raise TypeError(f"{name} must be a torch.uint8 CUDA tensor (or both numpy uint8 arrays)")
                if t.device.index != self.device:
                    raise ValueError(f"{name} is on {t.device}, the context on cuda:{self.device}")
                if not t.is_contiguous():
                    raise ValueError(f"{name} must be contiguous")
        else:
            for name, a in (("bases", bases), ("quals", quals)):
                if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
                    raise TypeError(f"{name} must be a numpy uint8 array (or both torch.uint8 CUDA tensors)")
                if not a.flags.c_contiguous:
                    raise ValueError(f"{name} must be C-contiguous")
        shape = tuple(bases.shape)
        if len(shape) != 3 or shape[2] != 31 or tuple(quals.shape) != shape:
            raise ValueError(f"bases and quals must both be [B, Lmax, 31], got {tuple(bases.shape)} and {tuple(quals.shape)}")
        B, Lmax = int(shape[0]), int(shape[1])
        lens = np.ascontiguousarray(np.asarray(lens), dtype=np.int32).reshape(-1)
        if len(lens) != B or len(indices) != B:
            raise ValueError(f"lens and indices must have B = {B} entries, got {len(lens)} and {len(indices)}")
        idx = [np.asarray(i, dtype=np.int32).reshape(-1) for i in indices]
        for b, i in enumerate(idx):
            if len(i) != lens[b]:
                raise ValueError(f"window {b}: lens says {int(lens[b])} positions, indices has {len(i)}")
        flat = np.ascontiguousarray(np.concatenate(idx) if idx else np.zeros(0, np.int32), dtype=np.int32)
        n = len(flat)
        sizes = [int(x) for x in lens]
        if on_device:
            info = torch.empty(max(n, 1), dtype=torch.float32, device=bases.device)
            bl = torch.empty((max(n, 1), 5), dtype=torch.float32, device=bases.device)
            stream = torch.cuda.current_stream(bases.device).cuda_stream
            self._check(self._L.hb_forward_batch(self._h, B, Lmax, bases.data_ptr(), quals.data_ptr(), lens.ctypes.data, flat.ctypes.data,
                                                 info.data_ptr(), bl.data_ptr(), HB_FWD_DEVICE_PTRS, stream))
            return list(torch.split(info[:n], sizes)), list(torch.split(bl[:n], sizes))
        info = np.zeros(max(n, 1), np.float32)
        bl = np.zeros((max(n, 1), 5), np.float32)
        self._check(self._L.hb_forward_batch(self._h, B, Lmax, bases.ctypes.data, quals.ctypes.data, lens.ctypes.data, flat.ctypes.data,
                                             info.ctypes.data, bl.ctypes.data, 0, None))
        cut = np.cumsum(sizes)[:-1]
        return np.split(info[:n], cut), np.split(bl[:n], cut)

    # -- consensus alone ----------------------------------------------------------------
    def consensus_batch(self, n_windows, rows, n_alns, bases, supported, bases_logits):
        """The reference's consensus() (src/consensus.rs:86-227) on the windows of several reads (hb_consensus_batch).
        n_windows: windows per read (all of a read's windows, in wid order); rows, n_alns: per window; bases [sum rows, 31] u8
        tokens, window after window; supported: per window a [n, 2] array of (pos, ins); bases_logits [sum n, 5] f32, one row per
        supported entry in the same order.  bases and bases_logits are both numpy arrays, or both CUDA tensors on the context's
        device (read after the work already queued on torch's current stream).  -> per read, a list of bytes segments (empty: the
        read gets no record)."""
        on_device = type(bases).__module__.split(".")[0] == "torch"
        if on_device:
            import torch
            for name, t, dt in (("bases", bases, torch.uint8), ("bases_logits", bases_logits, torch.float32)):
                if not isinstance(t, torch.Tensor) or t.dtype != dt or not t.is_cuda:
                    raise TypeError(f"{name} must be a {dt} CUDA tensor (or both numpy arrays)")
                if t.device.index != self.device:
                    raise ValueError(f"{name} is on {t.device}, the context on cuda:{self.device}")
                if not t.is_contiguous():
                    raise ValueError(f"{name} must be contiguous")
        else:
            for name, a, dt in (("bases", bases, np.uint8), ("bases_logits", bases_logits, np.float32)):
                if not isinstance(a, np.ndarray) or a.dtype != dt:
                    raise TypeError(f"{name} must be a numpy {np.dtype(dt).name} array (or both CUDA tensors)")
                if not a.flags.c_contiguous:
                    raise ValueError(f"{name} must be C-contiguous")

        def counts(name, x, hi):
            a = np.asarray(x).reshape(-1)
            if a.size and (a.dtype.kind not in "iu" or int(a.min()) < 0 or int(a.max()) > hi):
                raise ValueError(f"{name} must hold integers in [0, {hi}]")
            return np.ascontiguousarray(a, dtype=np.uint8 if hi == 255 else np.uint32)

        nwin = counts("n_windows", n_windows, 0xffffffff)
        W = int(nwin.sum())
        rows_a, nal = counts("rows", rows, 0xffffffff), counts("n_alns", n_alns, 255)
        if len(rows_a) != W or len(nal) != W or len(supported) != W:
            raise ValueError(f"rows, n_alns and supported must have one entry per window ({W}), got {len(rows_a)}, {len(nal)} and {len(supported)}")
        sup = [counts("supported", s, 0xffffffff).reshape(-1, 2) if np.asarray(s).size else np.zeros((0, 2), np.uint32) for s in supported]
        for w, s in enumerate(supported):
            if np.asarray(s).size and np.asarray(s).shape[-1] != 2:
                raise ValueError(f"supported[{w}] must be [n, 2] (pos, ins), got {np.asarray(s).shape}")
        nsup = np.array([len(s) for s in sup], dtype=np.uint32)
        N, S = int(rows_a.astype(np.uint64).sum()), int(nsup.sum())
        if tuple(bases.shape) != (N, 31):
            raise ValueError(f"bases must be [sum rows = {N}, 31], got {tuple(bases.shape)}")
        if tuple(bases_logits.shape) != (S, 5):
            raise ValueError(f"bases_logits must be [sum supported = {S}, 5], got {tuple(bases_logits.shape)}")
        flat = np.ascontiguousarray(np.concatenate(sup) if sup else np.zeros((0, 2), np.uint32), dtype=np.uint32)
        n_reads = len(nwin)
        seqs = np.zeros(max(N, 1), np.uint8)
        seg_len = np.zeros(max(W, 1), np.uint32)
        n_segs = np.zeros(max(n_reads, 1), np.uint32)
        keep = [nwin, rows_a, nal, nsup, flat]
        ptrs = [a.ctypes.data if a.size else np.zeros(1, np.uint32).ctypes.data for a in keep]
        keep.append(ptrs)
        if on_device:  # an empty tensor may have no storage: the library wants a pointer of the device all the same
            b = bases if N else torch.zeros((1, 31), dtype=torch.uint8, device=bases.device)
            bl = bases_logits if S else torch.zeros((1, 5), dtype=torch.float32, device=bases.device)
            stream = torch.cuda.current_stream(bases.device).cuda_stream
            self._check(self._L.hb_consensus_batch(self._h, n_reads, ptrs[0], ptrs[1], ptrs[2], b.data_ptr(), ptrs[3], ptrs[4],
                                                   bl.data_ptr(), seqs.ctypes.data, seg_len.ctypes.data, n_segs.ctypes.data,
                                                   HB_CONS_DEVICE_PTRS, stream))
        else:
            b = bases if N else np.zeros((1, 31), np.uint8)
            bl = bases_logits if S else np.zeros((1, 5), np.float32)
            self._check(self._L.hb_consensus_batch(self._h, n_reads, ptrs[0], ptrs[1], ptrs[2], b.ctypes.data, ptrs[3], ptrs[4],
                                                   bl.ctypes.data, seqs.ctypes.data, seg_len.ctypes.data, n_segs.ctypes.data, 0, None))
        out, s, o = [], 0, 0
        for i in range(n_reads):
            segs = []
            for _ in range(int(n_segs[i])):
                segs.append(seqs[o:o + int(seg_len[s])].tobytes())
                o += int(seg_len[s])
                s += 1
            out.append(segs)
        return out

    # -- the features stage alone -------------------------------------------------------
    def features_batch(self, targets, device: bool = False, batches: bool = False) -> Features:
        """extract_features (src/features.rs:326-583) on many targets (hb_features_batch + hb_features_fetch): targets is a list of
        (rid, overlaps), overlaps as make_overlaps builds them (`(tid, Vec<Alignment>)`).  device: the bulk arrays (bases, quals,
        batch_bases, batch_quals) become torch.uint8 tensors on the context's device, written on torch's current stream; batches:
        also collate the reference batches of `-b` (batch_size) windows.  -> Features."""
        if not isinstance(device, bool) or not isinstance(batches, bool):
            raise TypeError("device and batches must be bools")
        targets = list(targets)
        rids = np.zeros(len(targets), np.uint32)
        ovs = []
        for k, t in enumerate(targets):
            if not isinstance(t, (tuple, list)) or len(t) != 2:
                raise TypeError(f"targets[{k}] must be a (rid, overlaps) pair")
            rid, o = t
            if isinstance(rid, (bool, np.bool_)) or not isinstance(rid, (int, np.integer)) or not 0 <= int(rid) < 2 ** 32:
                raise ValueError(f"targets[{k}]: rid must be an integer in [0, 2^32), got {rid!r}")
            if not isinstance(o, np.ndarray) or o.dtype != OVERLAP_DTYPE or o.ndim != 1:
                raise TypeError(f"targets[{k}]: overlaps must be a 1-D OVERLAP_DTYPE array (Context.make_overlaps)")
            rids[k] = int(rid)
            ovs.append(o)
        n_ovl = np.array([len(o) for o in ovs], np.uint32)
        ovl = np.zeros(int(n_ovl.sum()), OVERLAP_DTYPE)  # not np.concatenate: its dtype promotion packs the padded hb_overlap layout
        o0 = 0
        for o in ovs:
            ovl[o0:o0 + len(o)] = o
            o0 += len(o)
        L = self._L
        sh = HbFeaturesShape()
        self._check(L.hb_features_batch(self._h, len(rids), rids.ctypes.data, n_ovl.ctypes.data, ovl.ctypes.data if len(ovl) else None,
                                        C.byref(sh)))
        nt, nw, nb, N, S, NI, NB = sh.n_targets, sh.n_windows, sh.n_batches, sh.n_rows, sh.n_sup, sh.n_ids, sh.n_batch_rows
        a = dict(status=np.zeros(max(nt, 1), np.int32), n_windows=np.zeros(max(nt, 1), np.uint32), rows=np.zeros(max(nw, 1), np.uint32),
                 n_alns=np.zeros(max(nw, 1), np.uint8), n_sup=np.zeros(max(nw, 1), np.uint32), n_ids=np.zeros(max(nw, 1), np.uint32),
                 supported=np.zeros((max(S, 1), 2), np.uint32), indices=np.zeros(max(S, 1), np.int32), ids=np.zeros(max(NI, 1), np.uint32))
        if device:
            import torch
            dev = torch.device("cuda", self.device)
            bulk = lambda n: torch.empty((max(n, 1), 31), dtype=torch.uint8, device=dev)  # noqa: E731
        else:
            bulk = lambda n: np.empty((max(n, 1), 31), np.uint8)  # noqa: E731
        a["bases"], a["quals"] = bulk(N), bulk(N)
        if batches:
            nslots = 0  # sum B, known once batch_B is fetched
            a["batch_B"], a["batch_Lmax"] = np.zeros(max(nb, 1), np.uint32), np.zeros(max(nb, 1), np.uint32)
            a["batch_bases"], a["batch_quals"] = bulk(NB), bulk(NB)
            o = HbFeaturesOut(C.sizeof(HbFeaturesOut))
            o.batch_B = a["batch_B"].ctypes.data
            self._check(L.hb_features_fetch(self._h, C.byref(sh), C.byref(o), 0, None))
            nslots = int(a["batch_B"][:nb].sum())
            a["batch_win"] = np.zeros(max(nslots, 1), np.uint32)
        o = HbFeaturesOut(C.sizeof(HbFeaturesOut))
        for name, x in a.items():
            setattr(o, name, x.data_ptr() if device and name in ("bases", "quals", "batch_bases", "batch_quals") else x.ctypes.data)
        stream = torch.cuda.current_stream(dev).cuda_stream if device else None
        self._check(L.hb_features_fetch(self._h, C.byref(sh), C.byref(o), HB_FEAT_DEVICE_PTRS if device else 0, stream))
        size = dict(status=nt, n_windows=nt, rows=nw, n_alns=nw, n_sup=nw, n_ids=nw, bases=N, quals=N, supported=S, indices=S, ids=NI,
                    batch_B=nb, batch_Lmax=nb, batch_bases=NB, batch_quals=NB)
        if batches:
            size["batch_win"] = nslots
        a = {k: v[:size[k]] for k, v in a.items()}
        self.last_features_shape = sh
        return Features([int(r) for r in rids], a, self.batch_size)

    def set_launch_targets(self, n: int):
        self._check(self._L.hb_set_launch_targets(self._h, n))

    def set_kernel_timing(self, on: bool):
        self._check(self._L.hb_set_kernel_timing(self._h, 1 if on else 0))

    def bind_calling_thread(self) -> bool:
        return self._check(self._L.hb_bind_calling_thread(self._h)) == 1

    def poll(self):
        """-> Corrected or None; raises HerroError (with .rid) for a target that failed (e.g. one the reference would
        have panicked on); the other targets are unaffected and polling can continue."""
        rid = C.c_uint32()
        seqs, seg_len = C.c_void_p(), C.c_void_p()
        n = C.c_uint32()
        rc = self._L.hb_poll_corrected(self._h, C.byref(rid), C.byref(seqs), C.byref(seg_len), C.byref(n))
        if rc == 0:
            return None
        try:
            if rc < 0:
                e = HerroError(rc, self._L.hb_last_error(self._h).decode())
                e.rid = rid.value
                raise e
            lens = np.ctypeslib.as_array(C.cast(seg_len, C.POINTER(C.c_uint32)), (max(n.value, 1),))[:n.value].copy()
            segs, o = [], 0
            for l in lens:
                segs.append(C.string_at(seqs.value + o, int(l)))
                o += int(l)
            return Corrected(rid.value, segs)
        finally:
            if seqs.value:
                self._L.hb_release_result(self._h, seqs)

    def drain(self, skip_failed: bool = False):
        """All queued results.  skip_failed: a failed target is recorded in `self.failed` as (rid, code, message) and the
        drain goes on (one bad read must not truncate the output of a whole run)."""
        out = []
        while True:
            try:
                r = self.poll()
            except HerroError as e:
                if not skip_failed:
                    raise
                self.failed.append((getattr(e, "rid", None), e.code, str(e)))
                continue
            if r is None:
                return out
            out.append(r)

    # -- counters / taps ----------------------------------------------------------------
    def stats(self) -> dict:
        s = HbStats()
        self._check(self._L.hb_get_stats(self._h, C.byref(s)))
        d = {n: getattr(s, n) for n, _ in HbStats._fields_ if n not in ("ms_kernel", "n_kernel", "ms_worker_phase", "class_flops")}
        d["class_flops"] = {k: int(s.class_flops[i]) for i, k in enumerate(KERNEL_CLASSES)}
        d["ms_worker_phase"] = [float(x) for x in s.ms_worker_phase]
        d["ms_kernel"] = {k: s.ms_kernel[i] for i, k in enumerate(KERNEL_CLASSES)}
        d["n_kernel"] = {k: int(s.n_kernel[i]) for i, k in enumerate(KERNEL_CLASSES)}
        return d

    def reset_stats(self):
        self._check(self._L.hb_reset_stats(self._h))

    def debug_window(self, rid: int, wid: int) -> dict:
        sh = (C.c_uint32 * 4)()
        self._check(self._L.hb_debug_window_shape(self._h, rid, wid, sh))
        L, n_alns, ns = int(sh[0]), int(sh[1]), int(sh[2])
        bases = np.zeros((L, 31), np.uint8)
        quals = np.zeros((L, 31), np.uint8)
        sup = np.zeros((max(ns, 1), 2), np.uint32)
        rows = np.zeros(max(ns, 1), np.uint32)
        info = np.zeros(max(ns, 1), np.float32)
        bl = np.zeros((max(ns, 1), 5), np.float32)
        self._check(self._L.hb_debug_dump_window(self._h, rid, wid, bases.ctypes.data, quals.ctypes.data,
                                                 sup.ctypes.data, rows.ctypes.data, info.ctypes.data, bl.ctypes.data))
        return dict(L=L, n_alns=n_alns, bases=bases, quals=quals, supported=sup[:ns], sup_rows=rows[:ns],
                    info_logits=info[:ns], bases_logits=bl[:ns])

    def dump_features(self, rid: int, out_dir: str, read_names: list):
        """`herro features` files of target `rid` (of the most recent launch; keep_debug) under out_dir/<read id>/."""
        if getattr(self, "_names_src", None) is not read_names:
            self._names_src = read_names
            self._names_buf = [n if isinstance(n, bytes) else str(n).encode() for n in read_names]
            self._names_arr = (C.c_char_p * len(read_names))(*self._names_buf)
        self._check(self._L.hb_dump_features(self._h, rid, out_dir.encode(), self._names_arr))

    def replay_last_launch(self, iters: int = 1) -> float:
        ms = C.c_float()
        self._check(self._L.hb_replay_last_launch(self._h, iters, C.byref(ms)))
        return float(ms.value)


# ------------------------------------------------------------------------------------------
# C++ host harness (herro_b200/host/harness.cpp): the Rust binary's thread topology over the C ABI
# ------------------------------------------------------------------------------------------
_host = None


def _host_lib():
    global _host
    if _host is None:
        load_library()
        H = C.CDLL(HOST_LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        H.hbh_pack_2bit.argtypes = [vp, vp, u32, vp, vp, C.c_int]
        H.hbh_windowing.argtypes = [vp, vp, vp, u32, u32, u32, C.c_int, vp, vp, C.c_uint64]
        H.hbh_run.argtypes = [vp, vp, vp, vp, u32, u32, u32, C.c_int, vp, vp, vp, vp, vp, vp]
        _host = H
    return _host


class HostHarness:
    """Feature threads + consumer thread over one Context, like src/lib.rs:154-200 for one device."""

    def __init__(self, ctx: "Context", ovl9: np.ndarray, cigars: np.ndarray, cig_off: np.ndarray, aln_off: np.ndarray,
                 read_len: np.ndarray):
        self.ctx = ctx
        self.cigars = cigars  # keep alive: hb_overlap.cigar points into it
        self.ovl = Context.make_overlaps(ovl9, cigars, cig_off)
        self.aln_off = np.ascontiguousarray(aln_off, dtype=np.uint64)
        self.read_len = np.ascontiguousarray(read_len, dtype=np.uint32)

    def windowing(self, t_begin: int, t_end: int, threads: int):
        H = _host_lib()
        off = np.zeros(t_end - t_begin + 1, dtype=np.uint64)
        rc = H.hbh_windowing(self.ovl.ctypes.data, self.aln_off.ctypes.data, self.read_len.ctypes.data, self.ctx.window_size,
                             t_begin, t_end, threads, off.ctypes.data, None, 0)
        if rc != 0:
            raise HerroError(rc, "windowing failed")
        ow = np.zeros(max(int(off[-1]), 1), dtype=OVERLAP_WINDOW_DTYPE)
        rc = H.hbh_windowing(self.ovl.ctypes.data, self.aln_off.ctypes.data, self.read_len.ctypes.data, self.ctx.window_size,
                             t_begin, t_end, threads, off.ctypes.data, ow.ctypes.data, len(ow))
        if rc != 0:
            raise HerroError(rc, "windowing failed")
        return ow, off

    def run(self, t_begin: int, t_end: int, threads: int, windows=None) -> dict:
        H = _host_lib()
        out3 = np.zeros(4, dtype=np.uint64)
        chk = C.c_uint64()
        sec = C.c_double()
        sub = C.c_double()
        ow_p = windows[0].ctypes.data if windows is not None else None
        off_p = windows[1].ctypes.data if windows is not None else None
        rc = H.hbh_run(self.ctx._h, self.ovl.ctypes.data, self.aln_off.ctypes.data, self.read_len.ctypes.data,
                       self.ctx.window_size, t_begin, t_end, threads, ow_p, off_p, out3.ctypes.data, C.byref(chk), C.byref(sec), C.byref(sub))
        if rc != 0:
            raise HerroError(rc, self.ctx._L.hb_last_error(self.ctx._h).decode())
        return dict(bases=int(out3[0]), records=int(out3[1]), targets=int(out3[2]), failed=int(out3[3]), checksum=int(chk.value),
                    seconds=sec.value, submit_seconds_sum=sub.value)


# ------------------------------------------------------------------------------------------
# FASTA record format of correction_writer / write_sequence (src/lib.rs:267-317)
# ------------------------------------------------------------------------------------------
def fasta_records(read_id: bytes, description, segments: list) -> bytes:
    out = bytearray()
    for i, seg in enumerate(segments):
        out += b">" + read_id
        out += b" " if len(segments) == 1 else b":%d " % i
        if description is not None:
            out += description
        out += b"\n" + seg + b"\n"
    return bytes(out)
