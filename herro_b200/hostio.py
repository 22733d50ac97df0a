"""ctypes view of the native host data plane (herro_b200/host/io.cpp): FASTQ -> packed read store, `--read-alns` batches ->
alignments grouped by target, FASTA writer, and the whole `herro inference` pipeline (hbh_inference).  In the deployed layout
the Rust host owns these stages (haec_io.rs, overlaps.rs, lib.rs); here they are C++ threads over the public C ABI."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

from . import api


def _lib():
    H = api._host_lib()
    if getattr(H, "_io_ready", False):
        return H
    vp, u32 = C.c_void_p, C.c_uint32
    H.hbh_last_error.restype = C.c_char_p
    H.hbh_reads_load.argtypes = [C.c_char_p, u32, vp, u32, vp, u32, C.c_int, C.POINTER(vp)]
    H.hbh_reads_free.argtypes = [vp]
    H.hbh_reads_free.restype = None
    H.hbh_reads_count.argtypes = [vp]
    H.hbh_reads_count.restype = u32
    for f in ("hbh_reads_lens", "hbh_reads_word_ptrs", "hbh_reads_qual_ptrs", "hbh_reads_names"):
        getattr(H, f).argtypes = [vp]
        getattr(H, f).restype = vp
    H.hbh_reads_description.argtypes = [vp, u32]
    H.hbh_reads_description.restype = C.c_char_p
    H.hbh_reads_stats.argtypes = [vp, vp]
    H.hbh_reads_stats.restype = None
    H.hbh_alns_load.argtypes = [C.c_char_p, vp, vp, u32, C.c_int, C.POINTER(vp)]
    H.hbh_alns_free.argtypes = [vp]
    H.hbh_alns_free.restype = None
    H.hbh_alns_targets.argtypes = [vp]
    H.hbh_alns_targets.restype = u32
    for f in ("hbh_alns_target_rids", "hbh_alns_target_offsets", "hbh_alns_overlaps"):
        getattr(H, f).argtypes = [vp]
        getattr(H, f).restype = vp
    H.hbh_alns_stats.argtypes = [vp, vp]
    H.hbh_alns_stats.restype = None
    H.hbh_alns_source.argtypes = [vp]
    H.hbh_alns_source.restype = C.c_char_p
    H.hbh_alns_budget_bytes.argtypes = [vp]
    H.hbh_alns_budget_bytes.restype = C.c_uint64
    H.hbh_alns_default_budget.argtypes = []
    H.hbh_alns_default_budget.restype = C.c_uint64
    H.hbh_alns_stream_open.argtypes = [C.c_char_p, vp, vp, u32, C.c_int, C.c_uint64, C.POINTER(vp)]
    H.hbh_alns_stream_next.argtypes = [vp, C.POINTER(vp)]
    H.hbh_alns_stream_close.argtypes = [vp]
    H.hbh_alns_stream_close.restype = None
    H.hbh_alns_stream_stats.argtypes = [vp, vp, C.POINTER(C.c_double)]
    H.hbh_alns_stream_stats.restype = None
    H.hbh_fasta_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    H.hbh_fasta_write.argtypes = [vp, C.c_char_p, C.c_char_p, vp, vp, u32]
    H.hbh_fasta_close.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    H.hbh_inference.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, u32, u32, C.c_int, vp, C.c_int, vp, u32, vp, u32,
                                C.c_int, C.c_uint64, C.c_uint64, vp, vp]
    H.hbh_reads_store_bytes.argtypes = [vp]
    H.hbh_reads_store_bytes.restype = C.c_uint64
    H.hbh_paf_open.argtypes = [C.c_char_p, vp, C.POINTER(vp)]
    H.hbh_paf_next.argtypes = [vp, u32, C.POINTER(u32)]
    H.hbh_paf_overlaps.argtypes = [vp]
    H.hbh_paf_overlaps.restype = vp
    H.hbh_paf_stats.argtypes = [vp, vp]
    H.hbh_paf_stats.restype = None
    H.hbh_paf_close.argtypes = [vp]
    H.hbh_paf_close.restype = None
    H.hbh_batches_open.argtypes = [C.c_char_p, vp, u32, C.POINTER(vp)]
    H.hbh_batches_write.argtypes = [vp, vp, vp, vp, vp, u32]
    H.hbh_batches_close.argtypes = [vp, vp]
    H.hbh_align.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, u32, u32, u32, u32, C.c_int, vp, vp]
    H._io_ready = True
    return H


def _strs(names):
    if names is None:
        return None, 0, None
    buf = [n if isinstance(n, bytes) else str(n).encode() for n in names]
    arr = (C.c_char_p * len(buf))(*buf)
    return arr, len(buf), buf


class Reads:
    """haec_io::get_reads (src/haec_io.rs:37-75): FASTQ file / directory -> ids, descriptions, 2-bit words, qualities."""

    def __init__(self, path: str, min_len: int = 4096, core=None, neighbour=None, threads: int = 0):
        H = _lib()
        self._H, self._h = H, C.c_void_p()
        ca, nc, self._k1 = _strs(core)
        na, nn, self._k2 = _strs(neighbour)
        rc = H.hbh_reads_load(path.encode(), min_len, ca, nc, na, nn, threads or min(os.cpu_count() or 1, 32), C.byref(self._h))
        if rc != 0:
            raise api.HerroError(rc, H.hbh_last_error().decode())
        self.n = H.hbh_reads_count(self._h)
        n = self.n
        self.lens = np.ctypeslib.as_array(C.cast(H.hbh_reads_lens(self._h), C.POINTER(C.c_uint32)), (n,)) if n else np.zeros(0, np.uint32)
        names = C.cast(H.hbh_reads_names(self._h), C.POINTER(C.c_char_p))
        self.ids = [names[i] for i in range(n)]
        self.descriptions = [H.hbh_reads_description(self._h, i) for i in range(n)]

    def words(self, i) -> np.ndarray:
        p = C.cast(self._H.hbh_reads_word_ptrs(self._h), C.POINTER(C.c_void_p))[i]
        nw = (int(self.lens[i]) + 31) // 32
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), (max(nw, 1),))[:nw].copy()

    def qual(self, i) -> bytes:
        p = C.cast(self._H.hbh_reads_qual_ptrs(self._h), C.POINTER(C.c_void_p))[i]
        return C.string_at(p, int(self.lens[i]))

    def stats(self) -> dict:
        s = np.zeros(4)
        self._H.hbh_reads_stats(self._h, s.ctypes.data)
        return dict(load_s=s[0], pack_s=s[1], skipped_short=int(s[2]), bases=int(s[3]))

    def upload(self, ctx: "api.Context"):
        """hb_upload_reads straight from the packed store (no copy through Python)."""
        H = self._H
        ctx._check(ctx._L.hb_upload_reads(ctx._h, self.n, H.hbh_reads_word_ptrs(self._h), H.hbh_reads_lens(self._h),
                                          H.hbh_reads_qual_ptrs(self._h)))
        ctx.read_len = self.lens.copy()

    def store_bytes(self) -> int:
        """Bytes of the packed store: 2-bit words and one quality byte per base."""
        return int(self._H.hbh_reads_store_bytes(self._h))

    def host_store(self) -> "api.ReadStore":
        """A read store in pinned host memory (hb_read_store_create) straight from the packed store (no copy through Python)."""
        H = self._H
        return api.ReadStore._create(self.n, H.hbh_reads_word_ptrs(self._h), H.hbh_reads_lens(self._h), H.hbh_reads_qual_ptrs(self._h))

    def load_into(self, ctx: "api.Context", device_bytes, read_store=None):
        """The reads into a context as `inference` chooses (host_store_above): uploaded, or attached as a host store, which is
        returned (it must outlive the context)."""
        if self.store_bytes() > host_store_above(device_bytes, read_store):
            store = self.host_store()
            ctx.attach_read_store(store)
            ctx.read_len = self.lens.copy()
            return store
        self.upload(ctx)
        return None

    def close(self):
        if self._h:
            self._H.hbh_reads_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


UNLIMITED = 2 ** 64 - 1  # a budget (bytes) that never holds the alignment reader back


def _budget(budget) -> int:
    """A budget argument -> the reader's: None is the default (1/8 of physical memory), anything else at least one byte."""
    if budget is None:
        return 0
    if int(budget) < 1:
        raise ValueError(f"the alignment budget must be at least 1 byte, got {budget}")
    return min(int(budget), UNLIMITED)


class Alignments:
    """overlaps::read_batches + parse_paf (src/overlaps.rs:288-323,117-202): every batch file, merged in sorted name order (a target
    named in several files appears once per file).  `Alignments.stream` yields the files one at a time instead."""

    def __init__(self, alns_dir: str, reads: Reads, core=None, threads: int = 0):
        H = _lib()
        h = C.c_void_p()
        ca, nc, self._k = _strs(core)
        rc = H.hbh_alns_load(alns_dir.encode(), reads._h, ca, nc, threads or min(os.cpu_count() or 1, 32), C.byref(h))
        if rc != 0:
            raise api.HerroError(rc, H.hbh_last_error().decode())
        self._wrap(H, h, reads)

    @classmethod
    def stream(cls, alns_dir: str, reads: "Reads", core=None, threads: int = 0, budget=None) -> "AlignmentStream":
        """The batch files one at a time, in sorted name order, while `threads` workers decode the next ones within `budget` bytes
        of decompressed text and overlap arrays (None: 1/8 of physical memory).  Iterating yields one Alignments per file; close
        each once its targets are submitted, since files held past the budget stop the workers."""
        return AlignmentStream(alns_dir, reads, core, threads, budget)

    def _wrap(self, H, h, reads):
        self._H, self._h, self.reads = H, h, reads
        nt = H.hbh_alns_targets(h)
        self.n_targets = nt
        self.target_rids = (np.ctypeslib.as_array(C.cast(H.hbh_alns_target_rids(h), C.POINTER(C.c_uint32)), (nt,))
                            if nt else np.zeros(0, np.uint32))
        self.offsets = np.ctypeslib.as_array(C.cast(H.hbh_alns_target_offsets(h), C.POINTER(C.c_uint64)), (nt + 1,))
        na = int(self.offsets[-1])
        buf = (C.c_char * (max(na, 1) * api.OVERLAP_DTYPE.itemsize)).from_address(H.hbh_alns_overlaps(h) or 0) if na else None
        self.overlaps = np.frombuffer(buf, dtype=api.OVERLAP_DTYPE, count=na) if na else np.zeros(0, api.OVERLAP_DTYPE)
        self.source = H.hbh_alns_source(h).decode()   # the batch file of a streamed file, "" when merged
        self.budget_bytes = int(H.hbh_alns_budget_bytes(h))  # what a streamed file holds of its stream's budget

    def target(self, k):
        """-> (rid, hb_overlap[] view) of the k-th target group."""
        return int(self.target_rids[k]), self.overlaps[int(self.offsets[k]):int(self.offsets[k + 1])]

    def cigar(self, a) -> bytes:
        o = self.overlaps[a]
        return C.string_at(int(o["cigar"]), int(o["cigar_len"]))

    def stats(self) -> dict:
        s = np.zeros(6)
        self._H.hbh_alns_stats(self._h, s.ctypes.data)
        return dict(decode_s_sum=s[0], parse_s_sum=s[1], lines=int(s[2]), kept=int(s[3]), compressed_bytes=int(s[4]), text_bytes=int(s[5]))

    def close(self):
        if self._h:
            self._H.hbh_alns_free(self._h)
            self._h = C.c_void_p()
            self.overlaps = np.zeros(0, api.OVERLAP_DTYPE)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AlignmentStream:
    """hbh_alns_stream_*: an iterator of Alignments, one per batch file (see Alignments.stream)."""

    def __init__(self, alns_dir: str, reads: Reads, core=None, threads: int = 0, budget=None):
        H = _lib()
        self._H, self._h, self.reads = H, C.c_void_p(), reads
        ca, nc, self._k = _strs(core)
        rc = H.hbh_alns_stream_open(alns_dir.encode(), reads._h, ca, nc, threads or min(os.cpu_count() or 1, 32), _budget(budget),
                                    C.byref(self._h))
        if rc != 0:
            raise api.HerroError(rc, H.hbh_last_error().decode())

    def __iter__(self):
        return self

    def __next__(self) -> Alignments:
        if not self._h:
            raise StopIteration
        h = C.c_void_p()
        rc = self._H.hbh_alns_stream_next(self._h, C.byref(h))
        if rc != 0:
            raise api.HerroError(rc, self._H.hbh_last_error().decode())
        if not h:
            raise StopIteration
        a = Alignments.__new__(Alignments)
        a._k = None
        a._wrap(self._H, h, self.reads)
        return a

    def stats(self) -> dict:
        c = np.zeros(6, np.uint64)
        t = C.c_double()
        self._H.hbh_alns_stream_stats(self._h, c.ctypes.data, C.byref(t))
        return dict(peak_bytes=int(c[0]), in_flight_bytes=int(c[1]), budget_bytes=int(c[2]), files=int(c[3]), files_parsed=int(c[4]),
                    peak_files=int(c[5]), ingest_s=t.value)

    def close(self):
        if self._h:
            self._H.hbh_alns_stream_close(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FastaWriter:
    """correction_writer / write_sequence (src/lib.rs:267-317)."""

    def __init__(self, path: str):
        H = _lib()
        self._H, self._h = H, C.c_void_p()
        if H.hbh_fasta_open(path.encode(), C.byref(self._h)) != 0:
            raise api.HerroError(-1, H.hbh_last_error().decode())

    def write(self, read_id: bytes, description, segments: list):
        seq = b"".join(segments)
        lens = np.array([len(s) for s in segments], dtype=np.uint32)
        buf = np.frombuffer(seq, dtype=np.uint8) if seq else np.zeros(1, np.uint8)
        self._H.hbh_fasta_write(self._h, read_id, description, buf.ctypes.data, lens.ctypes.data, len(segments))

    def close(self):
        rec, bases = C.c_uint64(), C.c_uint64()
        if self._h:
            self._H.hbh_fasta_close(self._h, C.byref(rec), C.byref(bases))
            self._h = C.c_void_p()
        return rec.value, bases.value


# ------------------------------------------------------------------------------------------
# `herro features` directories (src/features.rs:724-764) -> the reference's model batches (src/inference.rs:73-140,222-268)
# ------------------------------------------------------------------------------------------
BASES_MAP = np.full(256, 255, dtype=np.uint8)  # src/inference.rs:23-31: ASCII -> token, 255 elsewhere
for _tok, _ch in enumerate(b"ACGT*acgt#."):
    BASES_MAP[_ch] = _tok
TOK_GAP = 4          # BASES_MAP['*']: a row whose target column holds it is an insertion row
BASE_PADDING, QUAL_PADDING = 11, 126  # src/inference.rs:15-17


@dataclass
class FeatureBatch:
    """One collated reference batch of a read: the arguments of inference() (src/inference.rs:147-175)."""
    read: str
    wids: list           # [B] window ids, the batch's window order
    bases: np.ndarray    # [B, Lmax, 31] u8 tokens, padded with 11
    quals: np.ndarray    # [B, Lmax, 31] u8 quality bytes, padded with 126
    lens: np.ndarray     # [B] i32 supported positions per window
    indices: list        # B arrays of i32 rows: target_rows[pos] + ins


FEATURE_ASCII = np.frombuffer(b"ACGT*acgt#..", dtype=np.uint8)  # BASES_MAP inverted; token 11 (and anything above) as '.'
SUPPORTED_DTYPE = np.dtype([("pos", "<u2"), ("ins", "u1")])    # SupportedPos (src/features.rs:894-898)


def write_feature_window(read_dir: str, wid: int, tokens, quals, supported, id_names):
    """The `herro features` files of one window (src/features.rs:724-764,806-839) under read_dir: <wid>.features.npy (u8 [2, L, 31]:
    plane 0 the pileup as ASCII, plane 1 the qualities), <wid>.supported.npy (SupportedPos records) and <wid>.ids.txt (one read
    name per surviving overlap, in final rank order), written with numpy's .npy writer.  tokens / quals [L, 31] u8, supported
    [n, 2] (pos, ins), id_names: bytes."""
    os.makedirs(read_dir, exist_ok=True)
    tokens = np.asarray(tokens, dtype=np.uint8)
    feats = np.stack([FEATURE_ASCII[np.minimum(tokens, 11)], np.asarray(quals, dtype=np.uint8)]).astype(np.uint8)
    np.save(os.path.join(read_dir, f"{wid}.features.npy"), feats)
    sup_in = np.asarray(supported).reshape(-1, 2)
    sup = np.zeros(len(sup_in), dtype=SUPPORTED_DTYPE)
    sup["pos"] = sup_in[:, 0]
    sup["ins"] = sup_in[:, 1]
    np.save(os.path.join(read_dir, f"{wid}.supported.npy"), sup)
    with open(os.path.join(read_dir, f"{wid}.ids.txt"), "wb") as f:
        f.write(b"".join(n + b"\n" for n in id_names))


def read_feature_window(read_dir: str, wid: int):
    """-> (tokens [L, 31] u8, quals [L, 31] u8, indices [n] i32) of one window of a `herro features` read directory."""
    feats = np.load(os.path.join(read_dir, f"{wid}.features.npy"))
    sup = np.load(os.path.join(read_dir, f"{wid}.supported.npy"))
    if feats.ndim != 3 or feats.shape[0] != 2 or feats.shape[2] != 31:
        raise ValueError(f"{read_dir}/{wid}.features.npy: expected [2, L, 31], got {feats.shape}")
    tok = BASES_MAP[feats[0]]
    target_rows = np.flatnonzero(tok[:, 0] != TOK_GAP)                   # get_target_indices (:255-268)
    idx = target_rows[sup["pos"].astype(np.int64)] + sup["ins"].astype(np.int64)  # (:136-140)
    return tok, np.ascontiguousarray(feats[1]), idx.astype(np.int32)


def read_feature_batches(read_dir: str, batch_size: int):
    """The model batches of one read directory, in the order the reference runs them: the windows in wid order are taken `batch_size`
    at a time, as FeaturesOutput::update hands them over (src/features.rs:884-893); the windows of such a group with at least one
    supported position form one batch (prepare_examples, src/inference.rs:241-250), padded to its longest window (collate, :73-97)."""
    wids = sorted(int(f[:-len(".features.npy")]) for f in os.listdir(read_dir) if f.endswith(".features.npy"))
    read = os.path.basename(os.path.normpath(read_dir))
    out = []
    for g0 in range(0, len(wids), batch_size):
        wins = [(w,) + read_feature_window(read_dir, w) for w in wids[g0:g0 + batch_size]]
        wins = [w for w in wins if len(w[3]) > 0]
        if not wins:
            continue
        lmax = max(w[1].shape[0] for w in wins)
        bases = np.full((len(wins), lmax, 31), BASE_PADDING, dtype=np.uint8)
        quals = np.full((len(wins), lmax, 31), QUAL_PADDING, dtype=np.uint8)
        for b, (_, tok, q, _) in enumerate(wins):
            bases[b, :tok.shape[0]] = tok
            quals[b, :q.shape[0]] = q
        out.append(FeatureBatch(read, [w[0] for w in wins], bases, quals, np.array([len(w[3]) for w in wins], dtype=np.int32),
                                [w[3] for w in wins]))
    return out


@dataclass
class ConsensusWindow:
    """What consensus() reads of a ConsensusWindow (src/consensus.rs:22-33)."""
    wid: int
    n_alns: int
    bases: np.ndarray         # [L, 31] u8 tokens
    supported: np.ndarray     # [n, 2] u32 (pos, ins)
    bases_logits: np.ndarray  # [n, 5] f32


def read_consensus_windows(features_read_dir: str, logits_read_dir: str):
    """A read's ConsensusWindows in wid order, rebuilt from a `herro features` read directory (tokens from plane 0 through BASES_MAP,
    n_alns = min(lines of <wid>.ids.txt, 30) as src/features.rs:877 sets it, (pos, ins) from <wid>.supported.npy) and the `predict`
    output of the same read (<wid>.bases_logits.npy, required exactly for the windows with supported positions).  The wids must be
    0 .. n-1: consensus_worker waits for all n_total_wins windows of a read (src/consensus.rs:249)."""
    wids = sorted(int(f[:-len(".features.npy")]) for f in os.listdir(features_read_dir) if f.endswith(".features.npy"))
    missing = sorted(set(range(len(wids))) - set(wids))
    if missing or (wids and wids[-1] != len(wids) - 1):
        gap = missing[0] if missing else len(wids)
        raise ValueError(f"{features_read_dir}: window {gap} is missing (the windows must be 0 .. n-1; found {len(wids)} up to {wids[-1]})")
    out = []
    for wid in wids:
        feats = np.load(os.path.join(features_read_dir, f"{wid}.features.npy"))
        if feats.ndim != 3 or feats.shape[0] != 2 or feats.shape[2] != 31:
            raise ValueError(f"{features_read_dir}/{wid}.features.npy: expected [2, L, 31], got {feats.shape}")
        sup = np.load(os.path.join(features_read_dir, f"{wid}.supported.npy"))
        with open(os.path.join(features_read_dir, f"{wid}.ids.txt"), "rb") as f:
            n_ids = sum(1 for line in f if line.strip())
        supported = np.stack([sup["pos"].astype(np.uint32), sup["ins"].astype(np.uint32)], axis=1) if len(sup) else np.zeros((0, 2), np.uint32)
        if len(sup):
            p = os.path.join(logits_read_dir, f"{wid}.bases_logits.npy")
            if not os.path.exists(p):
                raise ValueError(f"{p} is missing: window {wid} has {len(sup)} supported positions")
            bl = np.load(p)
            if bl.shape != (len(sup), 5):
                raise ValueError(f"{p}: expected [{len(sup)}, 5], got {bl.shape}")
            bl = np.ascontiguousarray(bl, dtype=np.float32)
        else:
            bl = np.zeros((0, 5), np.float32)
        out.append(ConsensusWindow(wid, min(n_ids, 30), BASES_MAP[feats[0]], np.ascontiguousarray(supported), bl))
    return out


def consensus_args(reads):
    """The arguments of Context.consensus_batch for several reads, each a list of ConsensusWindow in wid order."""
    wins = [w for r in reads for w in r]
    bases = np.concatenate([w.bases for w in wins]) if wins else np.zeros((0, 31), np.uint8)
    bl = np.concatenate([w.bases_logits for w in wins]) if wins else np.zeros((0, 5), np.float32)
    return ([len(r) for r in reads], [w.bases.shape[0] for w in wins], [w.n_alns for w in wins], np.ascontiguousarray(bases),
            [w.supported for w in wins], np.ascontiguousarray(bl, dtype=np.float32))


def feature_reads(features_dir: str):
    """The read directories of a `herro features` output directory (those holding window files), sorted by name."""
    return [os.path.join(features_dir, d) for d in sorted(os.listdir(features_dir))
            if os.path.isdir(os.path.join(features_dir, d)) and any(f.endswith(".features.npy") for f in os.listdir(os.path.join(features_dir, d)))]


def host_store_above(device_bytes, read_store=None) -> int:
    """The packed read-store size (bytes) above which the reads stay in pinned host memory (one hb_read_store for all devices)
    instead of a copy in every device's memory: half the memory of the smallest selected device, which leaves the other half to
    the model and the launches.  read_store "host" / "device" forces one of the two."""
    if read_store == "host":
        return 0
    if read_store == "device":
        return 2 ** 64 - 1
    if read_store is not None:
        raise ValueError(f"read_store must be None, 'host' or 'device', got {read_store!r}")
    return min(int(b) for b in device_bytes) // 2


def device_bytes(devices) -> list:
    """Total memory of each CUDA device in `devices`."""
    import torch
    return [torch.cuda.get_device_properties(int(d)).total_memory for d in devices]


def inference(reads_path: str, alns_dir: str, model: str, output: str, window: int = 4096, batch: int = 64, threads: int = 1,
              devices=(0,), core=None, neighbour=None, io_threads: int = 0, read_store=None, aln_buffer_bytes=None) -> dict:
    """The reference's `herro inference --read-alns` command, natively (hbh_inference) -> stage times and counts.  The read store
    is chosen by host_store_above; read_store ("host" / "device") overrides it.  The alignment files are decoded while earlier ones
    are corrected, holding at most aln_buffer_bytes of them (None: 1/8 of physical memory; UNLIMITED: no limit) unless one file is
    larger on its own.  An alignment file that cannot be read or parsed raises HerroError naming it, after the records of the
    targets submitted before it have been written."""
    H = _lib()
    dev = np.asarray(list(devices), dtype=np.int32)
    ca, nc, k1 = _strs(core)
    na, nn, k2 = _strs(neighbour)
    above = host_store_above(None if read_store else device_bytes(dev), read_store)
    t9, c6 = np.zeros(9), np.zeros(6, np.uint64)
    rc = H.hbh_inference(reads_path.encode(), alns_dir.encode(), model.encode(), output.encode(), window, batch, threads,
                         dev.ctypes.data, len(dev), ca, nc, na, nn, io_threads or min(os.cpu_count() or 1, 32), above,
                         _budget(aln_buffer_bytes), t9.ctypes.data, c6.ctypes.data)
    if rc != 0:
        raise api.HerroError(rc, H.hbh_last_error().decode())
    return dict(fastq_load_s=t9[0], pack_s=t9[1], alignment_ingest_s=t9[2], read_store_upload_s=t9[3], correction_s=t9[4],
                fasta_close_s=t9[5], total_s=t9[6], corrected_bases=int(t9[7]), first_submit_s=t9[8], reads=int(c6[0]),
                targets=int(c6[1]), records=int(c6[2]), failed_targets=int(c6[3]), alignment_peak_bytes=int(c6[4]),
                alignment_budget_bytes=int(c6[5]))


class PafReader:
    """An overlap-only PAF (plain or gzip) in chunks of admitted lines (hbh_paf_*): unknown read names and self overlaps are skipped,
    a cg:Z: field is ignored, repeated pairs are kept."""

    def __init__(self, path: str, reads: Reads):
        H = _lib()
        self._H, self._h, self.reads = H, C.c_void_p(), reads
        rc = H.hbh_paf_open(path.encode(), reads._h, C.byref(self._h))
        if rc != 0:
            raise api.HerroError(rc, H.hbh_last_error().decode())

    def next(self, max_lines: int = 200_000):
        """-> the next chunk's overlaps (OVERLAP_DTYPE, no CIGARs), or None at the end of the file.  The chunk stays current for
        BatchWriter.write until the next call."""
        n = C.c_uint32()
        rc = self._H.hbh_paf_next(self._h, max_lines, C.byref(n))
        if rc != 0:
            raise api.HerroError(rc, self._H.hbh_last_error().decode())
        if not n.value:
            return None
        buf = (C.c_char * (n.value * api.OVERLAP_DTYPE.itemsize)).from_address(self._H.hbh_paf_overlaps(self._h))
        return np.frombuffer(buf, dtype=api.OVERLAP_DTYPE, count=n.value).copy()

    def stats(self) -> dict:
        c = np.zeros(3, np.uint64)
        self._H.hbh_paf_stats(self._h, c.ctypes.data)
        return dict(lines=int(c[0]), skipped=int(c[1]), bytes=int(c[2]))

    def close(self):
        if self._h:
            self._H.hbh_paf_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchWriter:
    """`--read-alns` batches as the reference's write mode makes them (hbh_batches_*): <k>.oec.zst holds the k-th run of batch_size
    reads in FASTQ order, a header (the count, then the ids) and the aligned lines of its targets in input order."""

    def __init__(self, out_dir: str, reads: Reads, batch_size: int = 50_000):
        H = _lib()
        self._H, self._h, self.n_batches = H, C.c_void_p(), (reads.n + batch_size - 1) // batch_size
        rc = H.hbh_batches_open(out_dir.encode(), reads._h, batch_size, C.byref(self._h))
        if rc != 0:
            raise api.HerroError(rc, H.hbh_last_error().decode())

    def write(self, paf: PafReader, aligned: np.ndarray, status: np.ndarray, matches: np.ndarray):
        """The current chunk of `paf` with the coordinates and CIGARs of `aligned` (Context.align's overlaps); lines whose status is
        negative are not written."""
        status = np.ascontiguousarray(status, np.int32)
        matches = np.ascontiguousarray(matches, np.uint32)
        aligned = np.ascontiguousarray(aligned)
        rc = self._H.hbh_batches_write(self._h, paf._h, aligned.ctypes.data, status.ctypes.data, matches.ctypes.data, len(aligned))
        if rc != 0:
            raise api.HerroError(rc, self._H.hbh_last_error().decode())

    def close(self) -> list:
        """Finishes the files -> lines written per batch."""
        lines = np.zeros(max(self.n_batches, 1), np.uint64)
        h, self._h = self._h, C.c_void_p()
        rc = self._H.hbh_batches_close(h, lines.ctypes.data)
        if rc != 0:
            raise api.HerroError(rc, self._H.hbh_last_error().decode())
        return [int(x) for x in lines[:self.n_batches]]


def align(reads_path: str, paf_path: str, out_dir: str, device: int = 0, min_len: int = 4096, band_w: int = 0, batch_size: int = 50_000,
          chunk_lines: int = 200_000, io_threads: int = 0) -> dict:
    """`herro align`, natively (hbh_align): an overlap-only PAF aligned on the device and written as `--read-alns` batches -> the
    wall time of each phase and the counts."""
    H = _lib()
    t6, c7 = np.zeros(6), np.zeros(7, np.uint64)
    rc = H.hbh_align(reads_path.encode(), paf_path.encode(), out_dir.encode(), device, min_len, band_w, batch_size, chunk_lines,
                     io_threads or min(os.cpu_count() or 1, 32), t6.ctypes.data, c7.ctypes.data)
    if rc != 0:
        raise api.HerroError(rc, H.hbh_last_error().decode())
    return dict(fastq_load_s=t6[0], upload_s=t6[1], paf_read_s=t6[2], align_s=t6[3], write_s=t6[4], total_s=t6[5], lines=int(c7[0]),
                skipped=int(c7[1]), aligned=int(c7[2]), band_edge=int(c7[3]), failed=int(c7[4]), cells=int(c7[5]),
                device_ms=int(c7[6]))


def paf_lines(R: "Reads", got: dict) -> list:
    """`qname qlen qstart qend +/- tname tlen tstart tend covered max(tspan, qspan) 255 s1:i:<score> cm:i:<n_anchors>` per record
    of Context.find_overlaps, as bytes lines; hbh_paf_* (`herro align`) reads them."""
    o, ids = got["overlaps"], R.ids
    rows = zip(o["qid"].tolist(), o["qlen"].tolist(), o["qstart"].tolist(), o["qend"].tolist(), o["strand"].tolist(),
               o["tid"].tolist(), o["tlen"].tolist(), o["tstart"].tolist(), o["tend"].tolist(), got["covered"].tolist(),
               got["score"].tolist(), got["n_anchors"].tolist())
    return [b"%s\t%d\t%d\t%d\t%c\t%s\t%d\t%d\t%d\t%d\t%d\t255\ts1:i:%d\tcm:i:%d\n" % (
        ids[q], ql, qs, qe, 45 if st else 43, ids[t], tl, ts, te, cov, max(te - ts, qe - qs), sc, na)
        for q, ql, qs, qe, st, t, tl, ts, te, cov, sc, na in rows]


def overlap(reads_path: str, out_path: str, device: int = 0, min_len: int = 4096, targets_per_call: int = 50_000, **params) -> dict:
    """`herro overlap`: the reads' all-vs-all overlaps found on the device (hb_find_overlaps), written as overlap-only PAF (gzip when
    out_path ends in .gz).  Each call takes the next `targets_per_call` loaded reads in FASTQ order as its targets and every loaded
    read as a query.  -> the wall time of each phase and the counts."""
    import gzip
    import time
    t0 = time.perf_counter()
    R = Reads(reads_path, min_len=min_len)
    t1 = time.perf_counter()
    ctx = api.Context(None, device)
    store = R.load_into(ctx, device_bytes([device]))
    t2 = time.perf_counter()
    find_s = write_s = device_ms = 0.0
    n_ovl = calls = 0
    step = max(1, targets_per_call)
    with (gzip.open(out_path, "wb", compresslevel=1) if out_path.endswith(".gz") else open(out_path, "wb")) as f:
        for a in range(0, R.n, step):
            ta = time.perf_counter()
            got = ctx.find_overlaps(np.arange(a, min(a + step, R.n), dtype=np.uint32), **params)
            tb = time.perf_counter()
            f.writelines(paf_lines(R, got))
            write_s += time.perf_counter() - tb
            find_s += tb - ta
            device_ms += got["shape"]["ms_device"]
            n_ovl += len(got["overlaps"])
            calls += 1
    ctx.close()
    del store
    R.close()
    return dict(reads=R.n, calls=calls, overlaps=n_ovl, device_ms=device_ms, fastq_load_s=t1 - t0, upload_s=t2 - t1, find_s=find_s,
                write_s=write_s, total_s=time.perf_counter() - t0)
