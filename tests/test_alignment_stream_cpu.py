"""The streaming alignment reader (hbh_alns_stream_*, hostio.Alignments.stream) on CPU: its files, concatenated in order, are the
whole-directory load; the budget bounds the bytes in flight; an unreadable file ends the stream with an error naming it after
the files before it."""
import os
import time

import numpy as np
import pytest

import helpers
from herro_b200 import api, hostio
from tools import synth

FIELDS = ("qid", "qlen", "qstart", "qend", "strand", "tid", "tlen", "tstart", "tend", "cigar_len")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """Reads and 6 batch files of 7 targets each, plus a seventh file (sorted last) naming again the targets of the first file, so
    those targets appear in two files."""
    rs = helpers.small_readset(n_reads=40, mean_len=3000, seed=91, coverage=12.0, min_ovl=500, sd_frac=0.4, min_len=300)
    d = tmp_path_factory.mktemp("stream")
    fq = str(d / "reads.fastq")
    synth.write_fastq(rs, fq)
    alns = str(d / "alns")
    synth.write_oec_batches(rs, alns, batch_size=7)
    import pyarrow as pa
    again = [t for t in range(7) if rs.aln_off[t + 1] > rs.aln_off[t]]
    body = f"{len(again)}\n".encode() + b"".join((rs.ids[t] + "\n").encode() for t in again) + b"".join(synth.paf_lines(rs, again))
    with open(os.path.join(alns, "x_again.oec.zst"), "wb") as f:
        f.write(pa.Codec("zstd").compress(body, asbytes=True))
    R = hostio.Reads(fq, min_len=1500)
    return rs, R, alns


def files_of(alns):
    return sorted(os.path.join(alns, f) for f in os.listdir(alns) if f.endswith(".oec.zst"))


def file_bytes(a):
    return a.stats()["text_bytes"] + a.stats()["kept"] * api.OVERLAP_DTYPE.itemsize


@pytest.mark.parametrize("core", [False, True])
def test_stream_concatenated_equals_the_whole_load(inputs, core):
    rs, R, alns = inputs
    core_ids = [rs.ids[t] for t in range(0, rs.n, 3)] if core else None
    whole = hostio.Alignments(alns, R, core=core_ids, threads=3)
    rids, offs, ovl, cig, sources = [], [0], [], [], []
    with hostio.Alignments.stream(alns, R, core=core_ids, threads=3, budget=hostio.UNLIMITED) as S:
        for a in S:
            base = offs[-1]
            rids += [int(x) for x in a.target_rids]
            offs += [base + int(x) for x in a.offsets[1:]]
            ovl.append(a.overlaps.copy())
            cig += [a.cigar(i) for i in range(len(a.overlaps))]
            assert a.budget_bytes == file_bytes(a)
            sources.append(a.source)
            a.close()
    assert sources == files_of(alns) and len(sources) == 7
    assert whole.n_targets > 0 and rids == [int(x) for x in whole.target_rids]
    assert offs == [int(x) for x in whole.offsets]
    ovl = np.concatenate(ovl)
    for f in FIELDS:
        assert np.array_equal(ovl[f], whole.overlaps[f]), f
    assert cig == [whole.cigar(i) for i in range(len(whole.overlaps))]
    assert len(rids) > len(set(rids))            # the first file's targets are sent again by the last one
    if core:
        assert {R.ids[r].decode() for r in rids} <= set(core_ids)


@pytest.mark.parametrize("threads", [1, 4])
def test_budget_of_one_byte_holds_one_file(inputs, threads):
    """Starting a file reserves the size its zstd frame records, so several workers do not start files side by side either."""
    rs, R, alns = inputs
    sizes = []
    with hostio.Alignments.stream(alns, R, threads=threads, budget=1) as S:
        for a in S:
            sizes.append(file_bytes(a))
            a.close()
        st = S.stats()
    assert len(sizes) == 7 and st["budget_bytes"] == 1 and st["files_parsed"] == 7
    assert st["peak_files"] == 1 and 0 < st["peak_bytes"] <= max(sizes)
    assert st["in_flight_bytes"] == 0                # every file freed gave its bytes back


def test_unlimited_budget_holds_every_file(inputs):
    """With no limit the workers decode every file before the first is taken."""
    rs, R, alns = inputs
    with hostio.Alignments.stream(alns, R, threads=4, budget=hostio.UNLIMITED) as S:
        deadline = time.time() + 60
        while S.stats()["files_parsed"] < 7 and time.time() < deadline:
            time.sleep(0.01)
        st = S.stats()
        files = list(S)
        assert st["files_parsed"] == 7 and st["peak_files"] == 7
        assert st["peak_bytes"] == st["in_flight_bytes"] == sum(file_bytes(a) for a in files)
        for a in files:
            a.close()
        assert S.stats()["in_flight_bytes"] == 0


def test_files_outlive_their_stream(inputs):
    rs, R, alns = inputs
    S = hostio.Alignments.stream(alns, R, threads=2, budget=hostio.UNLIMITED)
    a = next(S)
    S.close()
    whole = hostio.Alignments(alns, R)
    assert a.n_targets > 0 and a.cigar(0) == whole.cigar(0)
    a.close()


def test_default_budget_is_an_eighth_of_memory(inputs):
    rs, R, alns = inputs
    with hostio.Alignments.stream(alns, R) as S:
        assert S.stats()["budget_bytes"] == os.sysconf("SC_PHYS_PAGES") * os.sysconf("SC_PAGE_SIZE") // 8
    with pytest.raises(ValueError):
        hostio.Alignments.stream(alns, R, budget=0)


def broken_copy(rs, alns, tmp_path, how):
    """The first three batch files of `alns` in a new directory, the third one broken."""
    import pyarrow as pa
    d = tmp_path / f"broken_{how}"
    d.mkdir()
    names = [os.path.basename(f) for f in files_of(alns)][:3]
    for n in names[:2]:
        (d / n).write_bytes(open(os.path.join(alns, n), "rb").read())
    tg = range(14, 21)                           # the targets of the third file (write_oec_batches, batch_size=7)
    body = f"{len(tg)}\n".encode() + b"".join((rs.ids[t] + "\n").encode() for t in tg) + b"".join(synth.paf_lines(rs, tg))
    if how == "line":
        body += b"read_000001\t100\t0\t100\t+\n"
    elif how == "header":
        body = b"x" + body
    if how == "zstd":
        (d / names[2]).write_bytes(b"\x28\xb5\x2f\xfd" + b"\x00" * 40)
    else:
        (d / names[2]).write_bytes(pa.Codec("zstd").compress(body, asbytes=True))
    return str(d), names


@pytest.mark.parametrize("how", ["line", "header", "zstd"])
@pytest.mark.parametrize("budget", [1, None])
def test_broken_third_file_ends_the_stream(inputs, tmp_path, how, budget):
    rs, R, alns = inputs
    d, names = broken_copy(rs, alns, tmp_path, how)
    got = []
    with hostio.Alignments.stream(d, R, threads=3, budget=budget) as S:
        with pytest.raises(api.HerroError) as ei:
            for a in S:
                got.append(os.path.basename(a.source))
                a.close()
        assert ei.value.code == -4 and names[2] in str(ei.value)
        with pytest.raises(api.HerroError):      # and on every later call
            next(S)
    assert got == names[:2]
    with pytest.raises(api.HerroError) as ei:    # the whole load reports the same file
        hostio.Alignments(d, R)
    assert names[2] in str(ei.value)


def test_empty_directory_yields_nothing(inputs, tmp_path):
    rs, R, alns = inputs
    with hostio.Alignments.stream(str(tmp_path), R) as S:
        assert list(S) == []
    assert hostio.Alignments(str(tmp_path), R).n_targets == 0
    with pytest.raises(api.HerroError):
        hostio.Alignments.stream(str(tmp_path / "missing"), R)


def test_inference_declaration():
    """hbh_inference takes the alignment budget and fills nine times and six counts."""
    H = hostio._lib()
    assert len(H.hbh_inference.argtypes) == 18
    import inspect
    assert "aln_buffer_bytes" in inspect.signature(hostio.inference).parameters
