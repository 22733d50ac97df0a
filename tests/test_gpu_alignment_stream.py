"""Correction on the alignment stream: `inference` at the extremes of the budget and of the feature threads, with either read store,
writes the records of per-target hb_submit_alignments; `features` and `inference --torch` loop over the streamed files with the same
outputs; an alignment file that breaks after correction started ends the run with an error naming it, after the earlier records."""
import os
import shutil

import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api, cli, hostio
from tools import synth

pytestmark = pytest.mark.gpu
HB_ERR_INPUT = -4
W, B = 4096, 64


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """40 reads, their alignments in 7 batch files of 6 targets each."""
    rs = helpers.small_readset(n_reads=40, mean_len=7000, seed=14, min_len=4200)
    d = tmp_path_factory.mktemp("stream_gpu")
    fq, alns = str(d / "reads.fastq"), str(d / "alns")
    synth.write_fastq(rs, fq, [None if i % 3 else f"ch={i}" for i in range(rs.n)])
    synth.write_oec_batches(rs, alns, batch_size=6)
    assert len([f for f in os.listdir(alns) if f.endswith(".oec.zst")]) >= 6
    return rs, fq, alns


def records(path):
    return sorted(open(path, "rb").read().split(b">")[1:])


def submitted_records(fq, alns):
    """The FASTA records of every target of the whole load, each submitted alone through hb_submit_alignments on one context."""
    R = hostio.Reads(fq, min_len=W)
    A = hostio.Alignments(alns, R)
    ctx = api.Context(helpers.model_path(seed=3), 0, W, B)
    R.upload(ctx)
    for k in range(A.n_targets):
        ctx.submit_alignments(*A.target(k))
    ctx.flush()
    out = []
    for r in ctx.drain(skip_failed=True):
        if r.segments:
            out += api.fasta_records(R.ids[r.rid], R.descriptions[r.rid], r.segments).split(b">")[1:]
    assert not ctx.failed
    ctx.close()
    return sorted(out), A.n_targets


def file_sizes(fq, alns):
    R = hostio.Reads(fq, min_len=W)
    out = []
    with hostio.Alignments.stream(alns, R, budget=hostio.UNLIMITED) as S:
        for a in S:
            out.append(a.budget_bytes)
            a.close()
    return out


@pytest.fixture(scope="module")
def want(inputs):
    rs, fq, alns = inputs
    return submitted_records(fq, alns)


@pytest.mark.parametrize("budget,threads,store", [(1, 1, None), (1, 4, None), (hostio.UNLIMITED, 1, None), (hostio.UNLIMITED, 4, None),
                                                  (1, 4, "host"), (hostio.UNLIMITED, 1, "host")])
def test_inference_on_the_stream(inputs, want, tmp_path, budget, threads, store):
    rs, fq, alns = inputs
    out = str(tmp_path / "out.fasta")
    # one decoding worker at the one-byte budget, so that exactly one file is ever in flight
    r = hostio.inference(fq, alns, helpers.model_path(seed=3), out, W, B, threads=threads, read_store=store or "device",
                         io_threads=1 if budget == 1 else 0, aln_buffer_bytes=budget)
    assert records(out) == want[0] and len(want[0]) > 0
    assert r["targets"] == want[1] and r["failed_targets"] == 0 and r["records"] == len(want[0])
    sizes = file_sizes(fq, alns)
    assert r["alignment_budget_bytes"] == budget
    if budget == 1:
        assert 0 < r["alignment_peak_bytes"] <= max(sizes)
    else:
        assert max(sizes) <= r["alignment_peak_bytes"] <= sum(sizes)
    assert 0 < r["first_submit_s"] < r["total_s"] and r["alignment_ingest_s"] > 0
    for k in ("fastq_load_s", "pack_s", "read_store_upload_s", "correction_s", "fasta_close_s", "corrected_bases", "reads"):
        assert k in r


def force_budget(monkeypatch, budget):
    """The CLI commands with the stream's budget set to `budget` (they take the default)."""
    stream = hostio.Alignments.stream.__func__
    monkeypatch.setattr(hostio.Alignments, "stream",
                        classmethod(lambda cls, alns_dir, reads, core=None, threads=0, budget_=None:
                                    stream(cls, alns_dir, reads, core, threads, budget)))


@pytest.mark.parametrize("budget", [1, None])
def test_cli_features_on_the_stream_reproduces_the_golden_dump(tmp_path, monkeypatch, budget):
    import glob
    if budget is not None:
        force_budget(monkeypatch, budget)
    golden = os.path.join(helpers.ROOT, "tests", "golden", "features_dump")
    out = str(tmp_path / "feats")
    cli.main(["features", "--read-alns", os.path.join(golden, "alns"), "-w", "256", os.path.join(golden, "reads.fastq"), out])
    n = 0
    for d in sorted(glob.glob(os.path.join(golden, "read_*"))):
        for a in sorted(glob.glob(os.path.join(d, "*"))):
            b = os.path.join(out, os.path.basename(d), os.path.basename(a))
            assert open(a, "rb").read() == open(b, "rb").read(), b
            n += 1
    assert n >= 30


def test_cli_features_over_several_files_equals_one_file(inputs, tmp_path, monkeypatch):
    """The same alignments as one batch file or as seven, streamed at a one-byte budget: the same feature files."""
    import pyarrow as pa
    rs, fq, alns = inputs
    one = tmp_path / "one"
    one.mkdir()
    body = f"{rs.n}\n".encode() + b"".join((i + "\n").encode() for i in rs.ids) + b"".join(synth.paf_lines(rs))
    (one / "0.oec.zst").write_bytes(pa.Codec("zstd").compress(body, asbytes=True))
    cli.main(["features", "--read-alns", str(one), "--targets-per-launch", "4", fq, str(tmp_path / "a")])
    force_budget(monkeypatch, 1)
    cli.main(["features", "--read-alns", alns, "--targets-per-launch", "4", fq, str(tmp_path / "b")])
    fa = sorted(os.path.relpath(os.path.join(p, f), tmp_path / "a") for p, _, fs in os.walk(tmp_path / "a") for f in fs)
    fb = sorted(os.path.relpath(os.path.join(p, f), tmp_path / "b") for p, _, fs in os.walk(tmp_path / "b") for f in fs)
    assert fa == fb and len(fa) > 100
    for f in fa:
        assert open(tmp_path / "a" / f, "rb").read() == open(tmp_path / "b" / f, "rb").read(), f


def test_cli_inference_torch_same_fasta_at_any_budget(inputs, tmp_path, monkeypatch):
    from herro_b200 import weights as hbw
    from oracle import forward_ref
    rs, fq, alns = inputs
    cfg, T = hbw.load_blob(helpers.model_path(seed=3))
    pt = str(tmp_path / "model.pt")
    torch.jit.script(forward_ref.from_weights(cfg, T)).save(pt)
    outs = []
    for budget in (hostio.UNLIMITED, 1):
        force_budget(monkeypatch, budget)
        out = str(tmp_path / f"torch_{budget}.fasta")
        r = cli.main(["inference", "--torch", "--read-alns", alns, "-m", pt, "-b", "8", "--targets-per-launch", "5", fq, out])
        assert r["failed_targets"] == 0 and r["records"] > 0
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1]


def test_late_ingest_error_after_earlier_records(inputs, tmp_path):
    """A malformed last file: HB_ERR_INPUT naming it, and the records of every target of the files before it are written."""
    import pyarrow as pa
    rs, fq, alns = inputs
    d = tmp_path / "alns"
    shutil.copytree(alns, d)
    body = b"1\n" + rs.ids[0].encode() + b"\n" + next(iter(synth.paf_lines(rs, [0]))) + b"read_000001\t7000\t0\n"
    (d / "zz_bad.oec.zst").write_bytes(pa.Codec("zstd").compress(body, asbytes=True))
    want = submitted_records(fq, alns)[0]
    for budget, threads in ((1, 1), (hostio.UNLIMITED, 4)):
        out = str(tmp_path / f"out_{threads}.fasta")
        with pytest.raises(api.HerroError) as ei:
            hostio.inference(fq, str(d), helpers.model_path(seed=3), out, W, B, threads=threads, read_store="device",
                             aln_buffer_bytes=budget)
        assert ei.value.code == HB_ERR_INPUT and "zz_bad.oec.zst" in str(ei.value), budget
        assert records(out) == want, budget
    with pytest.raises(api.HerroError) as ei:      # `cli inference` fails with it (a non-zero exit as a command)
        cli.main(["inference", "--read-alns", str(d), "-m", helpers.model_path(seed=3), "-b", "64", fq, str(tmp_path / "cli.fasta")])
    assert "zz_bad.oec.zst" in str(ei.value)
