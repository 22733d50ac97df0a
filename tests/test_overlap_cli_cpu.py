"""The host side of `herro overlap` without a device: the PAF lines it writes, `herro align`'s PAF reader admitting them, and the
argument rules of `inference` / `features` (--read-alns and --write-alns exclude each other)."""
import gzip
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from herro_b200 import api, cli, hostio  # noqa: E402
from tools import synth  # noqa: E402


@pytest.fixture()
def reads(tmp_path):
    rs = synth.generate(6, 5000, profile="r10", seed=3, coverage=4.0, min_len=4500, max_len=6000)
    fq = str(tmp_path / "reads.fastq")
    synth.write_fastq(rs, fq)
    R = hostio.Reads(fq, min_len=0)
    yield R
    R.close()


def found(rows):
    o = np.zeros(len(rows), api.OVERLAP_DTYPE)
    for k, f in enumerate(("qid", "qlen", "qstart", "qend", "strand", "tid", "tlen", "tstart", "tend")):
        o[f] = [r[k] for r in rows]
    n = len(rows)
    return dict(overlaps=o, score=np.arange(n, dtype=np.uint32) + 2500, n_anchors=np.arange(n, dtype=np.uint32) + 3,
                covered=np.arange(n, dtype=np.uint32) + 100)


def test_paf_lines(reads):
    L = [int(x) for x in reads.lens]
    got = found([(1, L[1], 10, 4000, 0, 0, L[0], 20, 4100, 0), (0, L[0], 0, 3000, 1, 2, L[2], 500, 3400, 0)])
    lines = hostio.paf_lines(reads, got)
    assert lines[0] == (f"read_000001\t{L[1]}\t10\t4000\t+\tread_000000\t{L[0]}\t20\t4100\t100\t4080\t255\ts1:i:2500\tcm:i:3\n").encode()
    assert lines[1] == (f"read_000000\t{L[0]}\t0\t3000\t-\tread_000002\t{L[2]}\t500\t3400\t101\t3000\t255\ts1:i:2501\tcm:i:4\n").encode()


@pytest.mark.parametrize("gz", [False, True])
def test_align_reads_the_written_paf(reads, tmp_path, gz):
    L = [int(x) for x in reads.lens]
    rows = [(1, L[1], 10, 4000, 0, 0, L[0], 20, 4100, 0), (0, L[0], 0, 3000, 1, 2, L[2], 500, 3400, 0),
            (3, L[3], 5, 2000, 1, 4, L[4], 7, 1900, 0)]
    path = str(tmp_path / ("o.paf.gz" if gz else "o.paf"))
    with (gzip.open(path, "wb") if gz else open(path, "wb")) as f:
        f.writelines(hostio.paf_lines(reads, found(rows)))
    P = hostio.PafReader(path, reads)
    o = P.next()
    assert P.next() is None
    assert P.stats()["lines"] == 3 and P.stats()["skipped"] == 0
    P.close()
    for k, f in enumerate(("qid", "qlen", "qstart", "qend", "strand", "tid", "tlen", "tstart", "tend")):
        assert o[f].tolist() == [r[k] for r in rows], f


@pytest.mark.parametrize("cmd", [["inference", "-m", "m", "-b", "8"], ["features"]])
def test_read_alns_and_write_alns_exclude_each_other(cmd, capsys):
    with pytest.raises(SystemExit):
        cli.main(cmd + ["--read-alns", "a", "--write-alns", "b", "reads.fastq", "out"])
    assert "not allowed with argument" in capsys.readouterr().err
