"""`inference` and `features` from a FASTQ alone: overlaps found and aligned on the device (`overlap` -> `align`) give the same
outputs as the same steps run one by one and passed with --read-alns, and --write-alns keeps those batches."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import helpers  # noqa: E402
from herro_b200 import cli  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def prepared(tmp_path_factory):
    d = tmp_path_factory.mktemp("ovl_cli")
    rs = synth.generate(40, 9000, profile="r10", seed=12, coverage=12.0)
    fq = str(d / "reads.fastq")
    synth.write_fastq(rs, fq)
    paf = str(d / "ovl.paf.gz")
    r = cli.main(["overlap", "-d", "0", fq, paf])
    assert r["overlaps"] > 50
    alns = str(d / "alns")
    cli.main(["align", "-d", "0", fq, paf, alns])
    return d, fq, alns


def files(d):
    return sorted(os.listdir(d))


def test_inference_from_fastq_alone(prepared):
    d, fq, alns = prepared
    model = helpers.model_path(seed=3)
    ref, alone, kept = str(d / "ref.fasta"), str(d / "alone.fasta"), str(d / "kept.fasta")
    cli.main(["inference", "--read-alns", alns, "-m", model, "-b", "64", fq, ref])
    cli.main(["inference", "-m", model, "-b", "64", fq, alone])
    keep = str(d / "kept_alns")
    cli.main(["inference", "--write-alns", keep, "-m", model, "-b", "64", fq, kept])
    assert os.path.getsize(ref) > 0
    assert open(alone, "rb").read() == open(ref, "rb").read()
    assert open(kept, "rb").read() == open(ref, "rb").read()
    assert files(keep) == files(alns)
    for f in files(alns):
        assert open(os.path.join(keep, f), "rb").read() == open(os.path.join(alns, f), "rb").read()


def test_inference_torch_from_fastq_alone(prepared):
    import torch
    from herro_b200 import weights as hbw
    from oracle import forward_ref
    d, fq, alns = prepared
    cfg, T = hbw.load_blob(helpers.model_path(seed=3))
    pt = str(d / "model.pt")
    torch.jit.script(forward_ref.from_weights(cfg, T)).save(pt)
    ref, alone = str(d / "tref.fasta"), str(d / "talone.fasta")
    cli.main(["inference", "--torch", "--read-alns", alns, "-m", pt, "-b", "8", fq, ref])
    cli.main(["inference", "--torch", "-m", pt, "-b", "8", fq, alone])
    assert os.path.getsize(ref) > 0
    assert open(alone, "rb").read() == open(ref, "rb").read()


def test_features_from_fastq_alone(prepared):
    d, fq, alns = prepared
    ref, alone = str(d / "feat_ref"), str(d / "feat_alone")
    cli.main(["features", "--read-alns", alns, fq, ref])
    cli.main(["features", fq, alone])
    assert files(ref) and files(ref) == files(alone)
    for sub in files(ref):
        a, b = os.path.join(ref, sub), os.path.join(alone, sub)
        assert files(a) == files(b)
        for f in files(a):
            assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read()
