"""What each single-stage call (forward_batch, consensus_batch, features_batch) adds to hb_stats: exactly the counters of its own
stage, the same amount on every identical call, and nothing of the launch worker's; a flush on the same context still records
the launch worker's counters."""
import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api
from test_gpu_features_batch import overlaps
from test_gpu_forward_batch import targets_of

pytestmark = pytest.mark.gpu


def expect(fields, kernels, flops=()):
    """The non-zero counters of one call: `fields`, and n_kernel / ms_kernel of `kernels`, class_flops of `flops`."""
    return set(fields) | {f"n_kernel.{k}" for k in kernels} | {f"ms_kernel.{k}" for k in kernels} | {f"class_flops.{k}" for k in flops}


FORWARD = expect({"ms_forward", "supported", "kernel_launches", "gemm_flops", "forward_flops"},
                 {"lists", "stem", "qkv_attn", "ffn", "gemm", "heads"}, {"stem", "qkv_attn", "ffn", "gemm", "heads"})
CONSENSUS = expect({"ms_consensus", "kernel_launches"}, {"consensus", "scan"})
FEATURES = expect({"ms_features", "kernel_launches", "h2d_bytes", "d2h_bytes"},
                  {"tokenize", "pass1", "scores", "pass2a", "scan", "pileup", "lists"})


def flat(s):
    """hb_stats as {name: value}, one entry per scalar: n_kernel.<class>, ms_worker_phase.<i>, ..."""
    out = {}
    for k, v in s.items():
        if isinstance(v, dict):
            out.update({f"{k}.{c}": x for c, x in v.items()})
        elif isinstance(v, list):
            out.update({f"{k}.{i}": x for i, x in enumerate(v)})
        else:
            out[k] = v
    return out


@pytest.fixture(scope="module")
def setup():
    rs = helpers.small_readset(n_reads=24, mean_len=9000, seed=5)
    targets = targets_of(rs, 12)
    ctx = api.Context(helpers.model_path(seed=3), 0, 4096, 64, launch_targets=1 << 20)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    ctx.set_kernel_timing(True)
    tg = [(t, overlaps(rs, t)) for t in targets]
    F = ctx.features_batch(tg, batches=True)
    batches = list(F.batches())
    assert batches
    logits = [ctx.forward_batch(bases, quals, lens, idx)[1] for _, bases, quals, lens, idx in batches]
    cons = F.consensus_args(logits)
    return dict(ctx=ctx, rs=rs, targets=targets, tg=tg, batch=batches[0][1:], cons=cons)


def cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


CASES = {
    "forward-host": lambda d: d["ctx"].forward_batch(*d["batch"]),
    "forward-cuda": lambda d: d["ctx"].forward_batch(cuda(d["batch"][0]), cuda(d["batch"][1]), *d["batch"][2:]),
    "consensus-host": lambda d: d["ctx"].consensus_batch(*d["cons"]),
    "consensus-cuda": lambda d: d["ctx"].consensus_batch(*d["cons"][:3], cuda(d["cons"][3]), d["cons"][4], cuda(d["cons"][5])),
    "features-host": lambda d: d["ctx"].features_batch(d["tg"]),
    "features-device-batches": lambda d: d["ctx"].features_batch(d["tg"], device=True, batches=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_each_call_adds_its_own_counters(setup, case):
    ctx, call = setup["ctx"], CASES[case]
    call(setup)  # warm-up: the lane's regions reach this shape
    ctx.reset_stats()
    call(setup)
    one = flat(ctx.stats())
    want = FORWARD if case.startswith("forward") else CONSENSUS if case.startswith("consensus") else FEATURES
    got = {k for k, v in one.items() if v != 0}
    assert got == want, f"non-zero but not expected: {sorted(got - want)}; expected but 0: {sorted(want - got)}"
    if case.startswith("forward"):
        assert one["supported"] == int(np.sum(setup["batch"][2]))
    call(setup)
    two = flat(ctx.stats())
    ints = [k for k, v in one.items() if isinstance(v, int)]
    assert ints and {k: two[k] for k in ints} == {k: 2 * one[k] for k in ints}


def test_a_flush_still_records_the_launch_worker(setup):
    ctx, rs, targets = setup["ctx"], setup["rs"], setup["targets"]
    ctx.reset_stats()
    for t, o in setup["tg"]:
        ctx.submit_alignments(t, o)
    ctx.flush()
    assert len(ctx.drain()) == len(targets)
    s = ctx.stats()
    assert s["last_launch_targets"] == len(targets) and s["last_launch_windows"] == s["windows"] > 0
    assert s["last_launch_bases"] == s["corrected_bases"] > 0
    assert s["ms_worker_busy"] > 0 and all(p > 0 for p in s["ms_worker_phase"][:7])
