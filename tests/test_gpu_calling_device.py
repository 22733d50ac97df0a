"""Every call on a context returns with the calling thread's current CUDA device as it found it: a host thread that drives a context on
another GPU, or a torch program whose current device is not the context's, stays on its own device.  The context lives on the last
visible device and the thread's current device is 0."""
import ctypes

import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api
from test_gpu_features_batch import overlaps
from test_gpu_forward_batch import targets_of

pytestmark = pytest.mark.gpu


def test_every_call_returns_on_the_callers_device(tmp_path):
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs two visible GPUs")
    dev = n_dev - 1
    cudart = ctypes.CDLL("libcudart.so.12")  # the runtime torch loaded: cudaGetDevice reads the thread's current context

    def current():
        d = ctypes.c_int(-1)
        assert cudart.cudaGetDevice(ctypes.byref(d)) == 0
        return d.value

    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda:0")  # device 0's primary context exists and is current
    assert current() == 0
    moved = []

    def check(name):
        if current() != 0:
            moved.append(name)
            assert cudart.cudaSetDevice(0) == 0

    rs = helpers.small_readset(n_reads=24, mean_len=9000, seed=5)
    targets = targets_of(rs, 12)
    tg = [(t, overlaps(rs, t)) for t in targets]
    model = helpers.model_path(seed=3)

    with pytest.raises(api.HerroError):
        api.Context(str(tmp_path / "missing.bin"), dev)  # fails after the device was made current
    check("Context (failing)")
    ctx = api.Context(model, dev, 4096, 64, launch_targets=1 << 20, keep_debug=True)
    check("Context")
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    check("upload_reads")
    for t, o in tg:  # the first target grows the thread's pinned staging batch
        ctx.submit_alignments(t, o)
        check(f"submit_alignments({t})")
    ctx.flush()
    check("flush")
    assert len(ctx.drain()) == len(targets)
    check("drain")
    ctx.debug_window(targets[0], 0)
    check("debug_window")
    ctx.dump_features(targets[0], str(tmp_path), rs.ids)
    check("dump_features")
    ctx.replay_last_launch(1)
    check("replay_last_launch")
    F = ctx.features_batch(tg, batches=True)
    check("features_batch")
    batches = list(F.batches())
    assert batches
    logits = []
    for _, bases, quals, lens, idx in batches:
        logits.append(ctx.forward_batch(bases, quals, lens, idx)[1])
        check("forward_batch")
    ctx.consensus_batch(*F.consensus_args(logits))
    check("consensus_batch")
    ovl = rs.ovl9[:120]
    ctx.align(api.Context.make_overlaps(ovl, np.zeros(1, np.uint8), np.zeros(len(ovl) + 1, np.uint64)))
    check("align")
    ctx.find_overlaps(targets)
    check("find_overlaps")
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctx.attach_read_store(store)
    check("attach_read_store")
    ctx.close()
    check("close")
    store.close()
    api.selftest_gemm(128, 128, 64, device=dev)
    check("selftest_gemm")
    api.selftest_pos_attention([8], 4, 32, np.zeros((8, 3 * 128), np.float32), device=dev)
    check("selftest_pos_attention")
    assert moved == [], f"calls that left the thread on device {dev}: {moved}"
