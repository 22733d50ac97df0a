"""hb_align_overlaps and hb_find_overlaps on either read store, and the host store on a device other than 0: what each call adds to
hb_stats (exactly its own counters, the same amount on every identical call), exactly the call's distinct reads crossing PCIe with
a host store, and a launch, features_batch, align and find_overlaps on the last visible device equal to the same calls on
device 0."""
import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api
from test_gpu_host_read_store import CONFIGS, READ_COPY_BYTES, make_ctx, overlaps, padded_bytes, run, targets_of
from test_gpu_stage_counters import expect, flat

pytestmark = pytest.mark.gpu

OVERLAPS = expect({"kernel_launches", "h2d_bytes", "d2h_bytes"}, ())  # align and find_overlaps time no kernel class


def overlap_only(ovl9):
    """hb_overlap[] of (qid, qlen, qstart, qend, strand, tid, tlen, tstart, tend) rows, without CIGARs."""
    return api.Context.make_overlaps(ovl9, np.zeros(1, np.uint8), np.zeros(len(ovl9) + 1, np.uint64))


@pytest.fixture(scope="module")
def no_model():
    """Contexts without weights: one with the reads uploaded, one on a host read store."""
    rs = helpers.small_readset(n_reads=24, mean_len=9000, seed=5)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctxs = {}
    for kind in ("uploaded", "host-store"):
        c = api.Context(None)
        if kind == "uploaded":
            c.upload_reads(rs.seqs, rs.quals, rs.off)
        else:
            c.attach_read_store(store)
        c.set_kernel_timing(True)
        ctxs[kind] = c
    return dict(ctxs=ctxs, ovl=overlap_only(rs.ovl9[:120]), reads=list(range(rs.n)))


CALLS = {
    "align": lambda ctx, d: ctx.align(d["ovl"]),
    "find": lambda ctx, d: ctx.find_overlaps(d["reads"]),
}


@pytest.mark.parametrize("store", ["uploaded", "host-store"])
@pytest.mark.parametrize("stage", list(CALLS))
def test_each_call_adds_its_own_counters(no_model, stage, store):
    ctx = no_model["ctxs"][store]
    call = CALLS[stage]
    call(ctx, no_model)  # warm-up: the lane's regions reach this shape
    ctx.reset_stats()
    call(ctx, no_model)
    one = flat(ctx.stats())
    got = {k for k, v in one.items() if v != 0}
    assert got == OVERLAPS, f"non-zero but not expected: {sorted(got - OVERLAPS)}; expected but 0: {sorted(OVERLAPS - got)}"
    call(ctx, no_model)
    two = flat(ctx.stats())
    ints = [k for k, v in one.items() if isinstance(v, int)]
    assert ints and {k: two[k] for k in ints} == {k: 2 * one[k] for k in ints}


def test_align_and_find_gather_only_their_reads():
    """On a host store, align and find_overlaps move exactly their distinct reads (padded) and read-list entries more than on an
    uploaded store: for align the reads of the admitted overlaps, for find_overlaps in one chunk the targets and then every read."""
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=5)
    lens = np.diff(rs.off).astype(np.int64)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    up, host = api.Context(None), api.Context(None)
    up.upload_reads(rs.seqs, rs.quals, rs.off)
    host.attach_read_store(store)

    def h2d(call):
        out = []
        for ctx in (up, host):
            s0 = ctx.stats()["h2d_bytes"]
            out.append((call(ctx), ctx.stats()["h2d_bytes"] - s0))
        return out[0][0], out[1][0], out[1][1] - out[0][1]

    def gathered(reads):
        return sum(padded_bytes(int(lens[r])) + READ_COPY_BYTES for r in set(reads))

    ovl = overlap_only(rs.ovl9[:120])
    a, b, extra = h2d(lambda c: c.align(ovl))
    assert a["cigars"] == b["cigars"] and np.array_equal(a["status"], b["status"])
    ok = ovl[b["status"] >= 0]
    assert len(ok) > 100
    assert extra == gathered([int(r) for r in ok["tid"]] + [int(r) for r in ok["qid"]])
    targets = list(range(0, rs.n, 3))
    a, b, extra = h2d(lambda c: c.find_overlaps(targets))
    assert np.array_equal(a["overlaps"], b["overlaps"]) and len(a["overlaps"]) > 0
    assert extra == gathered(targets) + gathered(range(rs.n))
    host.close()
    up.close()
    store.close()


def test_host_store_on_the_last_device_matches_device_0():
    """A host-store context on the last visible device gives what the same calls give on device 0: every gather's read list is
    pinned for its own context's device."""
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs two visible GPUs")
    make, W, b = CONFIGS["r10-W4096-b64"]
    rs = make()
    targets = targets_of(rs)
    tl = [(t, overlaps(rs, t)) for t in targets]
    ovl = overlap_only(rs.ovl9[:120])
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    outs = []
    for device in (0, n_dev - 1):
        ctx = make_ctx(rs, W, b, store, device=device)
        segs = run(ctx, rs, targets, W, windows=False)[0]
        F = ctx.features_batch(tl, batches=True)
        feats = [getattr(F, k) for k in api.FEATURES_OUT_FIELDS]
        outs.append((segs, feats, ctx.align(ovl), ctx.find_overlaps(targets)))
        ctx.close()
    (s0, f0, a0, o0), (s1, f1, a1, o1) = outs
    assert s0 == s1 and any(s0.values())
    assert all(np.array_equal(x, y) for x, y in zip(f0, f1))
    assert a0["cigars"] == a1["cigars"] and np.array_equal(a0["status"], a1["status"]) and np.array_equal(a0["matches"], a1["matches"])
    for f in ("qstart", "qend", "tstart", "tend"):
        assert np.array_equal(a0["overlaps"][f], a1["overlaps"][f]), f
    for k in ("overlaps", "score", "n_anchors", "covered"):
        assert np.array_equal(o0[k], o1[k]), k
    store.close()
