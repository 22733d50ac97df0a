"""The read store in pinned host memory (hb_read_store_create / hb_attach_read_store, api.ReadStore): every output bit for bit equal to
an uploaded store's, through hb_submit_alignments, hb_submit_target and hb_features_batch; reads at the edges of a launch's gathered
layout; many launches on all lanes; only each launch's reads crossing PCIe; contexts sharing one store from two threads; replay,
failures, call-sequence errors and round trips; and `inference` forced to each store."""
import threading

import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api, hostio

pytestmark = pytest.mark.gpu
HB_ERR_INPUT, HB_ERR_STATE = -4, -6
READ_COPY_BYTES = 40  # one read-list entry (ReadCopy)


def overlaps(rs, t):
    a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
    return api.Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1])


def targets_of(rs):
    return [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]]


def make_ctx(rs, W, b, store=None, launch_targets=1 << 20, device=0):
    """A context with the reads uploaded (store None) or attached from `store`."""
    ctx = api.Context(helpers.model_path(seed=3), device, W, b, launch_targets=launch_targets, keep_debug=True)
    if store is None:
        ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    else:
        ctx.attach_read_store(store)
    return ctx


def run(ctx, rs, targets, W, submit_target=False, windows=True):
    """Every target through hb_submit_alignments (or hb_submit_target with host windowing) -> (segments by rid, failures by rid,
    debug windows of the last launch)."""
    for t in targets:
        o = overlaps(rs, t)
        if submit_target:
            nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
            ctx.submit_target(t, nw, o, api.extract_windows(o, W, nw))
        else:
            ctx.submit_alignments(t, o)
    ctx.flush()
    segs = {r.rid: r.segments for r in ctx.drain(skip_failed=True)}
    failed = {rid: code for rid, code, _ in ctx.failed}
    wins = {}
    if windows:
        for t in targets:
            if t in failed:
                continue
            for w in range((int(rs.off[t + 1] - rs.off[t]) + W - 1) // W):
                wins[(t, w)] = ctx.debug_window(t, w)
    return segs, failed, wins


def same_windows(a, b):
    assert a.keys() == b.keys() and len(a) > 0
    for k in a:
        for f in ("L", "n_alns"):
            assert a[k][f] == b[k][f], (k, f)
        for f in ("bases", "quals", "supported", "sup_rows", "info_logits", "bases_logits"):
            assert np.array_equal(a[k][f], b[k][f]), (k, f)


CONFIGS = {
    "r10-W4096-b64": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=5), 4096, 64),
    "r10-W1024-b4": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=5), 1024, 4),
    "r9": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=7, profile="r9"), 4096, 64),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_parity_with_uploaded_store(name):
    """One launch of every target: segments and every debug window (tokens, quals, supported, sup_rows, logits) are identical.
    Read 0 and read n-1 are targets and queries of that launch: the first and last reads of the uploaded store sit next to its
    padding, and in the gathered layout read 0 is the first read, next to the front padding."""
    make, W, b = CONFIGS[name]
    rs = make()
    targets = targets_of(rs)
    qids = set(int(q) for q in rs.ovl9[:, 0])
    assert {0, rs.n - 1} <= set(targets) and {0, rs.n - 1} <= qids and targets[0] == 0
    want = run(make_ctx(rs, W, b), rs, targets, W)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    got = run(make_ctx(rs, W, b, store), rs, targets, W)
    assert got[0] == want[0] and any(want[0].values()) and got[1] == want[1] == {}
    same_windows(got[2], want[2])
    if name != "r10-W4096-b64":
        return
    # hb_submit_target (host windowing) and hb_features_batch (host and device outputs)
    want_t = run(make_ctx(rs, W, b), rs, targets, W, submit_target=True)
    got_t = run(make_ctx(rs, W, b, store), rs, targets, W, submit_target=True)
    assert got_t[0] == want_t[0] == want[0]
    same_windows(got_t[2], want_t[2])
    up, host = make_ctx(rs, W, b), make_ctx(rs, W, b, store)
    tl = [(t, overlaps(rs, t)) for t in targets]
    for device in (False, True):
        F, G = up.features_batch(tl, device=device, batches=True), host.features_batch(tl, device=device, batches=True)
        for k in api.FEATURES_OUT_FIELDS + ("batch_win",):
            x, y = getattr(F, k), getattr(G, k)
            if isinstance(x, torch.Tensor):
                x, y = x.cpu().numpy(), y.cpu().numpy()
            assert np.array_equal(x, y), (device, k)


@pytest.mark.parametrize("launch_targets", [1, 3])
def test_many_launches_match_one_launch(launch_targets):
    """Small launches put every read of the set first (as a target) and last (as a query) in some gathered layout, and every lane
    gathers several different read lists: the results equal the one-launch run."""
    make, W, b = CONFIGS["r10-W4096-b64"]
    rs = make()
    targets = targets_of(rs)
    want = run(make_ctx(rs, W, b), rs, targets, W, windows=False)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctx = make_ctx(rs, W, b, store, launch_targets=launch_targets)
    got = run(ctx, rs, targets, W, windows=False)
    assert got[0] == want[0] and got[1] == {}
    assert ctx.stats()["device_launches"] == (len(targets) + launch_targets - 1) // launch_targets


def padded_bytes(n):
    """What k_reads_in moves for a read of n bases: its words and qualities, each rounded up to 16 bytes."""
    return (n + 63) // 64 * 16 + (n + 15) // 16 * 16


def test_only_the_launchs_reads_cross_pcie():
    """With 256 MB of filler reads that no alignment references (kept to a few hundred MB of pinned memory on a shared host),
    attaching moves len[] and the ln table only, and every launch moves exactly its distinct reads (padded) and its read list
    more than an uploaded-store context running the same launches."""
    base = helpers.small_readset(n_reads=40, mean_len=9000, seed=5)
    rng = np.random.default_rng(1)
    n_fill, fill_len = 12800, 20000
    fill = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n_fill * fill_len, dtype=np.uint8)]
    seqs = np.concatenate([base.seqs, fill])
    quals = np.concatenate([base.quals, np.full(n_fill * fill_len, 40, np.uint8)])
    off = np.concatenate([base.off, base.off[-1] + fill_len * np.arange(1, n_fill + 1, dtype=np.uint64)])
    lens = np.diff(off).astype(np.int64)
    assert int(lens.sum()) * 5 // 4 > 300 * 10 ** 6
    W, b, lt = 4096, 64, 3
    up = api.Context(helpers.model_path(seed=3), 0, W, b, launch_targets=lt)
    up.upload_reads(seqs, quals, off)
    store = api.ReadStore(seqs, quals, off)
    host = api.Context(helpers.model_path(seed=3), 0, W, b, launch_targets=lt)
    h0 = host.stats()["h2d_bytes"]
    host.attach_read_store(store)
    assert host.stats()["h2d_bytes"] - h0 == 4 * len(lens) + 8 * (int(lens.max()) + 2)
    targets = targets_of(base)
    for k in range(0, len(targets), lt):
        launch = targets[k:k + lt]
        reads = list(dict.fromkeys(launch + [int(q) for t in launch for q in base.ovl9[int(base.aln_off[t]):int(base.aln_off[t + 1]), 0]]))
        d = []
        res = []
        for ctx in (up, host):
            s0 = ctx.stats()["h2d_bytes"]
            for t in launch:
                ctx.submit_alignments(t, overlaps(base, t))
            ctx.flush()
            res.append({r.rid: r.segments for r in ctx.drain()})
            d.append(ctx.stats()["h2d_bytes"] - s0)
        assert res[0] == res[1] and len(res[0]) == len(launch)
        assert d[1] - d[0] == sum(padded_bytes(int(lens[r])) for r in reads) + READ_COPY_BYTES * len(reads), (k, d)
    host.close()
    up.close()
    store.close()


def test_contexts_share_one_store_from_two_threads():
    make, W, b = CONFIGS["r10-W4096-b64"]
    rs = make()
    targets = targets_of(rs)
    want = run(make_ctx(rs, W, b), rs, targets, W, windows=False)[0]
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    devs = (0, 1) if torch.cuda.device_count() > 1 else (0, 0)
    ctxs = [make_ctx(rs, W, b, store, launch_targets=4, device=d) for d in devs]
    out = [None, None]

    def work(i):
        out[i] = run(ctxs[i], rs, targets, W, windows=False)[0]

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert out[0] == want and out[1] == want


def test_replay_failures_state_and_round_trips():
    make, W, b = CONFIGS["r10-W4096-b64"]
    rs = make()
    targets = targets_of(rs)
    want = run(make_ctx(rs, W, b), rs, targets, W)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctx = make_ctx(rs, W, b, store)
    got = run(ctx, rs, targets, W)
    # replay re-runs the gather; the launch it re-runs still has the same windows
    assert ctx.replay_last_launch(2) > 0
    t = targets[0]
    same_windows({(t, 0): ctx.debug_window(t, 0)}, {(t, 0): got[2][(t, 0)]})
    # destroying an attached store is refused, and it stays usable
    with pytest.raises(api.HerroError) as ei:
        store.close()
    assert ei.value.code == HB_ERR_STATE
    assert run(ctx, rs, targets, W, windows=False)[0] == want[0]
    # attach with targets pending
    ctx.submit_alignments(t, overlaps(rs, t))
    with pytest.raises(api.HerroError) as ei:
        ctx.attach_read_store(store)
    assert ei.value.code == HB_ERR_STATE
    ctx.flush()
    ctx.drain()
    # attach -> upload -> attach
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    assert run(ctx, rs, targets, W, windows=False)[0] == want[0]
    store.close()  # nothing attached any more
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctx.attach_read_store(store)
    again = run(ctx, rs, targets, W)
    assert again[0] == want[0]
    same_windows(again[2], want[2])
    # a malformed CIGAR fails only its target
    victim = next(t for t in targets if rs.aln_off[t + 1] - rs.aln_off[t] >= 2)
    bad = np.frombuffer(b"999999M", dtype=np.uint8).copy()
    results = []
    for c in (make_ctx(rs, W, b), make_ctx(rs, W, b, store)):
        for t in targets:
            o = overlaps(rs, t)
            if t == victim:
                o["cigar"][0] = bad.ctypes.data
                o["cigar_len"][0] = len(bad)
            c.submit_alignments(t, o)
        c.flush()
        results.append(({r.rid: r.segments for r in c.drain(skip_failed=True)}, [(rid, code) for rid, code, _ in c.failed]))
    assert results[0] == results[1] and results[1][1] == [(victim, HB_ERR_INPUT)]
    assert all(results[1][0][t] == want[0][t] for t in targets if t != victim)


def test_inference_on_each_store(tmp_path):
    """`inference` forced to the host store and to uploaded stores writes the same FASTA records."""
    from tools import synth
    rs = helpers.small_readset(n_reads=40, mean_len=7000, seed=14, min_len=4200)
    fq = str(tmp_path / "reads.fastq")
    synth.write_fastq(rs, fq)
    synth.write_oec_batches(rs, str(tmp_path / "alns"), batch_size=7)
    outs = []
    for mode in ("device", "host"):
        out = str(tmp_path / f"{mode}.fasta")
        r = hostio.inference(fq, str(tmp_path / "alns"), helpers.model_path(seed=3), out, threads=2, read_store=mode)
        assert r["failed_targets"] == 0 and r["records"] > 0
        outs.append(sorted(open(out, "rb").read().split(b">")[1:]))
    assert outs[0] == outs[1]
