"""hb_consensus_batch (Context.consensus_batch): consensus alone on caller-supplied windows and logits.  Against the pipeline's own
segments byte for byte, against the oracle's consensus() on adversarial windows, on the hand-derived rules, on bad input, through
torch CUDA tensors fed by forward_batch, beside a running pipeline, in the steady state, and through `cli features -> predict ->
consensus` against `cli inference`."""
import os
import threading

import numpy as np
import pytest
import torch

import consensus_oracle
import helpers
from herro_b200 import api, cli, hostio
from test_consensus_batch_cpu import HAND
from test_gpu_forward_batch import pipeline, targets_of

pytestmark = pytest.mark.gpu
HB_ERR_ARG, HB_ERR_INPUT = -1, -4
DUMP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "features_dump")


def tap_windows(ctx, rs, targets, W):
    """Each target's windows in wid order, rebuilt from the pipeline's debug taps."""
    out = []
    for t in targets:
        nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
        wins = []
        for w in range(nw):
            d = ctx.debug_window(t, w)
            wins.append(hostio.ConsensusWindow(w, d["n_alns"], d["bases"], d["supported"].reshape(-1, 2), d["bases_logits"].reshape(-1, 5)))
        out.append(wins)
    return out


def want_segments(got, targets):
    return [got["segments"].get(t) or [] for t in targets]


# ------------------------------------------------------------------------------------------ 1. the pipeline's segments
@pytest.mark.parametrize("profile,W,b,seed", [("r10", 4096, 64, 5), ("r10", 1024, 4, 5), ("r9", 4096, 64, 7)],
                         ids=["r10-W4096-b64", "r10-W1024-b4", "r9"])
def test_same_segments_as_the_pipeline(profile, W, b, seed):
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=seed, profile=profile)
    targets = targets_of(rs, 40)
    got = helpers.run_product(rs, helpers.model_path(seed=3), W, b, targets=targets, keep_debug=True, dump=False)
    ctx = got["ctx"]
    reads = tap_windows(ctx, rs, targets, W)
    want = want_segments(got, targets)
    assert sum(len(s) for s in want) >= len(targets) // 2
    assert ctx.consensus_batch(*hostio.consensus_args(reads)) == want
    for r, w in zip(reads, want):
        assert ctx.consensus_batch(*hostio.consensus_args([r])) == [w]
    print(f"{profile} W{W} -b{b}: {len(targets)} reads, {sum(len(b) for s in want for b in s)} bases identical")


# ------------------------------------------------------------------------------------------ 2. the oracle on adversarial input
def row_keys(col0):
    idx = np.arange(len(col0), dtype=np.int64)
    tgt = col0 != 4
    pos = (np.cumsum(tgt) - 1) & 0xFFFF
    last = np.maximum.accumulate(np.where(tgt, idx + 1, 0))
    return pos.astype(np.uint32), ((idx + 1 - last) & 0xFF).astype(np.uint32)


LOGIT_VALUES = np.array([-1.0, 0.0, -0.0, 1.0, 1.0, np.nan, np.inf, -np.inf, 2.5], np.float32)


def random_window(rng, L, n_alns, gap_p=0.3, gap_run=0):
    b = rng.integers(11, 256, (L, 31), dtype=np.uint8)  # >= 11 wherever consensus does not read
    if n_alns >= 2:
        b[:, 1:n_alns + 1] = rng.integers(0, 11, (L, n_alns), dtype=np.uint8)
        col0 = rng.integers(0, 10, L, dtype=np.uint8)
        col0[rng.random(L) < gap_p] = 4
        if gap_run:
            s = int(rng.integers(0, max(L - gap_run, 1)))
            col0[s:s + gap_run] = 4
        b[:, 0] = col0
        pos, ins = row_keys(col0)
    else:
        pos = ins = np.zeros(0, np.uint32)
    n = int(rng.integers(0, max(L // 3, 1) + 1))
    keys = [(int(pos[r]), int(ins[r])) for r in rng.integers(0, L, n)] if L and len(pos) else []
    keys += [(int(rng.integers(0, 65536)), int(rng.integers(0, 256))) for _ in range(int(rng.integers(0, 4)))]  # unmatched (mostly)
    if keys and rng.random() < 0.5:
        keys += keys[:int(rng.integers(1, len(keys) + 1))]  # duplicates, later ones win
    rng.shuffle(keys)
    sup = np.array(keys, np.uint32).reshape(-1, 2)
    bl = rng.choice(LOGIT_VALUES, (len(sup), 5)).astype(np.float32)
    return hostio.ConsensusWindow(0, n_alns, b, sup, bl)


def as_oracle(reads):
    return [[(w.bases, w.n_alns, w.supported, w.bases_logits) for w in r] for r in reads]


def test_against_the_oracle_on_adversarial_windows():
    from herro_b200 import Context
    ctx = Context(helpers.model_path(seed=3), 0)
    rng = np.random.default_rng(23)
    reads = []
    for _ in range(60):
        reads.append([random_window(rng, int(rng.integers(0, 400)), int(rng.integers(0, 31))) for _ in range(int(rng.integers(0, 7)))])
    reads.append([random_window(rng, 70000, 2, gap_p=0.05)])  # more than 65 536 target rows: pos wraps, keys match two rows
    reads.append([random_window(rng, 2000, 3, gap_p=0.1, gap_run=600)])  # a '*' run over 256 rows: ins wraps
    assert sum(len(w.supported) for r in reads for w in r) > 5000
    want = consensus_oracle.consensus_windows(as_oracle(reads))
    assert ctx.consensus_batch(*hostio.consensus_args(reads)) == want
    assert sum(1 for s in want if s) > 20
    for k in (-2, -1):
        assert ctx.consensus_batch(*hostio.consensus_args([reads[k]])) == [want[k]]


# ------------------------------------------------------------------------------------------ 3. the rules and the errors
def hand_args(reads):
    return hostio.consensus_args([[hostio.ConsensusWindow(i, w[1], w[0], w[2], w[3]) for i, w in enumerate(r)] for r in reads])


def test_hand_derived_rules_and_errors():
    from herro_b200 import Context
    ctx = Context(helpers.model_path(seed=3), 0)
    rng = np.random.default_rng(31)
    good = [[random_window(rng, int(rng.integers(1, 300)), int(rng.integers(2, 31))) for _ in range(3)] for _ in range(6)]
    good_args = hostio.consensus_args(good)
    want_good = ctx.consensus_batch(*good_args)

    def still_good():
        assert ctx.consensus_batch(*good_args) == want_good

    for name, (reads, want) in HAND.items():
        if isinstance(want, tuple):
            with pytest.raises(api.HerroError) as e:
                ctx.consensus_batch(*hand_args(reads))
            assert e.value.code == HB_ERR_INPUT and "(%d, %d, %d, %d)" % want[1] in str(e.value), (name, str(e.value))
            still_good()
        else:
            assert ctx.consensus_batch(*hand_args(reads)) == want, name
    # HB_ERR_ARG: n_alns 31, pos 65536, ins 256
    base = hand_args(HAND["argmax"][0])
    for bad in ({2: [31]}, {4: [np.array([[65536, 0]] * 5, np.uint32)]}, {4: [np.array([[0, 256]] * 5, np.uint32)]}):
        args = list(base)
        for k, v in bad.items():
            args[k] = v
        with pytest.raises(api.HerroError) as e:
            ctx.consensus_batch(*args)
        assert e.value.code == HB_ERR_ARG, str(e.value)
        still_good()
    # NULL, and pointers that do not match the flag
    nwin, rows, nal = np.array([1], np.uint32), np.array([1], np.uint32), np.array([2], np.uint8)
    b, nsup, sup, bl = np.zeros((1, 31), np.uint8), np.zeros(1, np.uint32), np.zeros((1, 2), np.uint32), np.zeros((1, 5), np.float32)
    seqs, seg_len, n_segs = np.zeros(4, np.uint8), np.zeros(4, np.uint32), np.zeros(4, np.uint32)
    tb, tbl = torch.zeros((1, 31), dtype=torch.uint8, device="cuda"), torch.zeros((1, 5), device="cuda")
    torch.cuda.synchronize()

    def call(bases_p, logits_p, flags, n_alns_p=nal.ctypes.data):
        return ctx._L.hb_consensus_batch(ctx._h, 1, nwin.ctypes.data, rows.ctypes.data, n_alns_p, bases_p, nsup.ctypes.data,
                                         sup.ctypes.data, logits_p, seqs.ctypes.data, seg_len.ctypes.data, n_segs.ctypes.data, flags, None)

    assert call(b.ctypes.data, bl.ctypes.data, 0) == 0 and n_segs[0] == 1 and seqs[0] == ord("A")
    n_segs[:] = 7
    for args in ((None, bl.ctypes.data, 0), (b.ctypes.data, bl.ctypes.data, 0, None),
                 (b.ctypes.data, bl.ctypes.data, api.HB_CONS_DEVICE_PTRS), (tb.data_ptr(), bl.ctypes.data, api.HB_CONS_DEVICE_PTRS),
                 (tb.data_ptr(), tbl.data_ptr(), 0), (b.ctypes.data, tbl.data_ptr(), 0),
                 (tb.data_ptr(), tbl.data_ptr(), api.HB_CONS_DEVICE_PTRS, torch.tensor([2], dtype=torch.uint8, device="cuda").data_ptr())):
        assert call(*args) == HB_ERR_ARG, args
        assert n_segs[0] == 7  # nothing written
        still_good()
    assert call(tb.data_ptr(), tbl.data_ptr(), api.HB_CONS_DEVICE_PTRS) == 0 and n_segs[0] == 1


# ------------------------------------------------------------------------------------------ 4. device pointers
def test_cuda_tensors_and_forward_batch_without_a_host_round_trip():
    W, b = 1024, 4
    rs = helpers.small_readset(n_reads=30, mean_len=9000, seed=5)
    targets = targets_of(rs, 16)
    got = helpers.run_product(rs, helpers.model_path(seed=3), W, b, targets=targets, keep_debug=True, dump=False)
    ctx = got["ctx"]
    reads = tap_windows(ctx, rs, targets, W)
    want = want_segments(got, targets)
    args = hostio.consensus_args(reads)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        buf = torch.zeros(args[3].size + 1, dtype=torch.uint8, device="cuda")
        tb = buf[1:].view(args[3].shape)  # starts at an odd byte
        tb.copy_(torch.from_numpy(args[3]).cuda())
        assert ctx.consensus_batch(args[0], args[1], args[2], tb, args[4], torch.from_numpy(args[5]).cuda()) == want
    # forward_batch on CUDA tensors feeding consensus_batch: the logits stay on the device
    logits = {}
    for t, wins in zip(targets, reads):
        for g0 in range(0, len(wins), b):
            grp = [w for w in wins[g0:g0 + b] if len(w.supported)]
            if not grp:
                continue
            lmax = max(w.bases.shape[0] for w in grp)
            bases = np.full((len(grp), lmax, 31), 11, np.uint8)
            quals = np.full((len(grp), lmax, 31), 126, np.uint8)
            idx = []
            for k, w in enumerate(grp):
                d = ctx.debug_window(t, w.wid)
                bases[k, :d["L"]] = d["bases"]
                quals[k, :d["L"]] = d["quals"]
                idx.append(d["sup_rows"].astype(np.int32))
            _, bl = ctx.forward_batch(torch.from_numpy(bases).cuda(), torch.from_numpy(quals).cuda(), [len(i) for i in idx], idx)
            for w, x in zip(grp, bl):
                logits[(t, w.wid)] = x
    dev_bl = torch.cat([logits[(t, w.wid)] for t, r in zip(targets, reads) for w in r if len(w.supported)])
    assert dev_bl.is_cuda
    assert ctx.consensus_batch(args[0], args[1], args[2], torch.from_numpy(args[3]).cuda(), args[4], dev_bl) == want


# ------------------------------------------------------------------------------------------ 5. concurrency and steady state
def test_beside_the_pipeline_and_forward_batch_threads():
    from test_gpu_forward_batch import random_batch
    from herro_b200 import Context
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=8)
    targets = targets_of(rs, 40)
    ctx = Context(helpers.model_path(seed=3), 0)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    rng = np.random.default_rng(6)
    cons = [hostio.consensus_args([[random_window(rng, int(rng.integers(1, 500)), int(rng.integers(0, 31))) for _ in range(5)]
                                   for _ in range(8)]) for _ in range(10)]
    fwd = [random_batch(rng, int(rng.integers(1, 33)), int(rng.integers(50, 500))) for _ in range(6)]
    want_pipe = pipeline(ctx, rs, targets)
    want_cons = [ctx.consensus_batch(*x) for x in cons]
    want_fwd = [ctx.forward_batch(*x) for x in fwd]
    got_pipe, got_fwd, got_cons = {}, [], [[], []]
    ths = [threading.Thread(target=lambda: got_pipe.update(pipeline(ctx, rs, targets))),
           threading.Thread(target=lambda: got_fwd.extend(ctx.forward_batch(*x) for x in fwd))]
    ths += [threading.Thread(target=lambda k=k: got_cons[k].extend(ctx.consensus_batch(*x) for x in cons)) for k in range(2)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert got_pipe == want_pipe
    assert got_cons[0] == want_cons and got_cons[1] == want_cons
    for g, w in zip(got_fwd, want_fwd):
        assert all(np.array_equal(x, y) for x, y in zip(g[1], w[1]))


def test_steady_state_allocates_nothing():
    from herro_b200 import Context
    ctx = Context(helpers.model_path(seed=3), 0)
    rng = np.random.default_rng(2)
    big = hostio.consensus_args([[random_window(rng, 600, 20) for _ in range(6)] for _ in range(10)])
    ctx.consensus_batch(*big)
    ctx.consensus_batch(big[0], big[1], big[2], torch.from_numpy(big[3]).cuda(), big[4], torch.from_numpy(big[5]).cuda())
    ctx.set_kernel_timing(True)
    ctx.reset_stats()
    for k in range(10):
        x = big if k % 3 == 0 else hostio.consensus_args([[random_window(rng, int(rng.integers(1, 600)), int(rng.integers(0, 31)))
                                                            for _ in range(3)] for _ in range(4)])
        if k % 2:
            ctx.consensus_batch(x[0], x[1], x[2], torch.from_numpy(x[3]).cuda(), x[4], torch.from_numpy(x[5]).cuda())
        else:
            ctx.consensus_batch(*x)
    s = ctx.stats()
    assert s["host_allocs"] == 0, s["host_allocs"]
    assert s["n_kernel"]["consensus"] == 30 and s["n_kernel"]["scan"] == 10 and s["kernel_launches"] == 40
    assert s["ms_consensus"] > 0 and s["ms_kernel"]["consensus"] > 0
    assert s["targets"] == s["windows"] == s["rows"] == s["corrected_bases"] == s["supported"] == 0 and s["ms_forward"] == 0


# ------------------------------------------------------------------------------------------ 6. the CLI chain
def fasta_records(path):
    recs = open(path, "rb").read().split(b">")[1:]
    return sorted(recs)


def test_cli_features_predict_consensus_equals_inference(tmp_path):
    model = helpers.model_path(seed=3)
    reads, alns = os.path.join(DUMP, "reads.fastq"), os.path.join(DUMP, "alns")
    feats, logits = str(tmp_path / "features"), str(tmp_path / "logits")
    cli.main(["features", "--read-alns", alns, "-w", "256", "-m", model, reads, feats])
    cli.main(["predict", "-m", model, "-b", "4", feats, logits])
    cli.main(["consensus", "-m", model, "--rows-per-call", "2000", feats, logits, reads, str(tmp_path / "staged.fasta")])
    cli.main(["inference", "--read-alns", alns, "-w", "256", "-m", model, "-b", "4", reads, str(tmp_path / "fused.fasta")])
    got, want = fasta_records(str(tmp_path / "staged.fasta")), fasta_records(str(tmp_path / "fused.fasta"))
    assert len(want) >= 3
    assert got == want
