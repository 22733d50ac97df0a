"""hb_forward_batch (Context.forward_batch): the model call alone on caller-collated reference batches.  Against the pipeline's
own logits bit for bit, against the float64 graph on inputs the features stage never produces, across forward passes, through
torch CUDA tensors, on bad input, beside a running pipeline, in the steady state, and through `cli predict`."""
import os
import threading

import numpy as np
import pytest
import torch

import helpers
from herro_b200 import api, cli, hostio, weights as hbw
from test_gpu_model_shapes import SHAPES, pad_model, run_batch64

pytestmark = pytest.mark.gpu
HB_ERR_ARG, HB_ERR_INPUT = -1, -4
POS = hbw.NetConfig(pos_layers=2, pos_heads=8, pos_ffn=1024)
CFGS = dict({k: s.cfg for k, s in SHAPES.items()}, pos=POS)
DUMP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "features_dump")


def model(tmp_path, name):
    return pad_model(CFGS[name], str(tmp_path / f"{name}.hbw"))


def reference_net(name, path):
    """The reference graph of a model file in float64 (with the position-axis stage where the model has one)."""
    from oracle import forward_ref
    from tools import pos_forward_ref
    cfg, T = hbw.load_blob(path)
    net = pos_forward_ref.from_weights(cfg, T) if cfg.pos_layers else forward_ref.from_weights(cfg, T)
    return net.double()


def pipeline_batches(ctx, rs, targets, W, b):
    """Each read's reference batches rebuilt from the pipeline's debug taps (collate over groups of b windows), with the
    pipeline's logits of those windows."""
    out = []
    for t in targets:
        nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
        wins = [ctx.debug_window(t, w) for w in range(nw)]
        for g0 in range(0, nw, b):
            grp = [wins[w] for w in range(g0, min(g0 + b, nw)) if len(wins[w]["sup_rows"])]
            if not grp:
                continue
            lmax = max(d["L"] for d in grp)
            bases = np.full((len(grp), lmax, 31), 11, np.uint8)
            quals = np.full((len(grp), lmax, 31), 126, np.uint8)
            for k, d in enumerate(grp):
                bases[k, :d["L"]] = d["bases"]
                quals[k, :d["L"]] = d["quals"]
            out.append(dict(bases=bases, quals=quals, lens=[len(d["sup_rows"]) for d in grp],
                            indices=[d["sup_rows"].astype(np.int32) for d in grp],
                            info=[d["info_logits"] for d in grp], bl=[d["bases_logits"] for d in grp]))
    return out


def targets_of(rs, n=16):
    return [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]][:n]


def same_bits(got, want):
    return len(got) == len(want) and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------ 1. the pipeline's bits
PIPE = [(m, W, b, simt) for m in ("default", "ts-shape", "wide", "pos") for W, b in ((4096, 64), (1024, 4)) for simt in (False,)] + \
       [("default", W, b, True) for W, b in ((4096, 64), (1024, 4))]


@pytest.mark.parametrize("name,W,b,simt", PIPE, ids=[f"{m}-W{W}-b{b}" + ("-simt" if s else "") for m, W, b, s in PIPE])
def test_same_bits_as_the_pipeline(monkeypatch, tmp_path, name, W, b, simt):
    if simt:
        monkeypatch.setenv("HERRO_B200_STEM_SIMT", "1")
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=5)
    targets = targets_of(rs)
    got = helpers.run_product(rs, model(tmp_path, name), W, b, targets=targets, keep_debug=True, dump=False)
    ctx = got["ctx"]
    batches = pipeline_batches(ctx, rs, targets, W, b)
    assert batches
    if b == 4:  # windows shorter than their batch: the batch-padding rows are part of the input
        assert any(len({x.shape[0] for x in B["indices"]}) > 1 for B in batches)
    n = 0
    for B in batches:
        info, bl = ctx.forward_batch(B["bases"], B["quals"], B["lens"], B["indices"])
        assert same_bits(info, B["info"]) and same_bits(bl, B["bl"])
        n += sum(B["lens"])
    print(f"{name} W{W} -b{b}{' SIMT stem' if simt else ''}: {len(batches)} batches, {n} positions bit-identical")


# ------------------------------------------------------------------------------------------ 2. float64 on any input
def random_batch(rng, B, Lmax, qlo=33, qhi=126, max_len=24):
    """Tokens uniform in 0..11 (token 11 inside windows), some windows without positions, unsorted and duplicated indices
    that include rows 0 and Lmax - 1."""
    bases = rng.integers(0, 12, (B, Lmax, 31), dtype=np.uint8)
    quals = rng.integers(qlo, qhi, (B, Lmax, 31), dtype=np.uint8, endpoint=True)
    lens = rng.integers(1, max_len + 1, B)
    lens[rng.random(B) < 0.2] = 0
    lens[0] = max(int(lens[0]), 3)
    idx = []
    for n in lens:
        i = rng.integers(0, Lmax, int(n)).astype(np.int32)
        if n >= 3:
            i[0], i[-1], i[1] = 0, Lmax - 1, i[2]
        idx.append(i)
    return bases, quals, [int(x) for x in lens], idx


@pytest.mark.parametrize("name", list(CFGS))
def test_against_float64_on_any_input(tmp_path, name):
    from herro_b200 import Context
    path = model(tmp_path, name)
    net = reference_net(name, path)
    K = CFGS[name].stem_k
    ctx = Context(path, 0)
    rng = np.random.default_rng(17)
    cases = [(1, 1, 126), (64, max(1, K // 2), 126), (8, max(1, K - 1), 255), (8, 300, 126), (1, 5000, 126)]
    worst = 0.0
    for B, Lmax, qhi in cases:
        bases, quals, lens, idx = random_batch(rng, B, Lmax, qlo=0 if qhi == 255 else 33, qhi=qhi)
        info, bl = ctx.forward_batch(bases, quals, lens, idx)
        ri, rb = run_batch64(net, bases, quals, lens, idx)
        for k in range(B):
            err = max(float(np.abs(info[k] - ri[k]).max(initial=0.0)), float(np.abs(bl[k] - rb[k]).max(initial=0.0)))
            assert err <= 1e-3, (name, B, Lmax, k, err)
            worst = max(worst, err)
    print(f"{name}: worst |logit - float64| {worst:.2e}")


# ------------------------------------------------------------------------------------------ 3. forward passes
@pytest.mark.parametrize("name", ["default", "pos"])
def test_chunked_passes_give_the_same_bits(monkeypatch, tmp_path, name):
    from herro_b200 import Context
    path = model(tmp_path, name)
    rng = np.random.default_rng(5)
    bases, quals, lens, idx = random_batch(rng, 16, 400, max_len=60)
    lens[3] = 300
    idx[3] = rng.integers(0, 400, 300).astype(np.int32)
    assert sum(lens) > 4 * 128
    want = Context(path, 0).forward_batch(bases, quals, lens, idx)
    monkeypatch.setenv("HERRO_B200_CHUNK_POS", "128")
    ctx = Context(path, 0)
    got = ctx.forward_batch(bases, quals, lens, idx)
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1])
    assert ctx.stats()["n_kernel"]["heads"] >= 4  # several passes, one of them the window with 300 positions alone


# ------------------------------------------------------------------------------------------ 4. torch CUDA tensors
def test_torch_tensors_on_a_side_stream(tmp_path):
    from herro_b200 import Context
    ctx = Context(model(tmp_path, "default"), 0)
    rng = np.random.default_rng(9)
    bases, quals, lens, idx = random_batch(rng, 64, 500)
    want = ctx.forward_batch(bases, quals, lens, idx)
    src_b, src_q = torch.from_numpy(bases).cuda(), torch.from_numpy(quals).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        buf = torch.zeros(bases.size + 1, dtype=torch.uint8, device="cuda")
        tb = buf[1:].view(bases.shape)  # starts at an odd byte
        tb.copy_((src_b.to(torch.int32) * 3 - src_b.to(torch.int32) * 2).to(torch.uint8))
        tq = (src_q.to(torch.int32) + 0).to(torch.uint8)
        assert tb.data_ptr() % 2 == 1 and tb.is_contiguous()
        info, bl = ctx.forward_batch(tb, tq, torch.tensor(lens), [torch.from_numpy(i) for i in idx])
    assert all(t.is_cuda for t in info + bl)
    assert same_bits([t.cpu().numpy() for t in info], want[0]) and same_bits([t.cpu().numpy() for t in bl], want[1])


# ------------------------------------------------------------------------------------------ 5. errors
def pipeline(ctx, rs, targets):
    """Submit, flush, drain: {rid: segments}."""
    for t in targets:
        a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
        ctx.submit_alignments(t, api.Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
    ctx.flush()
    return {r.rid: r.segments for r in ctx.drain()}


def test_errors_leave_the_context_usable(tmp_path):
    from herro_b200 import Context
    path = model(tmp_path, "default")
    rs = helpers.small_readset(n_reads=24, mean_len=9000, seed=3)
    targets = targets_of(rs, 24)
    fresh = Context(path, 0)
    fresh.upload_reads(rs.seqs, rs.quals, rs.off)
    want_pipe = pipeline(fresh, rs, targets)
    ctx = Context(path, 0)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    rng = np.random.default_rng(4)
    bases, quals, lens, idx = random_batch(rng, 8, 200)
    want = ctx.forward_batch(bases, quals, lens, idx)

    def still_good():
        got = ctx.forward_batch(bases, quals, lens, idx)
        assert same_bits(got[0], want[0]) and same_bits(got[1], want[1])
        assert pipeline(ctx, rs, targets) == want_pipe

    bad = bases.copy()
    bad[5, 17, 30] = 12
    bad[6, 0, 0] = 200  # later in row-major order: not the one named
    with pytest.raises(api.HerroError) as e:
        ctx.forward_batch(bad, quals, lens, idx)
    assert e.value.code == HB_ERR_INPUT and "(5, 17, 30)" in str(e.value), str(e.value)
    still_good()
    for r in (200, -1):
        bidx = [i.copy() for i in idx]
        bidx[0][1] = r
        with pytest.raises(api.HerroError) as e:
            ctx.forward_batch(bases, quals, lens, bidx)
        assert e.value.code == HB_ERR_ARG, str(e.value)
        still_good()
    flat = np.concatenate(idx).astype(np.int32)
    ln = np.asarray(lens, np.int32)
    out_i, out_b = np.zeros(len(flat), np.float32), np.zeros((len(flat), 5), np.float32)
    rc = ctx._L.hb_forward_batch(ctx._h, 8, 200, bases.ctypes.data, quals.ctypes.data, ln.ctypes.data, flat.ctypes.data,
                                 out_i.ctypes.data, out_b.ctypes.data, api.HB_FWD_DEVICE_PTRS, None)
    assert rc == HB_ERR_ARG
    still_good()


# ------------------------------------------------------------------------------------------ 6. beside the pipeline
def test_concurrent_with_the_pipeline(tmp_path):
    from herro_b200 import Context
    path = model(tmp_path, "default")
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=8)
    targets = targets_of(rs, 40)
    ctx = Context(path, 0)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    rng = np.random.default_rng(6)
    batches = [random_batch(rng, int(rng.integers(1, 65)), int(rng.integers(50, 800))) for _ in range(12)]
    want_pipe = pipeline(ctx, rs, targets)
    want_fwd = [ctx.forward_batch(*x) for x in batches]
    got_pipe, got_fwd = {}, []
    th = threading.Thread(target=lambda: got_pipe.update(pipeline(ctx, rs, targets)))
    th.start()
    for x in batches:
        got_fwd.append(ctx.forward_batch(*x))
    th.join()
    assert got_pipe == want_pipe
    for g, w in zip(got_fwd, want_fwd):
        assert same_bits(g[0], w[0]) and same_bits(g[1], w[1])


# ------------------------------------------------------------------------------------------ 7. steady state
def test_steady_state_allocates_nothing(tmp_path):
    from herro_b200 import Context
    ctx = Context(model(tmp_path, "default"), 0)
    rng = np.random.default_rng(2)
    first = random_batch(rng, 64, 600)
    ctx.forward_batch(*first)
    ctx.reset_stats()
    for k in range(10):
        B, Lmax = (64, 600) if k % 3 == 0 else (int(rng.integers(1, 65)), int(rng.integers(1, 601)))
        x = first if k % 3 == 0 else random_batch(rng, B, Lmax)
        if k % 2:
            ctx.forward_batch(torch.from_numpy(x[0]).cuda(), torch.from_numpy(x[1]).cuda(), x[2], x[3])
        else:
            ctx.forward_batch(*x)
    s = ctx.stats()
    assert s["host_allocs"] == 0, s["host_allocs"]
    assert s["n_kernel"]["lists"] == 10 and s["n_kernel"]["heads"] >= 10 and s["supported"] > 0 and s["ms_forward"] > 0
    assert s["targets"] == s["windows"] == s["rows"] == s["corrected_bases"] == 0


# ------------------------------------------------------------------------------------------ 8. cli predict
def test_cli_predict_on_the_golden_dump(tmp_path):
    from oracle import forward_ref
    from tools import make_feature_fixture as mf
    path = helpers.model_path(seed=3)
    out = str(tmp_path / "logits")
    cli.main(["predict", "-m", path, "-b", "4", DUMP, out])
    cfg, T = hbw.load_blob(path)
    net = forward_ref.from_weights(cfg, T)
    rs = mf.readset()
    got = helpers.run_product(rs, path, mf.W, 4, targets=list(mf.TARGETS), keep_debug=True)
    n = 0
    for t in mf.TARGETS:
        read_dir = os.path.join(DUMP, rs.ids[t])
        for fb in hostio.read_feature_batches(read_dir, 4):
            ri, rb = forward_ref.run_batch(net, fb.bases, fb.quals, fb.lens, fb.indices)
            for k, wid in enumerate(fb.wids):
                info = np.load(os.path.join(out, rs.ids[t], f"{wid}.info_logits.npy"))
                bl = np.load(os.path.join(out, rs.ids[t], f"{wid}.bases_logits.npy"))
                assert info.dtype == np.float32 and bl.shape == (len(info), 5)
                assert np.abs(info - ri[k]).max() <= 1e-3 and np.abs(bl - rb[k]).max() <= 1e-3
                w = got["windows"][(t, wid)]
                assert np.array_equal(info, w["info_logits"]) and np.array_equal(bl, w["bases_logits"])
                n += 1
    assert n >= 6
    assert sum(len(f) for _, _, f in os.walk(out)) == 2 * n
