"""hb_features_batch / hb_features_fetch (Context.features_batch): the features stage alone.  Against the pipeline's debug taps
window by window, against the committed fixture and the oracle's batches, through the staged route features -> forward_batch ->
consensus_batch against the fused pipeline, with a TorchScript graph the library rejects run by `cli inference --torch`, and on
per-target failures, call errors, a context without weights, a pipeline running beside it and the steady state."""
import os
import threading
from typing import List, Tuple

import numpy as np
import pytest
import torch

import consensus_oracle
import helpers
from herro_b200 import api, cli, hostio
from test_gpu_forward_batch import model, pipeline_batches, targets_of

pytestmark = pytest.mark.gpu
HB_ERR_ARG, HB_ERR_INPUT, HB_ERR_MODEL, HB_ERR_STATE = -1, -4, -3, -6
DUMP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "features_dump")


def overlaps(rs, t):
    a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
    return api.Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1])


def same_window(f, d):
    assert f["L"] == d["L"] and f["n_alns"] == d["n_alns"]
    assert np.array_equal(f["bases"], d["bases"]) and np.array_equal(f["quals"], d["quals"])
    assert np.array_equal(f["supported"], d["supported"].reshape(-1, 2)) and np.array_equal(f["sup_rows"], d["sup_rows"])


def check_against_taps(ctx, F, rs, targets, W, b):
    """Every window of F equals the pipeline's debug taps, and F's batches equal the batches collated from them."""
    assert list(F.status) == [0] * len(targets) and F.rids == list(targets)
    n = 0
    for k, t in enumerate(targets):
        nw = (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W
        assert F.n_windows[k] == nw
        for wid in range(nw):
            same_window(F.window(int(F.win_off[k]) + wid), ctx.debug_window(t, wid))
            n += 1
    want = pipeline_batches(ctx, rs, targets, W, b)
    got = list(F.batches())
    assert len(got) == len(want) > 0
    for (wins, bases, quals, lens, idx), B in zip(got, want):
        assert np.array_equal(bases, B["bases"]) and np.array_equal(quals, B["quals"]) and list(lens) == list(B["lens"])
        assert all(np.array_equal(a, c) for a, c in zip(idx, B["indices"]))
    return n


def env_set(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ------------------------------------------------------------------------------------------ 1. the pipeline's windows
CONFIGS = {
    "r10-W4096-b64": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=5), 4096, 64, {}),
    "r10-W1024-b4": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=5), 1024, 4, {}),
    "r9": (lambda: helpers.small_readset(n_reads=40, mean_len=9000, seed=7, profile="r9"), 4096, 64, {}),
    "W8192": (lambda: helpers.small_readset(n_reads=30, mean_len=20000, seed=32, profile="r9", coverage=20.0, min_ovl=9000), 8192, 64, {}),
    "over-1024-overlaps": (lambda: helpers.synth.generate(2200, 5000, profile="r10", seed=52, coverage=1000.0, min_ovl=1100, sd_frac=0.05,
                                                          targets=(0, 3)), 1024, 16, {}),
    "arena-overflow": (lambda: helpers.small_readset(n_reads=30, mean_len=7000, seed=51), 4096, 64, {"HERRO_B200_ARENA_ROWS": "64"}),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_same_windows_as_the_pipeline(monkeypatch, name):
    make, W, b, env = CONFIGS[name]
    env_set(monkeypatch, env)
    rs = make()
    targets = targets_of(rs, 40)
    got = helpers.run_product(rs, helpers.model_path(seed=3), W, b, targets=targets, keep_debug=True, dump=False)
    ctx = got["ctx"]
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in targets], batches=True)
    n = check_against_taps(ctx, F, rs, targets, W, b)
    if name == "W8192":
        assert max(F.rows) > 5120 + 3000
    if name == "over-1024-overlaps":
        assert max(F.n_ids) > 1024
    # the device outputs hold the same bytes
    D = ctx.features_batch([(t, overlaps(rs, t)) for t in targets], device=True, batches=True)
    for k in ("bases", "quals", "batch_bases", "batch_quals"):
        assert isinstance(getattr(D, k), torch.Tensor) and np.array_equal(getattr(D, k).cpu().numpy(), getattr(F, k)), k
    for k in ("rows", "n_alns", "n_sup", "n_ids", "supported", "indices", "ids", "batch_B", "batch_Lmax", "batch_win"):
        assert np.array_equal(getattr(D, k), getattr(F, k)), k
    print(f"{name}: {len(targets)} targets, {n} windows identical to the taps")


# ------------------------------------------------------------------------------------------ 2. the fixture and the oracle
def test_fixture_and_oracle():
    """The fixture's targets at W 256 give exactly the tokens, qualities, SupportedPos and ids (as read names) of
    tests/golden/features_dump, and batches equal to the oracle's T.batch(b) and to hostio.read_feature_batches(read_dir, 4)."""
    from test_features_batch_cpu import oracle_targets
    rs, targets = oracle_targets()
    ctx = api.Context(None, 0, 256, 4)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    F = ctx.features_batch([(t, overlaps(rs, t)) for t, _ in targets], batches=True)
    assert list(F.status) == [0] * len(targets)
    got = list(F.batches())
    g = 0
    for k, (t, T) in enumerate(targets):
        read_dir = os.path.join(DUMP, rs.ids[t])
        for wid in range(int(F.n_windows[k])):
            w = F.window(int(F.win_off[k]) + wid)
            tok, q, _ = hostio.read_feature_window(read_dir, wid)
            sup = np.load(os.path.join(read_dir, f"{wid}.supported.npy"))
            assert np.array_equal(w["bases"], tok) and np.array_equal(w["quals"], q)
            assert np.array_equal(w["supported"][:, 0], sup["pos"]) and np.array_equal(w["supported"][:, 1], sup["ins"])
            names = open(os.path.join(read_dir, f"{wid}.ids.txt"), "rb").read().split(b"\n")[:-1]
            assert [rs.ids[int(i)].encode() for i in w["ids"]] == names
        want = hostio.read_feature_batches(read_dir, 4)
        assert len(want) == T.n_batches
        for bi, fb in enumerate(want):
            wins, bases, quals, lens, idx = got[g]
            B = T.batch(bi)
            for ref in (B, fb):
                assert np.array_equal(bases, ref.bases) and np.array_equal(quals, ref.quals) and np.array_equal(lens, ref.lens)
                assert all(np.array_equal(a, c) for a, c in zip(idx, ref.indices))
            assert [x - int(F.win_off[k]) for x in wins] == [int(i) for i in B.win_index] == fb.wids
            g += 1
    assert g == len(got) >= 3


# ------------------------------------------------------------------------------------------ 3. the staged route
@pytest.mark.parametrize("name", ["default", "pos"])
def test_staged_route_equals_the_fused_pipeline(tmp_path, name):
    """Device features -> forward_batch per batch -> consensus_batch, all on CUDA tensors: the pipeline's logits bit for bit, its
    segments byte for byte."""
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=5)
    targets = targets_of(rs, 24)
    got = helpers.run_product(rs, model(tmp_path, name), 4096, 64, targets=targets, keep_debug=True, dump=False)
    ctx = got["ctx"]
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in targets], device=True, batches=True)
    logits = []
    for wins, bases, quals, lens, idx in F.batches():
        info, bl = ctx.forward_batch(bases, quals, lens, idx)
        for w, i, l in zip(wins, info, bl):
            k = int(np.searchsorted(F.win_off, w, side="right")) - 1
            d = ctx.debug_window(targets[k], w - int(F.win_off[k]))
            assert np.array_equal(i.cpu().numpy(), d["info_logits"]) and np.array_equal(l.cpu().numpy(), d["bases_logits"])
        logits.append(bl)
    segs = ctx.consensus_batch(*F.consensus_args(logits))
    assert segs == [got["segments"].get(t) or [] for t in targets]
    assert sum(1 for s in segs if s) >= len(targets) // 2


# ------------------------------------------------------------------------------------------ 4. a graph the library rejects
class OtherNet(torch.nn.Module):
    """The reference's forward signature over a graph this library does not implement."""

    def __init__(self):
        super().__init__()
        self.emb = torch.nn.Embedding(12, 8)
        self.mix = torch.nn.Linear(31 * 9, 48)
        self.base = torch.nn.Linear(48, 5)
        self.info = torch.nn.Linear(48, 1)

    def forward(self, bases: torch.Tensor, quals: torch.Tensor, lens: torch.Tensor,
                indices: List[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        x = torch.cat([self.emb(bases), quals.unsqueeze(-1)], dim=-1)
        x = x.reshape(x.shape[0], x.shape[1], 31 * 9)
        sel: List[torch.Tensor] = []
        for b in range(len(indices)):
            sel.append(x[b].index_select(0, indices[b].to(torch.long)))
        z = torch.relu(self.mix(torch.cat(sel, dim=0)))
        return self.info(z).squeeze(-1), self.base(z)


def test_foreign_torchscript_graph_through_cli_inference_torch(tmp_path):
    from tools import synth
    torch.manual_seed(0)
    pt = str(tmp_path / "other.pt")
    torch.jit.script(OtherNet().eval()).save(pt)
    with pytest.raises(api.HerroError) as ei:
        api.inspect_model(pt)
    assert ei.value.code == HB_ERR_MODEL
    rs = helpers.small_readset(n_reads=30, mean_len=9000, seed=14, min_len=4200)
    fq, alns, out = str(tmp_path / "reads.fastq"), str(tmp_path / "alns"), str(tmp_path / "out.fasta")
    synth.write_fastq(rs, fq)
    synth.write_oec_batches(rs, alns, batch_size=7)
    r = cli.main(["inference", "--torch", "--read-alns", alns, "-m", pt, "-b", "8", "--targets-per-launch", "11", fq, out])
    assert r["failed_targets"] == 0 and r["records"] > 0
    # the expectation: the same windows and the module's own logits through the consensus oracle
    R = hostio.Reads(fq, min_len=4096)
    A = hostio.Alignments(alns, R)
    ctx = api.Context(None, 0, 4096, 8)
    R.upload(ctx)
    net = torch.jit.load(pt, map_location="cuda:0").eval()
    want = b""
    with torch.no_grad():
        for k0 in range(0, A.n_targets, 11):
            F = ctx.features_batch([A.target(k) for k in range(k0, min(k0 + 11, A.n_targets))], device=True, batches=True)
            bl = [net(b.to(torch.int32), cli.quals_normalised(q), torch.from_numpy(n).cuda(), [torch.from_numpy(i).cuda() for i in idx])[1]
                  for _, b, q, n, idx in F.batches()]
            flat = torch.cat(bl).cpu().numpy() if bl else np.zeros((0, 5), np.float32)
            bases = F.bases.cpu().numpy()
            reads = []
            for k in range(len(F.rids)):
                wins = []
                for w in range(int(F.win_off[k]), int(F.win_off[k + 1])):
                    x = F.window(w)
                    wins.append((bases[F.row_off[w]:F.row_off[w + 1]], x["n_alns"], x["supported"], flat[F.sup_off[w]:F.sup_off[w + 1]]))
                reads.append(wins)
            for k, segs in enumerate(consensus_oracle.consensus_windows(reads)):
                if segs:
                    rid = F.rids[k]
                    want += api.fasta_records(R.ids[rid], R.descriptions[rid], segs)
    assert open(out, "rb").read() == want


# ------------------------------------------------------------------------------------------ 5. errors and isolation
def test_failed_targets_fail_alone():
    rs = helpers.small_readset(n_reads=24, mean_len=9000, seed=3)
    targets = targets_of(rs, 12)
    ctx = api.Context(None, 0, 4096, 64)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    clean = ctx.features_batch([(t, overlaps(rs, t)) for t in targets], batches=True)
    clean_w = {t: [clean.window(w) for w in range(int(clean.win_off[k]), int(clean.win_off[k + 1]))] for k, t in enumerate(targets)}
    clean_b = [(list(x[0]), x[1].copy()) for x in clean.batches()]
    bad_cig = np.frombuffer(b"999999M", dtype=np.uint8).copy()
    v1, v2 = targets[2], targets[5]
    o1 = overlaps(rs, v1)
    i = int(np.argmax(o1["tend"].astype(np.int64) - o1["tstart"]))  # the longest alignment: it contributes windows, so its CIGAR is read
    o1["cigar"][i] = bad_cig.ctypes.data
    o1["cigar_len"][i] = len(bad_cig)
    o2 = overlaps(rs, v2)
    o2["tend"][0], o2["tstart"][0] = o2["tstart"][0], o2["tend"][0]  # inverted target range
    F = ctx.features_batch([(t, o1 if t == v1 else o2 if t == v2 else overlaps(rs, t)) for t in targets], batches=True)
    assert "target" in api.load_library().hb_last_error(ctx._h).decode()
    for k, t in enumerate(targets):
        wins = [F.window(w) for w in range(int(F.win_off[k]), int(F.win_off[k + 1]))]
        assert len(wins) == len(clean_w[t])
        if t in (v1, v2):
            assert F.status[k] == HB_ERR_INPUT
            assert all(w["L"] == 0 and len(w["supported"]) == 0 and len(w["ids"]) == 0 for w in wins)
            assert not any(int(F.win_off[k]) <= x < int(F.win_off[k + 1]) for x in F.batch_win)
        else:
            assert F.status[k] == 0
            for w, c in zip(wins, clean_w[t]):
                same_window(w, c)
                assert np.array_equal(w["ids"], c["ids"])
    kept = [b for b in clean_b if not any(clean.rids[int(np.searchsorted(clean.win_off, x, side="right")) - 1] in (v1, v2) for x in b[0])]
    got = list(F.batches())
    assert len(got) == len(kept) and all(np.array_equal(g[1], c[1]) for g, c in zip(got, kept))


def test_call_errors_and_a_context_without_weights():
    from herro_b200.api import HerroError
    rs = helpers.small_readset(n_reads=12, mean_len=9000, seed=3)
    targets = targets_of(rs, 4)
    ctx = api.Context(None, 0, 4096, 64)
    with pytest.raises(HerroError) as ei:
        ctx.features_batch([(targets[0], overlaps(rs, targets[0]))])
    assert ei.value.code == HB_ERR_STATE  # no hb_upload_reads
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    for bad in ([(rs.n, overlaps(rs, targets[0]))], [(targets[1], overlaps(rs, targets[0]))]):  # rid out of range, tid != rid
        with pytest.raises(HerroError) as ei:
            ctx.features_batch(bad)
        assert ei.value.code == HB_ERR_ARG
    o = overlaps(rs, targets[0])
    o["strand"][0] = 2
    with pytest.raises(HerroError) as ei:
        ctx.features_batch([(targets[0], o)])
    assert ei.value.code == HB_ERR_ARG
    # a stale ticket, and pointers that do not match the flag
    L = api.load_library()
    ctx.features_batch([(t, overlaps(rs, t)) for t in targets])
    old = api.HbFeaturesShape()
    old.ticket = ctx.last_features_shape.ticket
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in targets])
    sh = ctx.last_features_shape
    rows = np.zeros(sh.n_windows, np.uint32)
    out = api.HbFeaturesOut(api.C.sizeof(api.HbFeaturesOut))
    out.rows = rows.ctypes.data
    assert L.hb_features_fetch(ctx._h, api.C.byref(old), api.C.byref(out), 0, None) == HB_ERR_STATE
    assert L.hb_features_fetch(ctx._h, api.C.byref(sh), api.C.byref(out), 0, None) == 0 and np.array_equal(rows, F.rows)
    host = np.zeros((sh.n_rows, 31), np.uint8)
    dev = torch.zeros((sh.n_rows, 31), dtype=torch.uint8, device="cuda:0")
    for ptr, flags in ((host.ctypes.data, api.HB_FEAT_DEVICE_PTRS), (dev.data_ptr(), 0)):
        o = api.HbFeaturesOut(api.C.sizeof(api.HbFeaturesOut))
        o.bases = ptr
        assert L.hb_features_fetch(ctx._h, api.C.byref(sh), api.C.byref(o), flags, None) == HB_ERR_ARG
    o = api.HbFeaturesOut(api.C.sizeof(api.HbFeaturesOut))
    o.rows = dev.data_ptr()  # metadata is host memory whatever the flag
    assert L.hb_features_fetch(ctx._h, api.C.byref(sh), api.C.byref(o), api.HB_FEAT_DEVICE_PTRS, None) == HB_ERR_ARG
    o = api.HbFeaturesOut(api.C.sizeof(api.HbFeaturesOut) - 8)
    assert L.hb_features_fetch(ctx._h, api.C.byref(sh), api.C.byref(o), 0, None) == HB_ERR_ARG
    # the context without weights refuses what needs a model, and stays usable
    with pytest.raises(HerroError) as ei:
        ctx.submit_alignments(targets[0], overlaps(rs, targets[0]))
    assert ei.value.code == HB_ERR_STATE
    with pytest.raises(HerroError) as ei:
        ctx.forward_batch(np.zeros((1, 4, 31), np.uint8), np.zeros((1, 4, 31), np.uint8), [1], [[0]])
    assert ei.value.code == HB_ERR_STATE
    with pytest.raises(HerroError) as ei:
        ctx.flush()
    assert ei.value.code == HB_ERR_STATE
    again = ctx.features_batch([(t, overlaps(rs, t)) for t in targets])
    assert np.array_equal(again.bases, F.bases) and np.array_equal(again.ids, F.ids)


def test_beside_a_running_pipeline_and_in_the_steady_state():
    """A features call in another thread while the pipeline flushes leaves the pipeline's segments, debug taps and replayable launch
    as a run alone leaves them; repeated calls of one shape allocate nothing."""
    rs = helpers.small_readset(n_reads=40, mean_len=9000, seed=5)
    targets = targets_of(rs, 40)
    path = helpers.model_path(seed=3)
    alone = helpers.run_product(rs, path, 4096, 64, targets=targets, keep_debug=True)
    ctx = api.Context(path, 0, 4096, 64, launch_targets=1 << 20, keep_debug=True)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    want_F = ctx.features_batch([(t, overlaps(rs, t)) for t in targets[::-1]], batches=True)
    got_F = []
    for t in targets:
        ctx.submit_alignments(t, overlaps(rs, t))
    th = threading.Thread(target=lambda: got_F.extend(ctx.features_batch([(t, overlaps(rs, t)) for t in targets[::-1]], batches=True)
                                                      for _ in range(3)))
    th.start()
    ctx.flush()
    th.join()
    segs = {r.rid: r.segments or None for r in ctx.drain()}
    assert segs == alone["segments"]
    ctx.replay_last_launch(2)
    for (t, w), d in alone["windows"].items():
        g = ctx.debug_window(t, w)
        same_window(g, d)
        assert np.array_equal(g["bases_logits"], d["bases_logits"])
    for F in got_F:
        for k in ("bases", "quals", "supported", "indices", "ids", "batch_bases", "batch_quals", "batch_win"):
            assert np.array_equal(getattr(F, k), getattr(want_F, k)), k
    for device in (False, True):
        ctx.features_batch([(t, overlaps(rs, t)) for t in targets], device=device, batches=True)
        ctx.reset_stats()
        ctx.features_batch([(t, overlaps(rs, t)) for t in targets], device=device, batches=True)
        s = ctx.stats()
        assert s["host_allocs"] == 0, s["host_allocs"]
        assert s["targets"] == 0 and s["windows"] == 0 and s["corrected_bases"] == 0
        assert s["ms_features"] > 0 and s["n_kernel"]["lists"] >= 3 and s["d2h_bytes"] > 0
