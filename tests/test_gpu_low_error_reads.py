"""The features stage on low-error reads, through the C ABI: CIGAR ops that span whole windows (one op per overlap-window,
six-digit op lengths, every window boundary inside one op), rankings decided entirely by the tie rules, every window's ranked ids,
and launches without a single supported position.  The hand-built sets carry the answers derived in test_low_error_oracle_cpu.py;
every set is also compared with the oracle.  Each test asserts the preconditions that make it reach its path."""
import os
import re

import numpy as np
import pytest

import helpers
from herro_b200 import api
from oracle import pyoracle as po
from test_low_error_oracle_cpu import (N_COPIES, SNP_POS, SNP_QIDS, W as HAND_W, build_groups, full_copies, op_lengths, random_bases,
                                       random_quals)
from tools import synth

pytestmark = pytest.mark.gpu
LOGITS_TOL = 1e-3
PATHS = ("device-windowing", "host-windowing", "submit-target")


# ------------------------------------------------------------------------------------------ plumbing
def overlaps(rs, t):
    a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
    return api.Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1])


def targets_of(rs):
    return [t for t in range(rs.n) if rs.aln_off[t + 1] > rs.aln_off[t]]


def n_windows(rs, t, W):
    return (int(rs.off[t + 1] - rs.off[t]) + W - 1) // W


def run_path(monkeypatch, path, rs, W, b, targets=None):
    """helpers.run_product through one submission path: hb_submit_alignments with the device windowing, the same call with the
    host windowing (HERRO_B200_HOST_WINDOWING), or hb_submit_target with the oracle's overlap-windows."""
    if path == "host-windowing":
        monkeypatch.setenv("HERRO_B200_HOST_WINDOWING", "1")
    try:
        return helpers.run_product(rs, helpers.model_path(seed=3), W, b, targets=targets, keep_debug=True,
                                   use_submit_target=path == "submit-target")
    finally:
        monkeypatch.delenv("HERRO_B200_HOST_WINDOWING", raising=False)


def pipeline_ids(ctx, rs, targets, W, out_dir):
    """The ranked ids of every window of the most recent launch, from its `herro features` ids.txt files (hb_dump_features)."""
    index = {n: i for i, n in enumerate(rs.ids)}
    ids = {}
    for t in targets:
        ctx.dump_features(t, str(out_dir), rs.ids)
        for w in range(n_windows(rs, t, W)):
            names = open(os.path.join(str(out_dir), rs.ids[t], f"{w}.ids.txt"), "rb").read().split(b"\n")[:-1]
            ids[(t, w)] = [index[n.decode()] for n in names]
    return ids


def features_windows(F, targets):
    return {(t, w): F.window(int(F.win_off[k]) + w) for k, t in enumerate(targets) for w in range(int(F.n_windows[k]))}


def same_as_oracle(win, w: po.Window):
    assert win["L"] == w.bases.shape[0] and win["n_alns"] == w.n_alns
    assert np.array_equal(win["bases"], w.bases) and np.array_equal(win["quals"], w.quals)
    assert np.array_equal(win["supported"], w.supported.reshape(-1, 2)) and np.array_equal(win["sup_rows"], w.sup_rows)


def check_ids(ids, ora_windows):
    """Every window's ranked ids (all n overlaps, not only the 30 kept) equal the oracle's Window.qids."""
    assert set(ids) == set(ora_windows)
    for key, w in ora_windows.items():
        assert list(ids[key]) == [int(q) for q in w.qids], key


def interior_single_op_windows(rs, targets, W):
    """Overlap-windows of interior windows whose CIGAR slice is one op (k_tokenize's nops == 1 branch), from hb_extract_windows."""
    n = 0
    for t in targets:
        nw = n_windows(rs, t, W)
        cig = rs.cigars[int(rs.cig_off[int(rs.aln_off[t])]):int(rs.cig_off[int(rs.aln_off[t + 1])])]
        base = int(rs.cig_off[int(rs.aln_off[t])])
        for o in api.extract_windows(overlaps(rs, t), W, nw):
            if not 0 < int(o["window_idx"]) < nw - 1:
                continue
            a0 = int(rs.cig_off[int(rs.aln_off[t]) + int(o["overlap_idx"])]) - base
            sl = cig[a0 + int(o["cigar_start_idx"]):a0 + int(o["cigar_end_idx"])].tobytes()
            n += len(re.findall(rb"[MID]", sl)) == 1
    return n


# ------------------------------------------------------------------------------------------ 1. the hand-built sets
def hand_expectations(rs, with_snp):
    """The answers of test_low_error_oracle_cpu.py, as checks on one run's windows and ranked ids."""
    want_ids = [q for q in range(1, N_COPIES + 1) if q not in SNP_QIDS] + SNP_QIDS if with_snp else list(range(1, N_COPIES + 1))

    def check(windows, ids):
        assert sorted(windows) == [(0, w) for w in range(6)]
        for (_, wid), win in windows.items():
            assert win["n_alns"] == 30
            assert list(ids[(0, wid)]) == want_ids, wid
            sup = [[SNP_POS % HAND_W, 0]] if with_snp and wid == SNP_POS // HAND_W else []
            assert win["supported"].reshape(-1, 2).tolist() == sup and win["sup_rows"].tolist() == [s[0] for s in sup]
            assert bytes(win["bases"][:, 0]) == bytes(b"ACGT".index(c) for c in rs.seq(0)[wid * HAND_W:(wid + 1) * HAND_W])
    return check


@pytest.mark.parametrize("with_snp", [False, True], ids=["exact-copies", "ten-snp-copies"])
def test_hand_built_sets_through_every_path(monkeypatch, tmp_path, with_snp):
    """35 exact copies (every window ties, nothing supported, the record is the target) and 25 exact + 10 SNP copies (one
    supported position, exact copies ranked first): hand-derived ids, n_alns, SupportedPos and records, and the oracle's windows,
    logits and records, through hb_submit_alignments (device and host windowing), hb_submit_target and hb_features_batch."""
    rs, _ = full_copies(snp_qids=SNP_QIDS if with_snp else (), snp_pos=SNP_POS)
    ora = helpers.run_oracle(rs, helpers.model_path(seed=3), HAND_W, 4)
    check = hand_expectations(rs, with_snp)
    if not with_snp:
        assert ora["segments"][0] == [rs.seq(0)] and not ora["logits"]
    for path in PATHS:
        got = run_path(monkeypatch, path, rs, HAND_W, 4)
        helpers.compare(ora, got, LOGITS_TOL)
        check(got["windows"], pipeline_ids(got["ctx"], rs, [0], HAND_W, tmp_path / path))
        assert got["stats"]["supported"] == (1 if with_snp else 0)
        if not with_snp:
            assert got["segments"][0] == [rs.seq(0)]
        if path == "device-windowing":
            F = got["ctx"].features_batch([(0, overlaps(rs, 0))], batches=True)
            fw = features_windows(F, [0])
            check(fw, {k: v["ids"] for k, v in fw.items()})
            for key, w in ora["windows"].items():
                same_as_oracle(fw[key], w)
            assert len(list(F.batches())) == (1 if with_snp else 0)


# ------------------------------------------------------------------------------------------ 2. six-digit ops
@pytest.mark.parametrize("W", [4096, 8192])
def test_six_digit_ops(monkeypatch, W):
    """A 120 kb target and 34 full-length copies, ten with one substitution: every CIGAR is one six-digit M op, every window
    boundary lies inside it, and each overlap-window is a slice of that one op."""
    rs, _ = full_copies(tlen=120_000, n=34, seed=5, snp_qids=SNP_QIDS, snp_pos=61_234)
    assert (op_lengths(rs) >= 100_000).all() and len(op_lengths(rs)) == 34
    assert interior_single_op_windows(rs, [0], W) == 34 * (120_000 // W - 1)
    ora = helpers.run_oracle(rs, helpers.model_path(seed=3), W, 64)
    want_ids = [q for q in range(1, 35) if q not in SNP_QIDS] + SNP_QIDS
    for key, w in ora["windows"].items():
        assert list(w.qids) == want_ids and w.n_alns == 30
    assert sum(len(w.supported) for w in ora["windows"].values()) == 1
    for path in PATHS:
        got = run_path(monkeypatch, path, rs, W, 64)
        helpers.compare(ora, got, LOGITS_TOL)
    F = got["ctx"].features_batch([(0, overlaps(rs, 0))], batches=True)
    check_ids({k: v["ids"] for k, v in features_windows(F, [0]).items()}, ora["windows"])
    print(f"six-digit ops at W {W}: {len(op_lengths(rs))} ops of >= 100000 bases, "
          f"{interior_single_op_windows(rs, [0], W)} interior single-op overlap-windows")


# ------------------------------------------------------------------------------------------ 3. digit-position sweep
STEP = 22  # k_parse_cigars / k_tokenize<false>: lanes 10..31 are the 22 new bytes of a parse step, lanes 0..9 look back


def sweep_readset(tlen=120_000, seed=7):
    """One copy per (d, r), d = 1..6 digits, r = 0..21: its CIGAR is 10M 1I 5M 1D (a planted insertion of a random base and a
    deletion), 1M / 10M ops that shift the next op, a d-digit M op whose letter lies at a byte index = r (mod 22) past the first
    step, and an M op up to the end.  The copy is the target with the planted insertion and deletion applied."""
    rng = np.random.default_rng(seed)
    target, tqual = random_bases(rng, tlen), random_quals(rng, tlen)
    copies = []
    for d in range(1, 7):
        for r in range(STEP):
            ops = [(10, "M"), (1, "I"), (5, "M"), (1, "D")]
            L = next(L for L in range(STEP, 2 * STEP) if (L + d) % STEP == r)   # bytes before the d-digit op
            fill = L - 9
            if fill % 2:
                ops.append((10, "M"))
                fill -= 3
            ops += [(1, "M")] * (fill // 2)
            x = (10 ** (d - 1) if d > 1 else 1) + r % 9
            tspan = sum(n for n, k in ops if k != "I")
            ops += [(x, "M"), (tlen - tspan - x, "M")]
            cig = "".join(f"{n}{k}" for n, k in ops).encode()
            assert len(str(x)) == d and cig.index(b"%dM" % x, L) == L and (L + d) % STEP == r
            q, t = bytearray(), 0
            for n, k in ops:
                if k == "M":
                    q += target[t:t + n]
                    t += n
                elif k == "I":
                    q += random_bases(rng, 1)
                else:
                    t += n
            copies.append((bytes(q), random_quals(rng, len(q)), len(copies) % 2 == 1, 0, tlen, cig))
    return build_groups([(target, tqual, copies)])


def letter_lanes(cigar: bytes):
    """(digits, byte index mod 22) of every op letter of a CIGAR."""
    return {(len(m.group(1)), m.end(2) - 1) for m in re.finditer(rb"(\d+)([MID])", cigar)}


def test_digit_position_sweep(monkeypatch):
    """Op lengths of 1 to 6 digits whose letter ends on every lane 10..31 of a parse step, through k_parse_cigars
    (hb_submit_alignments) and k_tokenize<false> (hb_submit_target: window 0's slice starts at the CIGAR's first byte)."""
    rs = sweep_readset()
    seen = set()
    for a in range(len(rs.ovl9)):
        seen |= {(d, i % STEP) for d, i in letter_lanes(rs.cigar(a)) if i >= STEP}
    assert {(d, r) for d in range(1, 7) for r in range(STEP)} <= seen
    ora = helpers.run_oracle(rs, helpers.model_path(seed=3), 4096, 64)
    assert sum(len(w.supported) for w in ora["windows"].values()) > 0 and max(len(w.qids) for w in ora["windows"].values()) == 132
    for path in ("device-windowing", "submit-target"):
        got = run_path(monkeypatch, path, rs, 4096, 64)
        helpers.compare(ora, got, LOGITS_TOL)
    F = got["ctx"].features_batch([(0, overlaps(rs, 0))], batches=True)
    check_ids({k: v["ids"] for k, v in features_windows(F, [0]).items()}, ora["windows"])


# ------------------------------------------------------------------------------------------ 4. synthetic low-error sets
SYNTH = [(p, W, b) for p in ("exact", "q30") for W, b in ((1024, 4), (4096, 64), (8192, 64))]
N_TARGETS, N_FORWARD = 16, 3


def low_error_set(profile):
    return synth.generate(60, 30000, profile=profile, seed=61, coverage=40.0, min_ovl=2048, targets=(0, N_TARGETS))


@pytest.mark.parametrize("profile,W,b", SYNTH, ids=[f"{p}-W{W}-b{b}" for p, W, b in SYNTH])
def test_synthetic_low_error_sets(tmp_path, profile, W, b):
    """60 reads of 30 kb at 40x, the alignments of the first 16 targets: every window against the oracle (the torch forward on
    three targets), every window's ranked ids from hb_features_batch and from the `herro features` ids.txt files."""
    rs = low_error_set(profile)
    tg = targets_of(rs)
    assert len(tg) >= N_TARGETS - 1
    ops = op_lengths(rs)
    n_single = interior_single_op_windows(rs, tg, W)
    feat = helpers.run_oracle(rs, helpers.model_path(seed=3), W, b, targets=tg, with_forward=False)
    n_over_30 = sum(len(w.qids) > 30 for w in feat["windows"].values())
    print(f"{profile} W {W}: {int((ops >= 10000).sum())} ops >= 10000, {n_single} interior single-op overlap-windows, "
          f"{n_over_30} of {len(feat['windows'])} windows with > 30 ranked ids")
    assert n_over_30 > 0
    if profile == "exact":  # q30's indels come every ~2 kb: its ops reach thousands of bases, not 10 000, and none spans a whole 8 kb window
        assert (ops >= 10000).any() and n_single > 0
    else:
        assert (ops >= 4096).any() and (n_single > 0 or W == 8192)
    ora = helpers.run_oracle(rs, helpers.model_path(seed=3), W, b, targets=tg[:N_FORWARD])
    assert ora["logits"]
    got = helpers.run_product(rs, helpers.model_path(seed=3), W, b, targets=tg, keep_debug=True)
    helpers.compare({"windows": feat["windows"], "logits": ora["logits"], "segments": {}}, {**got, "segments": {}}, LOGITS_TOL)
    for t in tg[:N_FORWARD]:
        assert got["segments"][t] == ora["segments"][t]
    check_ids(pipeline_ids(got["ctx"], rs, tg, W, tmp_path), feat["windows"])
    F = got["ctx"].features_batch([(t, overlaps(rs, t)) for t in tg], batches=True)
    fw = features_windows(F, tg)
    check_ids({k: v["ids"] for k, v in fw.items()}, feat["windows"])
    for key, w in feat["windows"].items():
        same_as_oracle(fw[key], w)


def test_synthetic_low_error_set_on_a_host_read_store():
    """The exact profile at W 4096 through hb_features_batch on a read store in pinned host memory: the oracle's windows and ids."""
    rs = low_error_set("exact")
    tg = targets_of(rs)
    feat = helpers.run_oracle(rs, None, 4096, 64, targets=tg, with_forward=False)
    store = api.ReadStore(rs.seqs, rs.quals, rs.off)
    ctx = api.Context(None, 0, 4096, 64)
    ctx.attach_read_store(store)
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in tg], batches=True)
    fw = features_windows(F, tg)
    check_ids({k: v["ids"] for k, v in fw.items()}, feat["windows"])
    for key, w in feat["windows"].items():
        same_as_oracle(fw[key], w)


# ------------------------------------------------------------------------------------------ 5. ranked ids on noisy shapes
NOISY = {
    # the 70x set of test_gpu_edge_cases.py::test_more_overlaps_than_the_model_takes
    "70x": (lambda: helpers.small_readset(n_reads=60, mean_len=5000, seed=25, coverage=70.0, min_ovl=1500), 1024, 16, 30),
    # the set of test_gpu_shapes.py::test_more_than_1024_overlaps_in_a_window (sort keys in HBM)
    "over-1024": (lambda: synth.generate(2200, 5000, profile="r10", seed=52, coverage=1000.0, min_ovl=1100, sd_frac=0.05,
                                         targets=(0, 3)), 1024, 16, 1024),
}


@pytest.mark.parametrize("name", list(NOISY))
def test_ranked_ids_on_noisy_sets(name):
    """All n ranked ids of every window, beyond the 30 kept columns, equal the oracle's Window.qids."""
    make, W, b, more_than = NOISY[name]
    rs = make()
    tg = targets_of(rs)
    feat = helpers.run_oracle(rs, None, W, b, targets=tg, with_forward=False)
    assert max(len(w.qids) for w in feat["windows"].values()) > more_than
    ctx = api.Context(None, 0, W, b)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in tg], batches=True)
    check_ids({k: v["ids"] for k, v in features_windows(F, tg).items()}, feat["windows"])


# ------------------------------------------------------------------------------------------ 6. a launch with no supported position
def test_launch_without_a_supported_position():
    """Exact copies of four random targets (no het site anywhere): no window has a supported position, so the launch runs no
    forward pass, collates no reference batch, and every record is its target read."""
    rng = np.random.default_rng(9)
    groups = []
    for k in range(4):
        n = 6000 + 1500 * k
        target = random_bases(rng, n)
        groups.append((target, random_quals(rng, n), [(target, random_quals(rng, n), c % 2 == 1, 0, n, f"{n}M".encode())
                                                      for c in range(32)]))
    rs = build_groups(groups)
    tg = targets_of(rs)
    assert len(tg) == 4
    got = helpers.run_product(rs, helpers.model_path(seed=3), 1024, 8, keep_debug=True)
    s = got["stats"]
    assert s["supported"] == 0 and s["n_kernel"]["heads"] == 0 and s["device_launches"] == 1
    assert got["segments"] == {t: [rs.seq(t)] for t in tg}
    ctx = got["ctx"]
    F = ctx.features_batch([(t, overlaps(rs, t)) for t in tg], batches=True)
    assert list(F.status) == [0] * 4 and len(F.batch_B) == 0 and list(F.batches()) == [] and int(F.n_sup.sum()) == 0
    for (t, w), win in features_windows(F, tg).items():
        d = got["windows"][(t, w)]
        assert win["L"] == d["L"] and win["n_alns"] == d["n_alns"] == 30
        assert np.array_equal(win["bases"], d["bases"]) and np.array_equal(win["quals"], d["quals"])
        assert list(win["ids"]) == list(range(t + 1, t + 33))
    assert ctx.consensus_batch(*F.consensus_args([])) == [[rs.seq(t)] for t in tg]
    print("launch without a supported position: 4 targets, 0 supported, 0 head kernels, 0 batches")
