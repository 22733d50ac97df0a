"""Steady state of a launch context (GPU): after warm-up, running the same workload again allocates nothing."""
import pytest

import helpers

pytestmark = pytest.mark.gpu


def test_warm_context_allocates_nothing():
    """DESIGN.md §2: once a context with several lanes has run its workload twice, every lane has been pre-sized to the
    largest regions any lane needed and the staging pool is pinned, so running it a third time makes no allocation."""
    from herro_b200 import Context
    rs = helpers.small_readset(n_reads=30, mean_len=7000, seed=12)
    model = helpers.model_path(seed=3)
    ctx = Context(model, 0, 4096, 64, launch_targets=4)
    ctx.upload_reads(rs.seqs, rs.quals, rs.off)

    def run():
        for t in range(rs.n):
            a0, a1 = int(rs.aln_off[t]), int(rs.aln_off[t + 1])
            if a1 > a0:
                ctx.submit_alignments(t, Context.make_overlaps(rs.ovl9[a0:a1], rs.cigars, rs.cig_off[a0:a1 + 1]))
        ctx.flush()
        return {r.rid: r.segments for r in ctx.drain()}

    first = run()
    run()
    ctx.reset_stats()
    assert run() == first
    st = ctx.stats()
    assert st["device_launches"] >= 3
    assert st["host_allocs"] == 0, st["host_allocs"]
