"""The ping-pong consumer protocol of conv_pers_kernel on the CPU model of tests/pingpong_model.py: under random
interleavings of the producer, the TMA copies and the four warps of each consumer warpgroup, every warp reads exactly
the fill it expects and nothing deadlocks, over ring depths, k-iteration counts (below, at and above the ring depth;
HALO's 9 * cin_blocks with its patch ring) and 1-7 tiles per CTA.  Each invariant the kernel states is also shown to
matter: without the mainloop handover, with a handover that only the leader warp arrives on, with the cooperative
mode's two arrivals per fill, or with one staging set for both warpgroups the model fails.  Also checks the compiler's
report: no convolution instantiation spills."""
import os
import re

import pytest

import pingpong_model as M

SEEDS = 8
TILES = range(1, 8)


def _k_iters(stages):
    return sorted({1, 2, 3, stages - 1, stages, stages + 1})


@pytest.mark.parametrize("stages", [5, 6, 7, 8])
@pytest.mark.parametrize("has_res", [True, False], ids=["res", "nores"])
def test_flat_ring_reads_the_expected_fills(stages, has_res):
    for k in _k_iters(stages):
        for tiles in TILES:
            for seed in range(SEEDS):
                cfg = M.Config(stages, k, tiles, has_res=has_res)
                assert M.simulate(cfg, seed) == "ok", (cfg, seed)


@pytest.mark.parametrize("stages", [5, 6, 7, 8])
@pytest.mark.parametrize("cin_blocks", [1, 2, 4])
def test_halo_rings_read_the_expected_fills(stages, cin_blocks):
    for tiles in TILES:
        for seed in range(SEEDS):
            cfg = M.Config(stages, 9 * cin_blocks, tiles, halo=True)
            assert M.simulate(cfg, seed) == "ok", (cfg, seed)


def test_without_the_mainloop_handover_a_consumer_reads_a_stale_slot():
    """Invariant 1: with mma_done removed, some interleavings pass a full-barrier wait on the previous phase."""
    failures = []
    for stages in (5, 6, 7, 8):
        for k in _k_iters(stages):
            for tiles in range(2, 8):
                for seed in range(SEEDS):
                    r = M.simulate(M.Config(stages, k, tiles, order=False), seed)
                    if r != "ok":
                        failures.append(r)
    assert failures
    assert any("expected" in r for r in failures), "no stale read among %d failures" % len(failures)


def test_a_handover_from_the_leader_warp_alone_deadlocks_at_one_k_iteration():
    """Invariant 1, per warp: with mma_done at count 1 and only warp 0 arriving, a tile of one k-iteration lets the
    leader hand over while a sibling warp has not yet passed its own mma_done wait; the partner can then complete the
    barrier twice and the sibling waits on a parity that never returns.  With every warp arriving it cannot."""
    results = [M.simulate(M.Config(5, 1, tiles, handover_warps=1), seed) for tiles in range(3, 8) for seed in range(40)]
    assert "deadlock" in results
    assert all(M.simulate(M.Config(5, 1, tiles), seed) == "ok" for tiles in range(3, 8) for seed in range(40))


@pytest.mark.parametrize("halo", [False, True])
def test_two_arrivals_per_fill_deadlock(halo):
    """Invariant 3: only the warpgroup that reads a fill hands it back; an empty count of 2 stalls the producer as soon
    as the ring wraps."""
    stages = 5
    k = 9 if halo else stages + 1
    for seed in range(SEEDS):
        assert M.simulate(M.Config(stages, k, 2, halo=halo, empty_count=2), seed) == "deadlock"


def test_shared_staging_fails():
    """Invariant 4: one staging set and residual barrier for both warpgroups breaks the epilogue."""
    results = [M.simulate(M.Config(5, 3, 4, shared_staging=True), seed) for seed in range(SEEDS)]
    assert all(r != "ok" for r in results), results


def test_odd_tile_counts_leave_an_unmatched_handover_harmlessly():
    """Invariant 5: with an odd tile count warpgroup 0 takes one tile more; its last mma_done arrival has no waiter."""
    for tiles in (1, 3, 5, 7):
        sim = M.Sim(M.Config(6, 4, tiles), seed=tiles)
        assert sim.run() == "ok"
        assert sim.mma_done[0].phase == (tiles + 1) // 2 and sim.mma_done[1].phase == tiles // 2


def test_slot_counters_follow_the_tile_index():
    """Invariant 2: warpgroup w's j-th tile is CTA-local tile i = 2j + w and starts at fill i * k_iters."""
    cfg = M.Config(7, 5, 6)
    sim = M.Sim(cfg, seed=1)
    assert sim.run() == "ok"
    for wg in (0, 1):
        for wp in range(M.WARPS):
            ring = [g for w, p, kind, g in sim.reads if w == wg and p == wp and kind == "ring"]
            assert ring == [i * cfg.k_iters + it for i in range(wg, cfg.tiles, 2) for it in range(cfg.k_iters)]


LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deep-image-retrieval_b200", "build",
                   "conv.cu.log")


def test_no_convolution_instantiation_spills():
    """Invariant 6: ptxas -v of the last build reports 0 spill bytes for every conv_pers_kernel instantiation, and the
    ping-pong ones keep the 168-register launch allocation that setmaxnreg redistributes."""
    if not os.path.exists(LOG):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(LOG).read()
    blocks = re.findall(r"Compiling entry function '(_ZN4dirb16conv_pers_kernel\w+)'.*?\n(.*?)\nptxas info\s+: Used (\d+) registers",
                        text, re.S)
    assert len(blocks) >= 16, "expected every dense / ragged, flat / HALO, BN 64 / 128, cooperative / ping-pong kernel"
    for name, stats, regs in blocks:
        assert "0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
        if name.endswith("ELb1EEEv14CUtensorMap_stS1_S1_S1_NS_14ConvPersParamsE"):
            assert int(regs) == 168, (name, regs)
