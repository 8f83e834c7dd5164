"""The barrier protocol of conv_c31_kernel on the CPU model of tests/c31_model.py: under random interleavings of the two
consumer warpgroups, the weight refills, the TMA loads and the TMA stores' reads, every read sees the data it expects,
no load lands in a buffer something still reads, and nothing deadlocks - at the kernel's ring depths for Cm = 64 /
128 / 256, at shallower rings and over 1-4 tiles per CTA.  Each rule the kernel states is shown to matter: with one
arrival per empty barrier, with a residual load that skips the bulk read wait, or with one issued before the wait_group
that ends the previous conv1, the model fails.  Also checks the compiler's report: no conv_c31_kernel instantiation
spills."""
import os
import re

import pytest

import c31_model as M

SEEDS = 30


@pytest.mark.parametrize("cm", [64, 128, 256])
@pytest.mark.parametrize("tiles", [1, 2, 3, 4])
def test_kernel_rings_read_the_expected_data(cm, tiles):
    for seed in range(SEEDS):
        cfg = M.kernel_config(cm, tiles)
        assert M.simulate(cfg, seed) == "ok", (cfg, seed)


@pytest.mark.parametrize("stages", [2, 3, 4, 5])
def test_shallow_rings_read_the_expected_data(stages):
    for cm in (64, 128, 256):
        for seed in range(SEEDS):
            cfg = M.kernel_config(cm, 3, stages=stages)
            assert M.simulate(cfg, seed) == "ok", (cfg, seed)


def _results(**bug):
    return [M.simulate(M.kernel_config(cm, 3, **bug), seed) for cm in (64, 128, 256) for seed in range(SEEDS)]


def test_one_arrival_per_empty_barrier_fails():
    """Protocol 1: a slot is refilled only after BOTH warpgroups have released it; with one arrival the lagging one
    reads the next fill (or the ring stalls)."""
    rs = _results(empty_count=1)
    assert any(r.startswith("expected fill") for r in rs), set(rs)


def test_residual_load_without_the_bulk_read_wait_races_the_store():
    """Protocol 2: the residual of chunk q + 1 lands in the buffer that chunk q - 1's store may still read."""
    rs = _results(skip_wait_read=True)
    assert any(r.startswith("race") and "store" in r for r in rs), set(rs)


def test_residual_load_before_wait_group_0_races_conv1():
    """Protocol 2: conv1 of chunk q - 1 reads its staging buffer until the wait_group 0 of chunk q."""
    rs = _results(early_res=True)
    assert any(r.startswith("race") and "conv1" in r for r in rs), set(rs)


LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deep-image-retrieval_b200", "build",
                   "conv.cu.log")


def test_no_c31_instantiation_spills():
    """ptxas -v of the last build reports 0 spill bytes for every conv_c31_kernel instantiation (Cm 64 / 128 / 256,
    dense and ragged)."""
    if not os.path.exists(LOG):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(LOG).read()
    blocks = re.findall(r"Compiling entry function '(_ZN4dirb15conv_c31_kernel\w+)'.*?\n(.*?)\nptxas info\s+: Used (\d+) registers",
                        text, re.S)
    assert len(blocks) == 6, [b[0] for b in blocks]
    for name, stats, regs in blocks:
        assert "0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
