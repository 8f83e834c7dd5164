"""CPU checks of the test-only harness of csrc/block.cuh (tests/block_harness.cu): it cross-compiles for sm_90a into
libdirb200_blocktest.so, exports every launcher tests/test_gpu_block.py calls, builds without spills, and calls every
primitive the header declares, so that a primitive added later without a direct test fails here."""
import ctypes
import importlib.util
import os
import re

import pytest

from conftest import REPO

HERE = os.path.join(REPO, "deep-image-retrieval_b200")
HEADER = os.path.join(HERE, "csrc", "block.cuh")
HARNESS = os.path.join(REPO, "tests", "block_harness.cu")
GPU_TEST = os.path.join(REPO, "tests", "test_gpu_block.py")


@pytest.fixture(scope="module")
def built():
    """build_ext.build() (a no-op when the tree is up to date) -> (path of the harness library, its nvcc log)."""
    spec = importlib.util.spec_from_file_location("dirb200_build_ext", os.path.join(HERE, "build_ext.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()
    with open(os.path.join(HERE, "build", "block_harness.cu.log")) as f:
        return mod.BLOCKTEST_LIB, f.read()


def _declared(src):
    """Names of the functions and function templates a header declares at namespace scope."""
    return set(re.findall(r"^(?:template <[^\n]*>\n)?__device__[^(\n]*?\b(\w+)\(", src, flags=re.M))


def test_harness_exports_every_launcher_the_gpu_test_calls(built):
    path, log = built
    assert "sm_90a" in log
    import test_gpu_block as T                     # its calls go through T.SIGNATURES, which it checks on every call
    called = set(T.SIGNATURES)
    named = set(re.findall(r"\b(dirb_blocktest_\w+)", open(GPU_TEST).read()))
    assert {n for n in named if not n.endswith("_")} <= called and len(called) == 18
    so = ctypes.CDLL(path)
    missing = [n for n in sorted(called) if not hasattr(so, n)]
    assert not missing, missing


def test_harness_kernels_do_not_spill(built):
    _, log = built
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'.*?\n.*?\n(.*?)\n", log)
    assert len(blocks) >= 39                           # 25 sorts, 3 scans, 3 warp scans, 4 selects, 2 ranks, 2 maps
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)


def test_harness_calls_every_primitive_of_the_header():
    declared = _declared(open(HEADER).read())
    assert {"ranks_before", "f2key", "key2f", "fkey", "block_bitonic_sort", "warp_scan", "block_scan",
            "block_radix_kth", "rank_in_run"} <= declared
    harness = open(HARNESS).read()
    harness = re.sub(r"//[^\n]*", "", harness)        # calls, not mentions in comments
    uncalled = [n for n in sorted(declared) if not re.search(r"\b%s\s*(<[^;()]*>)?\s*\(" % n, harness)]
    assert not uncalled, uncalled
    # both forms of the overloaded primitives: the key form of ranks_before and the keys-only sort
    assert re.search(r"ranks_before\(fkey\(", harness)
    assert re.search(r"block_bitonic_sort<NT>\(key, P, ", harness) and re.search(r"block_bitonic_sort<NT>\(key, val, P, ", harness)


def test_declaration_scan_sees_a_new_primitive():
    extra = open(HEADER).read() + "\ntemplate <class T>\n__device__ __forceinline__ T block_new_thing(T v) { return v; }\n"
    assert "block_new_thing" in _declared(extra)
