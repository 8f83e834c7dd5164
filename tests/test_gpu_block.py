"""The block primitives of csrc/block.cuh, called directly from the test-only kernels of tests/block_harness.cu and
compared bit for bit with the numpy model of tests/block_model.py: the bitonic sort (with the barrier it ends with),
block and warp scans, the radix select, the rank of an entry in a run, and the order-preserving key maps.  The cases
cover every instantiation the retrieval kernels use, the block sizes around them, and the inputs where such code goes
wrong: ties, -0 against +0, padding, stale entries past a run's end, keys that share all but one byte."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import block_model as M
from conftest import REPO

pytestmark = pytest.mark.gpu

HERE = os.path.join(REPO, "deep-image-retrieval_b200")
LIB_PATH = os.path.join(HERE, "libdirb200_blocktest.so")

_P, _I, _L, _U = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint32
SIGNATURES = {
    "dirb_blocktest_sort_f64_i32": [_I, _P, _P, _I, _I, _I, _P, _P],
    "dirb_blocktest_sort_f64_i64": [_I, _P, _P, _I, _I, _I, _P, _P],
    "dirb_blocktest_sort_i32_f64": [_I, _P, _P, _I, _I, _I, _P, _P],
    "dirb_blocktest_sort_u64": [_I, _P, _I, _I, _I, _P],
    "dirb_blocktest_sort_u32": [_I, _P, _I, _I, _I, _P],
    "dirb_blocktest_scan_i32": [_I, _P, _P, _P, _I],
    "dirb_blocktest_scan_i64": [_I, _P, _P, _P, _I],
    "dirb_blocktest_scan_u64": [_I, _P, _P, _P, _I],
    "dirb_blocktest_warp_scan_i32": [_P, _P, _L],
    "dirb_blocktest_warp_scan_i64": [_P, _P, _L],
    "dirb_blocktest_warp_scan_u64": [_P, _P, _L],
    "dirb_blocktest_kth_u32": [_I, _P, _I, _P, _P, _I, _P],
    "dirb_blocktest_kth_u32_n64": [_I, _P, _L, _P, _P, _I, _P],
    "dirb_blocktest_kth_u64": [_I, _P, _L, _P, _P, _I, _P],
    "dirb_blocktest_kth_f32": [_I, _P, _I, _P, _P, _I, _P],
    "dirb_blocktest_rank": [_P, _P, _I, _P, _P, _I, _I, _P],
    "dirb_blocktest_key_sweep": [_U, _U, _P],
    "dirb_blocktest_elementwise": [_P] * 11 + [_I],
}


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB_PATH):
        spec = importlib.util.spec_from_file_location("dirb200_build_ext", os.path.join(HERE, "build_ext.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build()
    so = ctypes.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
        getattr(so, name).argtypes = args
        getattr(so, name).restype = ctypes.c_int

    def call(name, *args):
        assert name in SIGNATURES, name
        conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
        assert getattr(so, name)(*conv) == 0, name
        torch.cuda.synchronize()
    return call


def dev(a):
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "u" and a.dtype.itemsize > 1:          # moved as the signed type of the same width
        a = a.view({8: np.int64, 4: np.int32}[a.dtype.itemsize])
    return torch.from_numpy(a).cuda()


def host(t, dtype):
    """A device tensor's bytes as a numpy array of dtype (torch has no uint32 / uint64 arithmetic to rely on)."""
    return t.cpu().numpy().view(dtype)


def distinct(r, hi, n):
    """n distinct integers from [0, hi), in random order."""
    v = np.unique(r.randint(0, hi, n + 64, dtype=np.int64))
    assert len(v) >= n
    r.shuffle(v)
    return v[:n]


def bits(a):
    a = np.asarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


# ------------------------------------------------------------------------------------------------ bitonic sort
INT_MAX, INT64_MAX = 2**31 - 1, 2**63 - 1
# Each caller's instantiation: kind of entries, its block size, its largest P in shared memory and how it pads.
SORTS = {
    "search": ("f64_i32", 512, 2048),          # search_finish_kernel, deep_run_sort_kernel: (-inf, INT_MAX)
    "graph": ("f64_i64", 512, 2048),           # graph_search_kernel: (-inf, INT64_MAX)
    "diffusion": ("i32_f64", 128, 2048),       # nbr_sort: index INT_MAX, payload left as it was
    "trunc": ("u64", 256, 16384),              # trunc_build_kernel: ~0, in global memory beyond 16384
    "prune": ("u32", 128, 128),                # graph_prune_kernel: 0xffffffff
}
PAIR_KINDS = ["random", "sorted", "reversed", "equal", "zeros"]
KEY_KINDS = ["random", "sorted", "reversed", "equal", "duplicates"]


def _pair_block(form, kind, n, P, r):
    """One block of P (key, val) entries: n real ones of this kind, then the caller's padding."""
    if form == "i32_f64":                      # (index, weight) by index: indices distinct, weights any bits
        idx = distinct(r, 10**6, n).astype(np.int32)
        w = r.choice([0.0, -0.0, 0.25, -1.5, np.inf], n) * r.uniform(0.5, 1.0, n)
        if kind in ("sorted", "equal"):
            idx = np.sort(idx)
        elif kind in ("reversed", "zeros"):
            idx = np.sort(idx)[::-1].copy()
        key = np.full(P, INT_MAX, np.int32)
        val = np.full(P, np.nan)
        key[:n], val[:n] = idx, w
        return key, val
    idx_dtype = np.int32 if form == "f64_i32" else np.int64
    hi = 10**6 if form == "f64_i32" else 2**40
    idx = distinct(r, hi, n).astype(idx_dtype)
    if kind == "equal":
        sc = np.full(n, 0.5)
    elif kind == "zeros":
        sc = r.choice([-0.0, 0.0, 1.0, -np.inf], n)
    else:
        sc = np.round(r.uniform(-1, 1, n), 3)  # coarse: many ties that the index decides
    if kind in ("sorted", "reversed"):
        p = M.result_order(sc, idx)
        if kind == "reversed":
            p = p[::-1]
        sc, idx = sc[p], idx[p]
    key = np.full(P, -np.inf)
    val = np.full(P, INT_MAX if form == "f64_i32" else INT64_MAX, idx_dtype)
    key[:n], val[:n] = sc, idx
    return key, val


def _key_block(form, kind, n, P, r):
    dt = np.uint64 if form == "u64" else np.uint32
    top = np.iinfo(dt).max
    if kind == "equal":
        k = np.full(n, 12345, dt)
    elif kind == "duplicates":
        k = r.choice(np.array([0, 7, top - 1], dt), n)
    else:
        k = r.randint(0, 2**63 if form == "u64" else 2**32, n, dtype=np.uint64).astype(dt) * dt(1 + (form == "u64"))
        if kind == "sorted":
            k = np.sort(k)
        elif kind == "reversed":
            k = np.sort(k)[::-1].copy()
    key = np.full(P, top, dt)
    key[:n] = k
    return key


def _sort_sizes(name, nt, limit):
    Ps = {1, 2, 8, 64, 256, 2048, limit, 2 * nt, 4 * nt}
    if name == "trunc":
        Ps |= {16384, 32768}
    return sorted(p for p in Ps if p <= max(limit, 4 * nt) or name == "trunc")


@pytest.mark.parametrize("name", list(SORTS))
@pytest.mark.parametrize("nt", [32, 128, 256, 512, 1024])
def test_bitonic_sort(lib, name, nt):
    form, _, limit = SORTS[name]
    r = np.random.RandomState(nt + len(name))
    pairs = form in ("f64_i32", "f64_i64", "i32_f64")
    for P in _sort_sizes(name, nt, limit):
        ns = sorted({n for n in (0, 1, P // 2 + 1, P - 1, P) if 0 <= n <= P})
        kinds = PAIR_KINDS if pairs else KEY_KINDS
        cases = [(kind, n) for kind in kinds for n in ns]
        in_smem = int(not (form == "u64" and P > 16384))
        if pairs:
            blocks = [_pair_block(form, kind, n, P, r) for kind, n in cases]
            key, val = np.stack([b[0] for b in blocks]), np.stack([b[1] for b in blocks])
            k_d, v_d = dev(key), dev(val)
            sk_d, sv_d = torch.empty_like(k_d), torch.empty_like(v_d)
            lib("dirb_blocktest_sort_" + form, nt, k_d, v_d, P, len(cases), in_smem, sk_d, sv_d)
            got_k, got_v, seen_k, seen_v = (t.cpu().numpy() for t in (k_d, v_d, sk_d, sv_d))
        else:
            key = np.stack([_key_block(form, kind, n, P, r) for kind, n in cases])
            k_d = dev(key)
            sk_d = torch.empty_like(k_d)
            lib("dirb_blocktest_sort_" + form, nt, k_d, P, len(cases), in_smem, sk_d)
            got_k, seen_k = (host(t, key.dtype) for t in (k_d, sk_d))
        perm = (7 * np.arange(P) + 3) % P
        for c, (kind, n) in enumerate(cases):
            what = (name, nt, P, kind, n)
            if form == "i32_f64":
                p = np.argsort(key[c], kind="stable")        # real indices are distinct: only padding ties
                want_k, want_v = key[c][p], val[c][p]
                assert np.array_equal(got_k[c], want_k), what
                assert np.array_equal(bits(got_v[c][:n]), bits(want_v[:n])), what
                assert np.array_equal(seen_k[c], want_k[perm]), what
                assert np.array_equal(bits(seen_v[c]), bits(got_v[c][perm])), what
            elif pairs:
                p = M.result_order(key[c], val[c])
                want_k, want_v = key[c][p], val[c][p]
                assert np.array_equal(bits(got_k[c]), bits(want_k)) and np.array_equal(got_v[c], want_v), what
                assert np.array_equal(bits(seen_k[c]), bits(want_k[perm])), what
                assert np.array_equal(seen_v[c], want_v[perm]), what
            else:
                want_k = np.sort(key[c])                     # equal keys: the sorted multiset
                assert np.array_equal(got_k[c], want_k), what
                assert np.array_equal(seen_k[c], want_k[perm]), what


# ------------------------------------------------------------------------------------------------ scans
SCAN_TYPES = {"i32": np.int32, "i64": np.int64, "u64": np.uint64}


def _scan_values(t, shape, r):
    if t == "i32":                             # |sum| < 2^31 over 1024 threads
        return r.randint(-2**20, 2**20, shape).astype(np.int32)
    if t == "i64":                             # above 2^32, negative too, |sum| < 2^63
        return (r.randint(-2**52, 2**52, shape, dtype=np.int64) * np.where(r.rand(*shape) < 0.3, 1, 2**9)).astype(np.int64)
    return r.randint(0, 2**64, shape, dtype=np.uint64)   # wraps modulo 2^64


@pytest.mark.parametrize("t", list(SCAN_TYPES))
def test_block_scan_three_calls_in_a_row(lib, t):
    nts = range(32, 1025, 32) if t == "i32" else (32, 64, 96, 256, 512, 992, 1024)
    r = np.random.RandomState(len(t))
    blocks = 16
    for nt in nts:
        x = _scan_values(t, (blocks, 3, nt), r)
        if t == "u64" and nt == 1024:
            x[0] = np.iinfo(np.uint64).max                           # all ones: carries through every bit
        x_d = dev(x)
        incl_d, tot_d = torch.empty_like(x_d), torch.empty_like(x_d)
        lib("dirb_blocktest_scan_" + t, nt, x_d, incl_d, tot_d, blocks)
        incl, tot = host(incl_d, x.dtype), host(tot_d, x.dtype)
        want, want_tot = M.inclusive_sum(x, axis=2)
        assert np.array_equal(incl.astype(want.dtype), want), (t, nt)
        assert np.array_equal(tot.astype(want.dtype), np.broadcast_to(want_tot, want.shape)), (t, nt)


@pytest.mark.parametrize("t", list(SCAN_TYPES))
def test_warp_scan(lib, t):
    r = np.random.RandomState(7)
    x = _scan_values(t, (64, 32), r)
    x_d = dev(x)
    out_d = torch.empty_like(x_d)
    lib("dirb_blocktest_warp_scan_" + t, x_d, out_d, x.size)
    want, _ = M.inclusive_sum(x, axis=1)
    assert np.array_equal(host(out_d, x.dtype).astype(want.dtype), want)


# ------------------------------------------------------------------------------------------------ radix select
KTH_NTS = (32, 256, 512, 1024)
KTH_NS = sorted({1, 31, 32, 33, 4097, 2**20 + 17} | {nt + d for nt in KTH_NTS for d in (-1, 0, 1)})


def _kth_keys(keyset, n, bits_, r):
    dt = np.uint64 if bits_ == 64 else np.uint32
    top = bits_ - 8
    if keyset == "uniform":
        return r.randint(0, 2**63, n, dtype=np.uint64).astype(dt) * dt(1 + (bits_ == 64)) + dt(r.randint(0, 2))
    if keyset == "equal":
        return np.full(n, 0x5a5a5a5a, dt)
    if keyset == "two":
        return r.choice(np.array([0x40000001, 0x40000002], dt), n)
    if keyset == "low_byte":                   # all passes but the last see a single bin
        return (dt(0x3c3c3c3c) << dt(bits_ - 32)) | r.randint(0, 256, n).astype(dt)
    if keyset == "high_byte":                  # only the first pass separates them
        return (r.randint(0, 256, n).astype(dt) << dt(top)) | dt(0x00abcdef)
    if keyset == "adc":                        # pq.cu's adc_key: one score's key on top, 2^31 - 1 - row below
        return (np.uint64(0xbf333333) << np.uint64(32)) | (np.uint64(0x7fffffff) - r.permutation(n).astype(np.uint64))
    raise ValueError(keyset)


def _ks(n):
    return sorted({k for k in (1, 2, math.ceil(n / 2), n - 1, n) if 1 <= k <= n})


def _run_kth(lib, fn, keys_d, n, ks, nt, dtype):
    k1 = np.array(ks, np.int32)
    k2 = np.roll(k1, 1)                        # the second call of each block asks for a different k
    out_d = torch.empty(2 * len(ks) * np.dtype(dtype).itemsize, dtype=torch.uint8, device="cuda")
    lib(fn, nt, keys_d, n, dev(k1), dev(k2), len(ks), out_d)
    out = host(out_d, dtype).reshape(-1, 2)
    return k1, k2, out


KEYSETS = ["uniform", "equal", "two", "low_byte", "high_byte"]


@pytest.mark.parametrize("form, keyset", [(f, k) for f in ("u32", "u32_n64", "u64") for k in KEYSETS] + [("u64", "adc")])
def test_radix_select(lib, form, keyset):
    bits_ = 64 if form == "u64" else 32
    r = np.random.RandomState(bits_ + len(keyset))
    for n in KTH_NS:
        keys = _kth_keys(keyset, n, bits_, r)
        keys_d = dev(keys)
        ks = _ks(n)
        want = {k: M.kth_largest(keys, k) for k in ks}
        for nt in KTH_NTS:
            k1, k2, out = _run_kth(lib, "dirb_blocktest_kth_" + form, keys_d, n, ks, nt, keys.dtype)
            for (ka, kb), (ga, gb) in zip(zip(k1, k2), out):
                assert ga == want[ka] and gb == want[kb], (form, keyset, n, nt, ka, kb, ga, gb, want[ka], want[kb])


def test_radix_select_on_float_keys(lib):
    """The search's form: f2key of cosine-like fp32 scores sharing their high bits, with -0, +0 and -inf mixed in."""
    r = np.random.RandomState(11)
    for n in KTH_NS:
        x = (0.7 + r.uniform(-1e-4, 1e-4, n)).astype(np.float32)
        x[r.rand(n) < 0.05] = -0.0
        x[r.rand(n) < 0.05] = 0.0
        x[r.rand(n) < 0.02] = -np.inf
        x[r.rand(n) < 0.02] = -0.7
        x_d = dev(x)
        ks = _ks(n)
        want = {k: bits(M.kth_largest_float(x, k)) for k in ks}
        for nt in KTH_NTS:
            k1, k2, out = _run_kth(lib, "dirb_blocktest_kth_f32", x_d, n, ks, nt, np.uint32)
            # the keys map back to the model's k-th largest floats, bit for bit
            got = bits(_elementwise(lib, keys=out.reshape(-1))["k2f"]).reshape(-1, 2)
            for (ka, kb), (ga, gb) in zip(zip(k1, k2), got):
                assert ga == want[ka] and gb == want[kb], (n, nt, ka, kb, hex(ga), hex(gb))


# ------------------------------------------------------------------------------------------------ rank in a run
def _run(L, real, r, with_zeros=True):
    """A run of L entries in the result order: `real` valid ones, then empty ones (index -1) whose stale scores include
    values above every real score."""
    sc = r.choice([0.9, 0.5, 0.25, 0.0, -0.0, -0.5, -np.inf] if with_zeros else [0.9, 0.5, 0.25, -0.5], real)
    sc = sc + np.where(r.rand(real) < 0.5, 0.0, r.uniform(-1e-3, 1e-3, real)) * np.isfinite(sc) * (sc != 0)
    ix = distinct(r, 2**40, real)
    p = M.result_order(sc, ix)
    tail = L - real
    stale = r.choice([np.inf, 2.0, 0.9, 0.0, -np.inf], tail)
    return np.concatenate([sc[p], stale]), np.concatenate([ix[p], np.full(tail, -1, np.int64)])


def _probes(sc, ix, r):
    real = ix >= 0
    s, i = sc[real], ix[real]
    ps, pi = [s, s, s], [i, i - 1, i + 1]                      # present, and equal score with a smaller / larger index
    if len(s) > 1:
        ps.append((s[:-1] + s[1:]) / 2)                       # between neighbours
        pi.append(r.randint(0, 2**40, len(s) - 1))
    ps.append(np.array([np.inf, 10.0, -np.inf, -np.inf, 0.0, -0.0, 0.0, -0.0]))   # beyond both ends, and the zeros
    pi.append(np.array([0, 2**41, 0, 2**41, 0, 0, 2**41, 2**41]))
    zs = i[s == 0]
    for z in (0.0, -0.0):
        ps.append(np.full(3 * len(zs), z))
        pi.append(np.concatenate([zs, zs - 1, zs + 1]))
    ps, pi = np.concatenate(ps), np.concatenate(pi).astype(np.int64)
    ps = np.where(np.isnan(ps), 0.0, ps)                      # midpoint of +-inf neighbours
    return ps, pi


def _ranks(lib, sc, ix, ps, pi, ldcg):
    out = torch.empty(len(ps), dtype=torch.int32, device="cuda")
    sc_d = dev(sc) if len(sc) else torch.empty(1, dtype=torch.float64, device="cuda")
    ix_d = dev(ix) if len(ix) else torch.empty(1, dtype=torch.int64, device="cuda")
    lib("dirb_blocktest_rank", sc_d, ix_d, len(sc), dev(ps), dev(pi), len(ps), ldcg, out)
    return out.cpu().numpy()


@pytest.mark.parametrize("L", [0, 1, 2047, 2048])
def test_rank_in_run(lib, L):
    r = np.random.RandomState(L)
    reals = sorted({0, L, L - 1, L - L // 3} & set(range(L + 1)))
    for real in reals:
        sc, ix = _run(L, real, r)
        ps, pi = _probes(sc, ix, r)
        want = np.array([M.rank_in_run(sc, ix, s, i) for s, i in zip(ps, pi)])
        plain, cg = _ranks(lib, sc, ix, ps, pi, 0), _ranks(lib, sc, ix, ps, pi, 1)
        assert np.array_equal(plain, want), (L, real)
        assert np.array_equal(cg, want), (L, real)


@pytest.mark.parametrize("la, lb", [(0, 5), (1, 1), (2047, 2048), (2048, 700)])
def test_rank_merge_of_two_runs(lib, la, lb):
    r = np.random.RandomState(la + 3 * lb)
    A, B = _run(la, la - la // 8, r), _run(lb, lb - lb // 5, r)
    A[1][A[1] >= 0] *= 2                                      # distinct entries, interleaved indices: both maps keep
    B[1][B[1] >= 0] = 2 * B[1][B[1] >= 0] + 1                 # each run in the result order
    ma, mb = int((A[1] >= 0).sum()), int((B[1] >= 0).sum())
    want_sc, want_ix = M.merge(A[0][:ma], A[1][:ma], B[0][:mb], B[1][:mb])
    for ldcg in (0, 1):
        pa = np.arange(ma) + (_ranks(lib, *B, A[0][:ma], A[1][:ma], ldcg) if ma else np.zeros(0, int))
        pb = np.arange(mb) + (_ranks(lib, *A, B[0][:mb], B[1][:mb], ldcg) if mb else np.zeros(0, int))
        pos = np.concatenate([pa, pb])
        assert np.array_equal(np.sort(pos), np.arange(ma + mb)), (la, lb, ldcg)
        got_sc, got_ix = np.empty(ma + mb), np.empty(ma + mb, np.int64)
        got_sc[pos], got_ix[pos] = np.concatenate([A[0][:ma], B[0][:mb]]), np.concatenate([A[1][:ma], B[1][:mb]])
        assert np.array_equal(bits(got_sc), bits(want_sc)) and np.array_equal(got_ix, want_ix), (la, lb, ldcg)


# ------------------------------------------------------------------------------------------------ key maps
def _elementwise(lib, f=None, keys=None, sa=None, ia=None, sb=None, ib=None):
    """f2key(f), key2f(keys), fkey(sa) and both ranks_before overloads on (sa, ia, sb, ib), element by element; inputs
    left out are zeros."""
    n = max(len(a) for a in (f, keys, sa) if a is not None)

    def d(a, dt):
        return dev(np.zeros(n, dt) if a is None else np.asarray(a, dt))
    out = [torch.empty(n, dtype=t, device="cuda") for t in (torch.int32, torch.float32, torch.int64, torch.uint8, torch.uint8)]
    lib("dirb_blocktest_elementwise", d(f, np.float32), out[0], d(keys, np.uint32), out[1], d(sa, np.float64),
        d(ia, np.int64), d(sb, np.float64), d(ib, np.int64), out[2], out[3], out[4], n)
    return dict(f2k=host(out[0], np.uint32), k2f=out[1].cpu().numpy(), fk=host(out[2], np.uint64),
                before=out[3].cpu().numpy().astype(bool), before_key=out[4].cpu().numpy().astype(bool))


def test_f2key_key2f_over_every_key(lib):
    """f2key(key2f(k)) == k for all 2^32 keys, and key2f rises with k (NaNs aside), -0 immediately below +0."""
    bad = torch.zeros(2, dtype=torch.int64, device="cuda")
    lib("dirb_blocktest_key_sweep", 0, 2**31, bad)
    lib("dirb_blocktest_key_sweep", 2**31, 2**31, bad)
    assert bad.cpu().tolist() == [0, 0]
    out = _elementwise(lib, keys=np.array([0x7fffffff, 0x80000000, 0, 0xffffffff], np.uint32))
    assert bits(out["k2f"]).tolist()[:2] == [0x80000000, 0x00000000]
    assert np.isnan(out["k2f"][2:]).all()                    # the two ends of the key range are NaNs


def _neighbours(dt, tiny, big):
    v = [0.0, -0.0, tiny, -tiny, big, -big, np.inf, -np.inf]
    for c in (tiny, 1.0, -1.0, 0.5, -0.5):
        c = dt(c)
        v += [np.nextafter(c, dt(np.inf)), np.nextafter(c, dt(-np.inf))]
    for c in (1.0, -1.0, 0.5, -0.5):
        v.append(c)
    return np.array(v, dt)


def test_f2key_orders_special_floats(lib):
    fi = np.finfo(np.float32)
    x = _neighbours(np.float32, fi.smallest_subnormal, fi.max)
    x = np.concatenate([x, x[::-1], np.random.RandomState(1).standard_normal(200).astype(np.float32)])
    out = _elementwise(lib, f=x)
    order = M.float_total_order(x)
    keys, xs = out["f2k"][order], bits(x[order])
    same = xs[1:] == xs[:-1]
    assert ((keys[1:] > keys[:-1]) | same).all() and (keys[1:][same] == keys[:-1][same]).all()
    assert np.array_equal(bits(_elementwise(lib, keys=out["f2k"])["k2f"]), bits(x))


def test_fkey_and_ranks_before(lib):
    fi = np.finfo(np.float64)
    v = _neighbours(np.float64, fi.smallest_subnormal, fi.max)
    a, b = np.repeat(v, len(v)), np.tile(v, len(v))
    idx = [(0, 0), (0, 1), (1, 0), (5, 2**40), (2**40, 5)]
    sa, sb = np.tile(a, len(idx)), np.tile(b, len(idx))
    ia = np.repeat([p[0] for p in idx], len(a)).astype(np.int64)
    ib = np.repeat([p[1] for p in idx], len(a)).astype(np.int64)
    out = _elementwise(lib, sa=sa, ia=ia, sb=sb, ib=ib)
    fa, fb = out["fk"], _elementwise(lib, sa=sb)["fk"]
    assert np.array_equal(fa < fb, sa < sb) and np.array_equal(fa == fb, sa == sb)   # -0 and +0 share a key
    want = M.ranks_before(sa, ia, sb, ib)
    assert np.array_equal(out["before"], want)
    assert np.array_equal(out["before_key"], want)
