"""The stream contract of include/dirb200.h and INTEGRATION.md: every launch, memset and copy runs on the caller's
stream, every host read-back waits for the kernels that produce it, and handles or handle-less calls on different
streams do not share device memory unordered.

torch's default stream is the legacy stream, which serialises with everything, so a call made from it cannot show such
a bug.  Here every case of tests/stream_cases.py runs once on the default stream and once on a non-blocking side stream
behind a gate: the buffers the call reads hold poison (all bits set: NaN, -1) until the side stream, after a ~30 ms
spin, copies the real inputs in.  Work put on stream 0 or on a stream of the library's own runs during the spin and
reads poison, a read-back that does not wait reads values from before the kernels, and output written off the side
stream misses the clone taken there.  The two runs must agree bit for bit.  Needs an H100: -m gpu."""
import threading
from contextlib import contextmanager

import numpy as np
import pytest
import torch

import stream_cases as SC

pytestmark = pytest.mark.gpu

GATE_CYCLES = 50_000_000            # torch.cuda._sleep: ~25-35 ms at the H100's clocks


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


@contextmanager
def global_options(options):
    ops = _ops()
    saved = {k: ops.get_global_option(k) for k in options}
    try:
        for k, v in options.items():
            ops.set_global_option(k, v)
        yield
    finally:
        for k, v in saved.items():
            ops.set_global_option(k, v)


@contextmanager
def recorded_calls(monkeypatch):
    """The names of the entry points reached through lib.call."""
    from dirb200 import lib
    names = set()
    real = lib.call

    def call(name, *args):
        names.add(name)
        return real(name, *args)
    monkeypatch.setattr(lib, "call", call)
    try:
        yield names
    finally:
        monkeypatch.setattr(lib, "call", real)


def snapshot(out):
    """Copies of the outputs, taken on the current stream: tensors cloned, host values kept."""
    if isinstance(out, torch.Tensor):
        return out.clone()
    if isinstance(out, dict):
        return {k: snapshot(v) for k, v in out.items()}
    if isinstance(out, (list, tuple)):
        return [snapshot(v) for v in out]
    if isinstance(out, np.ndarray):
        return out.copy()
    assert out is None or isinstance(out, (bool, int, float, str, np.generic)), type(out)
    return out


def bits(out):
    """Outputs as comparable host values: tensors and arrays as (dtype, shape, raw bytes), so that NaN equals NaN."""
    if isinstance(out, torch.Tensor):
        a = out.detach().cpu().contiguous().numpy()
        return (str(a.dtype), a.shape, a.tobytes())
    if isinstance(out, np.ndarray):
        return (str(out.dtype), out.shape, np.ascontiguousarray(out).tobytes())
    if isinstance(out, dict):
        return {k: bits(v) for k, v in out.items()}
    if isinstance(out, list):
        return [bits(v) for v in out]
    if isinstance(out, float):
        return float.hex(out)
    return out


def first_difference(got, want, path="out"):
    if type(got) is not type(want):
        return "%s: %r vs %r" % (path, type(got), type(want))
    if isinstance(want, dict):
        if set(got) != set(want):
            return "%s: keys %s vs %s" % (path, sorted(got), sorted(want))
        for k in want:
            d = first_difference(got[k], want[k], "%s[%r]" % (path, k))
            if d:
                return d
        return None
    if isinstance(want, list):
        if len(got) != len(want):
            return "%s: %d vs %d items" % (path, len(got), len(want))
        for i, (g, w) in enumerate(zip(got, want)):
            d = first_difference(g, w, "%s[%d]" % (path, i))
            if d:
                return d
        return None
    if isinstance(want, tuple) and len(want) == 3 and isinstance(want[2], bytes):
        if got[:2] != want[:2]:
            return "%s: %s %s vs %s %s" % (path, got[0], got[1], want[0], want[1])
        if got[2] != want[2]:
            g = np.frombuffer(got[2], np.uint8)
            w = np.frombuffer(want[2], np.uint8)
            return "%s (%s %s): %d of %d bytes differ" % (path, want[0], want[1], int((g != w).sum()), w.size)
        return None
    return None if got == want else "%s: %r vs %r" % (path, got, want)


def assert_same(got, want, what):
    d = first_difference(got, want)
    assert d is None, "%s: the side stream differs from the default stream at %s" % (what, d)


def poison(t):
    buf = torch.empty(t.shape, dtype=t.dtype, device=t.device)
    buf.view(-1).view(torch.uint8).fill_(0xFF)
    return buf


def run_default(case):
    torch.cuda.synchronize()
    run = case.build(lambda t: t)
    out = snapshot(run())
    torch.cuda.synchronize()
    return out


def run_gated(case):
    fills = []

    def mk(t):
        buf = poison(t)
        fills.append((buf, t))
        return buf
    run = case.build(mk)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(GATE_CYCLES)
        for buf, t in fills:
            buf.copy_(t)
        out = snapshot(run())
    torch.cuda.synchronize()
    return out


# Host-visible results that show a case took the path it is there for.
def _first(out, *keys):
    for k in keys:
        out = out[k]
    return out


TOOK_ITS_PATH = {
    "index_search_forced_retry": lambda out: _first(out, 1, "retries") >= 1,
    "index_deferred_check_overflow": lambda out: out == -4,
    "count_ge_band_recount": lambda out: _first(out, 1, "retries") >= 1,
    "self_join": lambda out: _first(out, 1, "reruns") >= 1,
    "jpeg_decode": lambda out: out[2] > 1 and out[1] == [True, True, True, True, False],
    "kmeans_fit_relocate": lambda out: _first(out, 5, "relocations") >= 1,
}


@pytest.mark.parametrize("case", SC.STREAM_CASES, ids=lambda c: c.name)
def test_gated_side_stream_equals_the_default_stream(case, monkeypatch):
    _ops()
    with global_options(case.options):
        with recorded_calls(monkeypatch) as names:
            want = run_default(case)
        missed = set(case.covers) - names
        assert not missed, "case %s did not reach %s" % (case.name, sorted(missed))
        if case.name in TOOK_ITS_PATH:
            assert TOOK_ITS_PATH[case.name](want), "case %s did not take its path" % case.name
        got = run_gated(case)
    assert_same(bits(got), bits(want), case.name)


# ------------------------------------------------------------------------------------------------ concurrent handles
def run_threads(fns):
    """fns[i]() in thread i on a stream of its own; every stream waits on one event recorded after a spin on another
    stream, so the threads' kernels become ready together.  -> the snapshots of the results."""
    gate = torch.cuda.Stream()
    streams = [torch.cuda.Stream() for _ in fns]
    ev = torch.cuda.Event()
    torch.cuda.synchronize()
    with torch.cuda.stream(gate):
        torch.cuda._sleep(GATE_CYCLES)
        ev.record(gate)
    results, errors = [None] * len(fns), []

    def work(i):
        try:
            with torch.cuda.device(0), torch.cuda.stream(streams[i]):
                streams[i].wait_event(ev)
                results[i] = snapshot(fns[i]())
        except BaseException as e:               # noqa: B902 - re-raised in the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(len(fns))]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in threads), "a thread did not finish"
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    return results


def _pair_index():
    ops = _ops()
    a, b = ops.Index(SC.unit(6000, 256, seed=200)), ops.Index(SC.unit(4000, 256, seed=201))
    qa, qb = SC.unit(30, 256, seed=202), SC.unit(20, 256, seed=203)
    return (lambda: (a.search(qa, 40), a.search(qa, 1200), a.stats()["retries"]),
            lambda: (b.search(qb, 40), b.search(qb, 1200), b.stats()["retries"]))


def _pair_jpeg():
    from test_jpeg_host import encode, make_image
    ops = _ops()
    fa = [encode(make_image(64 + 8 * i, 48, "smooth", seed=i), quality=90, subsampling=2) for i in range(6)]
    fb = [encode(make_image(40, 72 + 8 * i, "noise", seed=10 + i), quality=80, subsampling=1) for i in range(5)]
    da, db = ops.JpegDecoder(subseq_bits=64), ops.JpegDecoder(subseq_bits=64)

    def dec(d, files):
        def run():
            imgs, ok = d.decode(files)
            return imgs, ok, d.last_rounds
        return run
    return dec(da, fa), dec(db, fb)


def _pair_graph():
    from dirb200.graph import GraphIndex
    ga = GraphIndex(SC.clustered(2500, 128, seed=204), degree=16, build_k=32, n_entry=256)
    gb = GraphIndex(SC.clustered(1800, 128, seed=205), degree=16, build_k=32, n_entry=256)
    qa, qb = SC.clustered(12, 128, seed=206), SC.clustered(9, 128, seed=207)
    return (lambda: ga.search(qa, 10, itopk=64, max_iter=32)), (lambda: gb.search(qb, 10, itopk=64, max_iter=32))


def _pair_diffusion():
    from dirb200.diffusion import Diffusion
    da, db = Diffusion(SC.clustered(1500, 128, seed=208), k=20), Diffusion(SC.clustered(1200, 128, seed=209), k=20)
    qa, qb = SC.clustered(6, 128, seed=210), SC.clustered(5, 128, seed=211)
    return (lambda: da.search(qa, 30, kq=5, iters=15)), (lambda: db.search(qb, 30, kq=5, iters=15))


@pytest.mark.parametrize("pair", [_pair_index, _pair_jpeg, _pair_graph, _pair_diffusion],
                         ids=["index", "jpeg", "graph", "diffusion"])
def test_two_handles_on_two_streams_equal_their_sequential_results(pair):
    fa, fb = pair()
    torch.cuda.synchronize()
    want = [bits(snapshot(fa())), bits(snapshot(fb()))]
    torch.cuda.synchronize()
    got = [bits(r) for r in run_threads([fa, fb])]
    assert_same(got[0], want[0], "handle A")
    assert_same(got[1], want[1], "handle B")


# -------------------------------------------------------------------------------------------------- shared scratch
def _whiten_call(n, d, dout, seed):
    """A whitening on the tensor-core path (its split buffers live in the process-wide scratch)."""
    x = SC.unit(n, d, seed=seed)
    comp = SC.randn(dout, d, seed=seed + 1, scale=d ** -0.5)
    mean = SC.randn(d, seed=seed + 2, scale=0.01 * (seed % 7 + 1))
    return lambda: _ops().whiten(x, comp, mean, None, l2norm=False)


def _gram_call(n, d, seed):
    x = SC.randn(n, d, seed=seed, scale=seed % 5 + 1)
    mean = SC.randn(d, seed=seed + 1, dtype=torch.float64, scale=0.1)
    return lambda: _ops().gram_f64(x, mean)


def run_two_streams(fa, fb):
    """fa on stream A, then fb on stream B, from this thread; both streams gated by one event, so that without the
    scratch's ordering the two calls would run on the scratch at the same time."""
    gate, sa, sb = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    ev = torch.cuda.Event()
    torch.cuda.synchronize()
    with torch.cuda.stream(gate):
        torch.cuda._sleep(GATE_CYCLES)
        ev.record(gate)
    sa.wait_event(ev)
    sb.wait_event(ev)
    with torch.cuda.stream(sa):
        ra = snapshot(fa())
    with torch.cuda.stream(sb):
        rb = snapshot(fb())
    torch.cuda.synchronize()
    return ra, rb


def _sequential(*fns):
    torch.cuda.synchronize()
    out = [bits(snapshot(f())) for f in fns]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("kind", ["whiten", "gram_f64"])
def test_scratch_users_on_two_streams(kind):
    if kind == "whiten":
        fa, fb = _whiten_call(8192, 1024, 512, seed=300), _whiten_call(2048, 1024, 512, seed=305)
    else:
        fa, fb = _gram_call(60000, 512, seed=310), _gram_call(50000, 512, seed=312)
    want = _sequential(fa, fb)
    got = [bits(r) for r in run_two_streams(fa, fb)]
    assert_same(got, want, kind)


def test_scratch_grows_while_another_stream_uses_it():
    """B needs more scratch than anything before it in the process (2 GiB of split buffers): its acquire frees and
    reallocates the buffer while A's call, queued behind the gate, has not run yet.  The gated pair runs first, so
    that the growth happens there."""
    fa = _whiten_call(4096, 2048, 256, seed=320)
    fb = _whiten_call(1 << 18, 2048, 128, seed=322)
    got = [bits(r) for r in run_two_streams(fa, fb)]
    want = _sequential(fa, fb)
    assert_same(got, want, "whiten with growth")


def test_scratch_users_on_two_threads():
    """One run from two threads, each on its own gated stream: the lease neither deadlocks nor mis-orders."""
    fa, fb = _whiten_call(8192, 1024, 512, seed=330), _whiten_call(6000, 1024, 384, seed=333)
    want = _sequential(fa, fb)
    got = [bits(r) for r in run_threads([fa, fb])]
    assert_same(got, want, "whiten from two threads")
