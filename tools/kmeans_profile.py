"""Timings of spherical k-means on one GPU -> results/h100_kmeans.json (or --out).

Data: N = 1M clustered unit rows of D = 2048 generated on the GPU from a seed (one centre per 100 rows, per-entry noise
0.6, within-cluster scores ~0.74; the rows of tools/join_profile.py without the duplicate groups).  For K = 1024, 16384
and 65536 centres drawn from the rows: the assignment by Index(C).nearest(X) (rules K2 / K3, checked equal to
Index(C).search(X, 1) in the same run) and by Index(C).search(X, 1), the statistics pass and one centre update (rule
K5), each timed with CUDA events over --reps rounds after a warm-up round (median, min, max).  Then k-means++ at
K = 1024 and one fit of 20 iterations at K = 1024.  For scale, one iteration of scikit-learn's KMeans (init = an array, n_init = 1,
max_iter = 1, all host CPUs) at 100k x 2048, K = 1024.  The card's name, power limit and max SM clock are read in the
same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dirb200  # noqa: E402,F401
from dirb200 import cluster, lib, ops  # noqa: E402


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def _rows(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((max(2, n // 100), d), generator=g, device="cuda")
    x = c[torch.randint(0, c.shape[0], (n,), generator=g, device="cuda")]
    x += 0.6 * torch.randn((n, d), generator=g, device="cuda")
    del c
    return torch.nn.functional.normalize(x, dim=1).contiguous()


def _events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def _spread(ms):
    return dict(median=float(np.median(ms)), min=float(min(ms)), max=float(max(ms)), reps=len(ms))


def _search_top1(x, centres):
    idx = ops.Index(centres, check_norms=False)
    try:
        return idx.search(x, 1)
    finally:
        idx.close()


def _iteration(x, k, seed, reps):
    n, d = x.shape
    rows = torch.from_numpy(np.random.RandomState(seed).permutation(n)[:k]).to(x.device)
    centres = x[rows].contiguous()
    counts = torch.empty(k, dtype=torch.int32, device=x.device)
    ws_s = torch.empty(256, dtype=torch.uint8, device=x.device)
    ws_u = torch.empty(lib.raw("dirb200_kmeans_update_workspace_bytes")(n, k, d), dtype=torch.uint8, device=x.device)
    out = (C.c_int64 * 3)()
    z = C.c_int64()
    times = dict(nearest=[], search=[], stats=[], update=[])
    stats = dict(band_rows=0, full_rescores=0)
    for rep in range(reps + 1):                               # round 0 warms every shape up and is not kept
        st = dict(band_rows=0, full_rescores=0)
        (lab, sc), t_near = _events_ms(lambda: cluster.assign(x, centres, st))
        (s1, i1), t_search = _events_ms(lambda: _search_top1(x, centres))
        same = bool(torch.equal(lab, i1[:, 0]) and torch.equal(sc, s1[:, 0]))
        del s1, i1
        _, t_stats = _events_ms(lambda: lib.call("dirb200_kmeans_stats", ops._ptr(lab), ops._ptr(sc), None, n, k,
                                                 ops._ptr(ws_s), ops._ptr(counts), out, ops._stream()))
        c2 = centres.clone()
        _, t_update = _events_ms(lambda: lib.call("dirb200_kmeans_update", ops._ptr(x), n, d, ops._ptr(lab), ops._ptr(counts),
                                                  k, ops._ptr(c2), ops._ptr(ws_u), C.byref(z), ops._stream()))
        if rep:
            for key, t in (("nearest", t_near), ("search", t_search), ("stats", t_stats), ("update", t_update)):
                times[key].append(t)
            stats = st
    del ws_u
    res = dict(k=k, empty_clusters=int(out[2]), nearest_equals_search=same, nearest_stats=stats)
    for key, ms in times.items():
        res[key + "_ms"] = _spread(ms)
    res["nearest_tflops_2nkd"] = 2.0 * n * k * d / res["nearest_ms"]["median"] / 1e9
    res["search_tflops_2nkd"] = 2.0 * n * k * d / res["search_ms"]["median"] / 1e9
    return res


def _sklearn(d, k, seed):
    try:
        from sklearn.cluster import KMeans
    except ImportError:
        return dict(skipped="scikit-learn is not installed")
    n = 100000
    r = np.random.RandomState(seed)
    c = r.standard_normal((n // 100, d)).astype(np.float32)
    x = c[r.randint(0, c.shape[0], n)] + 0.6 * r.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    init = x[r.permutation(n)[:k]]
    t = time.perf_counter()
    KMeans(n_clusters=k, init=init, n_init=1, max_iter=1).fit(x)
    return dict(n=n, d=d, k=k, seconds=time.perf_counter() - t, cpus=os.cpu_count())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--ks", type=str, default="1024,16384,65536")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-sklearn", action="store_true")
    ap.add_argument("--out", type=str, default="results/h100_kmeans.json")
    a = ap.parse_args()
    ops.require_gpu(0)
    res = dict(card=_card(), n=a.n, d=a.d, iterations=[])
    x = _rows(a.n, a.d, 0)
    for k in [int(s) for s in a.ks.split(",")]:
        r = _iteration(x, k, 1, a.reps)
        print(r, flush=True)
        res["iterations"].append(r)
    cluster.kmeans_pp_rows(x[:4096].contiguous(), 16, 0)     # warm-up
    _, t_pp = _events_ms(lambda: cluster.kmeans_pp_rows(x, 1024, 0))
    res["kmeans_pp_1024_ms"] = t_pp
    print("k-means++ K=1024: %.1f ms" % t_pp, flush=True)
    km = cluster.SphericalKMeans(1024, init="k-means++", max_iter=20, seed=0)
    _, t_fit = _events_ms(lambda: km.fit(x))
    res["fit_1024"] = dict(ms=t_fit, n_iter=km.n_iter_, objective=km.objective_, stats=km.stats_)
    print("fit K=1024: %.1f ms, %d iterations" % (t_fit, km.n_iter_), flush=True)
    if not a.no_sklearn:
        res["sklearn_one_iteration"] = _sklearn(a.d, 1024, 2)
        print(res["sklearn_one_iteration"], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
