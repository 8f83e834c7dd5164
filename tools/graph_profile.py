"""Graph search against the exact search and IVF on an H100 -> results/h100_graph.json (DESIGN.md section 4.12).

Data, D = 2048, drawn for N + 10 000 rows in one call, the last 10 000 held out as queries:
- "clustered": tools/kmeans_profile.py's rows (N / 100 Gaussian centres, each row a centre plus 0.6 Gaussian noise,
  normalised), about 10^4 tight clusters, so the graph is expected to fall apart into many components;
- "gaussian": unclustered Gaussian rows with a per-dimension scale exp(-j / 32), normalised.
For each set: the build (GraphIndex, degree 32, build_k 64) split into kNN, prune and merge, n_components_, then at
Q = 1, 70, 1000, 10 000 and k = 100 the CUDA-event time (median of 3 after a warm-up) of GraphIndex.search for a few
(itopk, width, max_iter), the mean rows visited and iterations per query, recall@100 against Index.search, and in the
same call Index.search and IVFIndex (K = 1024 lists from 5 k-means iterations, nprobe 1 and 32, probe + list search).
Usage: python tools/graph_profile.py [--rows 1048576] [--out results/h100_graph.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dirb200 import cluster, graph, ivf, ops  # noqa: E402

QS = (1, 70, 1000, 10000)
WALKS = ((128, 1, 256), (256, 1, 256), (256, 4, 64))     # (itopk, width, max_iter)


def _clustered(n, d, seed):
    """tools/kmeans_profile.py's rows."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((max(2, n // 100), d), generator=g, device="cuda")
    x = c[torch.randint(0, c.shape[0], (n,), generator=g, device="cuda")]
    x += 0.6 * torch.randn((n, d), generator=g, device="cuda")
    del c
    return torch.nn.functional.normalize(x, dim=1).contiguous()


def _gaussian(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((n, d), generator=g, device="cuda")
    x *= torch.exp(-torch.arange(d, device="cuda", dtype=torch.float32) / 32)
    return torch.nn.functional.normalize(x, dim=1).contiguous()


def _timed(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2], out


def _recall(i, ei):
    return (i[:, :, None] == ei[:, None, :]).any(2).float().mean().item()


def _one(name, X, Qmax, k, res):
    exact = ops.Index(X)
    base = {}
    for Q in QS:
        q = Qmax[:Q].contiguous()
        ms, out = _timed(lambda: exact.search(q, k))
        base[Q] = out[1]
        res["exact"].append(dict(data=name, Q=Q, ms=ms))
        print(name, "exact Q=%d %.3f ms" % (Q, ms), flush=True)
    exact.close()
    torch.cuda.synchronize()
    g = graph.GraphIndex(X, degree=32, build_k=64)
    torch.cuda.synchronize()
    res["builds"].append(dict(data=name, degree=32, build_k=64, n_components=g.n_components_, **g.build_ms_))
    print(json.dumps(res["builds"][-1]), flush=True)
    for itopk, width, max_iter in WALKS:
        for Q in QS:
            q = Qmax[:Q].contiguous()
            ms, (s, i) = _timed(lambda: g.search(q, k, itopk=itopk, width=width, max_iter=max_iter))
            st = g.stats()
            row = dict(data=name, itopk=itopk, width=width, max_iter=max_iter, Q=Q, ms=ms,
                       visited_mean=st["visited"].float().mean().item(),
                       iterations_mean=st["iterations"].float().mean().item(), recall_at_100=_recall(i, base[Q]))
            res["graph"].append(row)
            print(json.dumps(row), flush=True)
    g.close()
    torch.cuda.synchronize()
    km = cluster.SphericalKMeans(1024, init="random", max_iter=5, seed=0).fit(X)
    index = ivf.IVFIndex(X, km)
    for nprobe in (1, 32):
        for Q in QS:
            q = Qmax[:Q].contiguous()
            ms, (s, i) = _timed(lambda: index.search(q, k, nprobe))
            row = dict(data=name, K=1024, nprobe=nprobe, Q=Q, ms=ms, recall_at_100=_recall(i, base[Q]))
            res["ivf"].append(row)
            print(json.dumps(row), flush=True)
    index.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--out", default="results/h100_graph.json")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    D, k = 2048, 100
    res = dict(card=smi, rows=a.rows, dim=D, k=k, builds=[], exact=[], graph=[], ivf=[])
    for name, make in (("clustered", _clustered), ("gaussian", _gaussian)):
        allx = make(a.rows + 10000, D, 1)
        X = allx[:a.rows].contiguous()
        Qmax = allx[a.rows:].contiguous()
        del allx
        _one(name, X, Qmax, k, res)
        del X, Qmax
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
