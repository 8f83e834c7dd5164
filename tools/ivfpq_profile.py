"""IVF-PQ against the fp16 IVF path and the exact search on an H100 -> results/h100_ivfpq.json (DESIGN.md section 4.11).

Data: the rows of tools/kmeans_profile.py (as tools/ivf_profile.py draws them): 2^20 + 10 000 rows, D = 2048, the last
10 000 the queries.  K = 1024 lists from 5 iterations of SphericalKMeans (init 'random', seed 0); k = 100.  Per M in
{32, 64, 128}: device bytes per row and build time (training on 65 536 rows with 25 iterations, then the encoding).
Searches (CUDA events, median of 3 after a warm-up; stages from option profile in a separate call): M = 64 over
nprobe {8, 32, 128} x R {k, 4k, 16k} x Q {70, 1000, 10 000} with the rows on the device; every M at nprobe 32, R 4k,
Q 1000; the rows in pinned host memory at nprobe 32, R {k, 4k, 16k}, Q {70, 1000}.  Each next to IVFIndex.search at
the same nprobe and Index.search, with recall@100 against Index.search.
Usage: python tools/ivfpq_profile.py [--rows 1048576] [--out results/h100_ivfpq.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dirb200 import cluster, ivf, ivfpq, ops  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_profile import _rows, _timed  # noqa: E402


def _recall(a, b):
    hit = sum(len(set(x.tolist()) & set(y.tolist())) for x, y in zip(a.cpu(), b.cpu()))
    return hit / float(b.numel())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--out", default="results/h100_ivfpq.json")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    D, k, K = 2048, 100, 1024
    allx = _rows(a.rows + 10000, D, 1)
    X = allx[:a.rows].contiguous()
    Qall = allx[a.rows:].contiguous()
    del allx
    km = cluster.SphericalKMeans(K, init="random", max_iter=5, seed=0).fit(X)
    exact = ops.Index(X)
    lists = ivf.IVFIndex(X, km)
    res = dict(card=smi, rows=a.rows, dim=D, k=k, n_lists=K,
               data="tools/kmeans_profile.py rows: N/100 centres + 0.6 noise (synthetic: recall here says nothing "
                    "about real descriptors)",
               builds=[], runs=[])
    truth, base = {}, {}
    for Q in (70, 1000, 10000):
        q = Qall[:Q]
        t, (_, truth[Q]) = _timed(lambda: exact.search(q, k))
        base[("exact", Q)] = t
        for nprobe in (8, 32, 128):
            t, (_, got) = _timed(lambda: lists.search(q, k, nprobe))
            base[(nprobe, Q)] = (t, _recall(got, truth[Q]))
    res["exact_ms"] = {str(Q): base[("exact", Q)] for Q in (70, 1000, 10000)}
    res["ivf"] = [dict(nprobe=p, queries=Q, ms=base[(p, Q)][0], recall=base[(p, Q)][1])
                  for p in (8, 32, 128) for Q in (70, 1000, 10000)]

    def run(index, M, where, nprobe, R, Q):
        q = Qall[:Q]
        t, (_, got) = _timed(lambda: index.search(q, k, nprobe, refine=R))
        index.set_option("profile", 1)
        index.search(q, k, nprobe, refine=R)
        index.set_option("profile", 0)
        st = index.stats()
        row = dict(M=M, rows=where, nprobe=nprobe, refine=R, queries=Q, ms=t, recall=_recall(got, truth[Q]),
                   ivf_ms=base[(nprobe, Q)][0], ivf_recall=base[(nprobe, Q)][1], exact_ms=base[("exact", Q)], stages=st)
        res["runs"].append(row)
        print(json.dumps(row), flush=True)

    for M in (32, 64, 128):
        for where in ("device", "host"):
            if where == "host" and M != 64:
                continue
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            index = ivfpq.IVFPQIndex(X, km, M, rows=where)
            torch.cuda.synchronize()
            b = dict(M=M, rows=where, build_s=time.perf_counter() - t0, device_bytes=index.device_bytes_,
                     device_bytes_per_row=index.device_bytes_ / a.rows, empty_codewords=index.empty_codewords_)
            res["builds"].append(b)
            print(json.dumps(b), flush=True)
            if where == "device" and M == 64:
                for nprobe in (8, 32, 128):
                    for R in (k, 4 * k, 16 * k):
                        for Q in (70, 1000, 10000):
                            run(index, M, where, nprobe, R, Q)
            elif where == "device":
                run(index, M, where, 32, 4 * k, 1000)
            else:
                for R in (k, 4 * k, 16 * k):
                    for Q in (70, 1000):
                        run(index, M, where, 32, R, Q)
            index.close()
            del index
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
