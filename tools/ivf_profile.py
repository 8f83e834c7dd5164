"""Inverted-file search against the exact search on an H100 -> results/h100_ivf.json (DESIGN.md section 4.10).

Data: the rows of tools/kmeans_profile.py - N / 100 Gaussian centres, each row a centre plus 0.6 Gaussian noise,
normalised (D = 2048) - drawn for 2^20 + 10 000 rows in one call; the last 10 000 are the queries, held-out rows of the
same clusters.  Lists from 5 iterations of SphericalKMeans (init 'random', seed 0).  k = 100.  For each (K, nprobe, Q):
CUDA-event time of the probe and of the list search (median of 3 after a warm-up), the list search's own stages
(option profile, a separate call), queries/s next to Index.search on the same queries, recall@100 against it, issued
against useful FLOPs of the grouped passes (issued = tiles * 2 * 128 * 128 * D per pass; useful = sum_q |R(q)| * 2 * D),
and a bit-identity check at nprobe = K (at Q = 10 000 that call runs in several query blocks within ws_budget).
Usage: python tools/ivf_profile.py [--rows 1048576] [--out results/h100_ivf.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dirb200 import cluster, ivf, ops  # noqa: E402


def _rows(n, d, seed):
    """tools/kmeans_profile.py's rows."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((max(2, n // 100), d), generator=g, device="cuda")
    x = c[torch.randint(0, c.shape[0], (n,), generator=g, device="cuda")]
    x += 0.6 * torch.randn((n, d), generator=g, device="cuda")
    del c
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--out", default="results/h100_ivf.json")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    D, k = 2048, 100
    allx = _rows(a.rows + 10000, D, 1)
    X = allx[:a.rows].contiguous()
    Qmax = allx[a.rows:].contiguous()
    del allx
    exact = ops.Index(X)
    res = dict(card=smi, rows=a.rows, dim=D, k=k, data="tools/kmeans_profile.py rows: N/100 centres + 0.6 noise", runs=[], exact=[])
    base = {}
    for Q in (70, 1000, 10000):
        q = Qmax[:Q].contiguous()
        ms, out = _timed(lambda: exact.search(q, k))
        base[Q] = out
        res["exact"].append(dict(Q=Q, ms=ms, qps=Q / ms * 1e3))
        print("exact Q=%d %.2f ms" % (Q, ms), flush=True)
    for K in (1024, 4096):
        km = cluster.SphericalKMeans(K, init="random", max_iter=5, seed=0).fit(X)
        index = ivf.IVFIndex(X, km)
        sizes = index.list_sizes_.float()
        for nprobe in (1, 8, 32, 128, K):
            for Q in (70, 1000, 10000):
                q = Qmax[:Q].contiguous()
                probe_ms, probes = _timed(lambda: index.probe(q, nprobe))
                ms, (s, i) = _timed(lambda: index.index.search_lists(q, k, probes))
                st = index.stats()
                index.set_option("profile", 1)
                index.index.search_lists(q, k, probes)
                prof = index.stats()
                index.set_option("profile", 0)
                es, ei = base[Q]
                hit = (i[:, :, None] == ei[:, None, :]).any(2).float().mean().item()
                row = dict(K=K, nprobe=nprobe, Q=Q, probe_ms=probe_ms, search_ms=ms, qps=Q / (probe_ms + ms) * 1e3,
                           exact_qps=Q / [e for e in res["exact"] if e["Q"] == Q][0]["ms"] * 1e3, recall_at_100=hit,
                           stages_ms={n: prof[n] for n in ("build_ms", "gmax_ms", "filter_ms", "finish_ms")},
                           tiles=st["tiles"], pairs=st["pairs"], query_rows=st["query_rows"], probed_rows=st["probed_rows"],
                           candidates=st["candidates"], reruns=st["reruns"],
                           issued_tflop_per_pass=st["tiles"] * 2 * 128 * 128 * D / 1e12,
                           useful_tflop_per_pass=st["probed_rows"] * 2 * D / 1e12,
                           brute_force_tflop=-(-Q // 128) * 128 * a.rows * 2 * D / 1e12,
                           largest_list=int(sizes.max()))
                if nprobe == K:
                    row["bit_identical_to_search"] = bool(torch.equal(i, ei) and torch.equal(s.view(torch.int64), es.view(torch.int64)))
                res["runs"].append(row)
                print(json.dumps(row), flush=True)
        index.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
