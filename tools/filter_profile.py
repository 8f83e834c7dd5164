"""Filtered exact search on an H100 -> results/h100_filter.json (DESIGN.md section 4.13).

Data: 2^20 unclustered Gaussian rows (per-dimension scale exp(-j / 32), normalised; tools/graph_profile.py's "gaussian"
set), D = 2048, k = 100, queries held out from the same draw.  Allow sets: none, every bit set, random 50 / 10 / 1 %,
the last 10 % of the rows as one block (all of them outside the unfiltered seed rows), and per-query self-exclusion
with the queries drawn from the database rows (ops.allow_exclude).  Q = 1, 70, 1000, and 10 000 for the shared sets.
Per run: the CUDA-event time of Index.search (median of 3 after a warm-up), then one run with option "profile" for the
phase times (seed = gather + seed GEMM, filter pass, finish), the candidates and the retry passes; for the shared sets
also what a user does without the filter, Index(X[A]) built and then searched, timed the same way.
The card's name, power limit and SM clocks are read in the same call.
Usage: python tools/filter_profile.py [--rows 1048576] [--out results/h100_filter.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dirb200 import ops  # noqa: E402

QS = (1, 70, 1000)
Q_SHARED_ONLY = 10000


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


def _shared_sets(n):
    g = torch.Generator(device="cuda").manual_seed(5)
    u = torch.rand(n, generator=g, device="cuda")
    yield "all", torch.ones(n, dtype=torch.bool, device="cuda")
    for pct in (50, 10, 1):
        yield "random_%d%%" % pct, u < pct / 100
    blk = torch.zeros(n, dtype=torch.bool, device="cuda")
    blk[n - n // 10:] = True
    yield "block_last_10%", blk


def _run(index, q, k, allow, row):
    ms, _ = _timed(lambda: index.search(q, k, allow=allow))
    index.set_option("profile", 1)
    index.search(q, k, allow=allow)
    torch.cuda.synchronize()
    pr, st = index.profile(), index.stats()
    index.set_option("profile", 0)
    row.update(ms=ms, seed_ms=pr["seed_gemm"] + pr["seed_kth"], filter_ms=pr["filter_gemm"], select_ms=pr["cand_select"],
               finish_ms=pr["finish"], candidates=st["candidates"], retries=st["retries"], retried=st["retries"] > 0)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--out", default="results/h100_filter.json")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    D, k, n = 2048, 100, a.rows
    allx = _gaussian(n + Q_SHARED_ONLY, D, 1)
    X = allx[:n].contiguous()
    Qmax = allx[n:].contiguous()
    del allx
    index = ops.Index(X)
    res = dict(card=smi, rows=n, dim=D, k=k, runs=[])
    sets = list(_shared_sets(n))
    for Q in QS + (Q_SHARED_ONLY,):
        q = Qmax[:Q].contiguous()
        res["runs"].append(_run(index, q, k, None, dict(set="none", Q=Q)))
        print(json.dumps(res["runs"][-1]), flush=True)
        for name, mask in sets:
            w = ops.allow_rows(mask)
            row = _run(index, q, k, w, dict(set=name, Q=Q, allowed=int(mask.sum())))

            def today():
                rows = mask.nonzero().squeeze(1)
                sub = ops.Index(X[rows].contiguous())
                out = sub.search(q, k)
                sub.close()
                return out

            row["subset_index_ms"], _ = _timed(today)
            res["runs"].append(row)
            print(json.dumps(row), flush=True)
        if Q in QS:                                   # per-query sets: leave each query's own row out (queries = rows)
            qr = X[:Q].contiguous()
            w = ops.allow_exclude(ops.allow_rows(torch.ones(n, dtype=torch.bool, device="cuda")), Q,
                                  [[i] for i in range(Q)])
            res["runs"].append(_run(index, qr, k, w, dict(set="self_exclusion", Q=Q, allowed=n - 1)))
            print(json.dumps(res["runs"][-1]), flush=True)
            row = _run(index, qr, k, None, dict(set="none_rows_as_queries", Q=Q))
            res["runs"].append(row)
            print(json.dumps(row), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
