"""Timings of truncated diffusion on one GPU -> results/h100_diffusion_trunc.json (or --out).

The setup of tools/diffusion_profile.py: D = 2048 clustered unit rows, N = 5063 / 100k / 1M, Q = 70 and 1000 queries,
defaults k 50, kq 10, gamma 3, alpha 0.99, 20 iterations.  For m = 500 / 1000 / 2000 / 5000 (m <= N), CUDA events
time, over the whole query set in the blocks ws_budget allows: the exact top-m search, the local build
(dirb200_diffusion_trunc_build), the fused CG (dirb200_diffusion_trunc_solve) and the rule-T6 ordering of the m rows
(dirb200_diffusion_trunc_topk at k = 100), each summed over the blocks; the full solve of the same queries over the
whole graph (Diffusion.solve) is timed in the same run alongside.  The card's name, power limit and max SM clock are
read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dirb200  # noqa: E402,F401
from dirb200 import lib, ops  # noqa: E402
from dirb200.diffusion import DEFAULTS, Diffusion  # noqa: E402
from dirb200.inputs import rows64  # noqa: E402


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def _rows(n, d, seed, centres=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((max(2, n // 100) if centres is None else centres, d), generator=g, device="cuda")
    x = c[torch.randint(0, c.shape[0], (n,), generator=g, device="cuda")] + 0.6 * torch.randn((n, d), generator=g, device="cuda")
    return torch.nn.functional.normalize(x, dim=1).contiguous()


class _Clock:
    """Sums CUDA-event intervals per stage."""
    def __init__(self):
        self.marks = []

    def mark(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.marks.append((name, e))

    def totals(self):
        torch.cuda.synchronize()
        out = {}
        for (_, a), (name, b) in zip(self.marks, self.marks[1:]):
            out[name] = out.get(name, 0.0) + a.elapsed_time(b) / 1e3
        return out


def _truncated(d, q, m, topk, p):
    """The four stages of search(q, topk, truncate=m), each timed with events over all blocks."""
    mm = min(m, d.n)
    qs = rows64(q)
    nq, kw = qs.shape[0], d.ell
    depth = max(topk, mm)
    qb = d.trunc_query_block(nq, mm, depth)
    g, w = d.graph, d.weights
    ck = _Clock()
    ck.mark("start")
    for q0 in range(0, nq, qb):
        qc = qs[q0:q0 + qb].contiguous()
        b = qc.shape[0]
        sc, idx = d.index.search(qc, depth)
        li, ls = idx[:, :mm].contiguous(), sc[:, :mm].contiguous()
        ck.mark("search_s")
        loc = [torch.empty((b, mm), dtype=torch.int64, device="cuda"), torch.empty((b, mm), dtype=torch.int32, device="cuda"),
               torch.empty((b, kw, mm), dtype=torch.int32, device="cuda"),
               torch.empty((b, kw, mm), dtype=torch.float64, device="cuda")] + \
              [torch.empty((b, mm), dtype=torch.float64, device="cuda") for _ in range(3)]
        ws = torch.empty(lib.raw("dirb200_diffusion_trunc_build_workspace_bytes")(b, mm), dtype=torch.uint8, device="cuda")
        ck.mark("alloc_s")
        lib.call("dirb200_diffusion_trunc_build", ops._ptr(g.row_ptr), ops._ptr(g.col), ops._ptr(w.a), d.n, kw,
                 ops._ptr(li), ops._ptr(ls), b, mm, p["kq"], d.gamma, ops._ptr(ws), *(ops._ptr(t) for t in loc),
                 ops._stream())
        ck.mark("build_s")
        ws = torch.empty(lib.raw("dirb200_diffusion_trunc_solve_workspace_bytes")(b, mm), dtype=torch.uint8, device="cuda")
        f = torch.empty((b, mm), dtype=torch.float64, device="cuda")
        it = torch.empty(b, dtype=torch.int32, device="cuda")
        res = torch.empty(b, dtype=torch.float64, device="cuda")
        ck.mark("alloc_s")
        lib.call("dirb200_diffusion_trunc_solve", ops._ptr(loc[1]), ops._ptr(loc[2]), ops._ptr(loc[3]), kw,
                 ops._ptr(loc[6]), b, mm, p["alpha"], p["iters"], p["tol"], ops._ptr(ws), ops._ptr(f), ops._ptr(it),
                 ops._ptr(res), ops._stream())
        ck.mark("cg_s")
        ws = torch.empty(lib.raw("dirb200_diffusion_trunc_topk_workspace_bytes")(b, mm, topk), dtype=torch.uint8,
                         device="cuda")
        out_s = torch.empty((b, topk), dtype=torch.float64, device="cuda")
        out_i = torch.empty((b, topk), dtype=torch.int64, device="cuda")
        ck.mark("alloc_s")
        lib.call("dirb200_diffusion_trunc_topk", ops._ptr(loc[0]), ops._ptr(f), b, mm, ops._ptr(idx), ops._ptr(sc),
                 idx.shape[1], topk, ops._ptr(ws), ops._ptr(out_s), ops._ptr(out_i), ops._stream())
        ck.mark("rank_s")
        del loc, ws, f
    t = ck.totals()
    t["total_s"] = sum(t.values())
    return dict(m=m, m_eff=mm, q_block=qb, blocks=-(-nq // qb), ell_width=kw, **t)


def run(sizes, queries, ms, dim, topk, out):
    p = dict(DEFAULTS)
    res = dict(card=_card(), params=p, dim=dim, topk=topk, runs=[])
    for n in sizes:
        db = _rows(n, dim, 1)
        d0 = Diffusion(db[:512], k=p["k"], truncation=True)              # warm the modules
        d0.solve_truncated(db[:2], 100, iters=2)
        d0.search(db[:2], 10, truncate=100)
        d = Diffusion(db, k=p["k"], truncation=True)
        entry = dict(n=n, nnz=int(d.graph.row_ptr[-1]), solves=[])
        for nq in queries:
            q = _rows(nq, dim, 2 + nq, centres=max(2, n // 100))
            qb = d.query_block(nq)
            d.solve(q[:qb], q_block=qb, iters=2)                          # warm-up of the full solve
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            d.solve(q)
            s1.record()
            torch.cuda.synchronize()
            row = dict(q=nq, full_solve_s=s0.elapsed_time(s1) / 1e3, full_q_block=qb, truncated=[])
            for m in ms:
                if m > n:
                    continue
                _truncated(d, q[:min(nq, 8)], m, topk, p)                 # warm-up of these shapes
                row["truncated"].append(_truncated(d, q, m, topk, p))
            entry["solves"].append(row)
            print(json.dumps(dict(n=n, **row)), flush=True)
        res["runs"].append(entry)
        del d, d0, db
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[5063, 100_000, 1_000_000])
    ap.add_argument("--queries", type=int, nargs="+", default=[70, 1000])
    ap.add_argument("--m", type=int, nargs="+", default=[500, 1000, 2000, 5000])
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--topk", type=int, default=100)
    ap.add_argument("--out", default="results/h100_diffusion_trunc.json")
    a = ap.parse_args()
    run(a.sizes, a.queries, a.m, a.dim, a.topk, a.out)
