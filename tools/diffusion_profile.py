"""Timings of diffusion re-ranking on one GPU -> results/h100_diffusion.json (or --out).

At D = 2048 and N = 5063 / 100k / 1M clustered unit rows, with Q = 70 and 1000 queries: the graph (the exact top-(k+1)
search of every row, then the CSR build), nnz, the CG solve per block and per iteration, the bytes one iteration needs
(from nnz and the block width Qb) over its time as a share of the H100 SXM's 3.35 TB/s, the dense-row rank counts, and
on the host's CPUs scipy's `cg` on the same systems at 5063 and 100k rows.  The card's name, power limit and max SM
clock are read in the same run.  Defaults: k 50, kq 10, gamma 3, alpha 0.99, 20 iterations (dirb200.diffusion)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dirb200  # noqa: E402,F401
from dirb200.diffusion import DEFAULTS, Diffusion, graph_from_knn  # noqa: E402

HBM = 3.35e12


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def _rows(n, d, seed, centres=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((max(2, n // 100) if centres is None else centres, d), generator=g, device="cuda")
    x = c[torch.randint(0, c.shape[0], (n,), generator=g, device="cuda")] + 0.6 * torch.randn((n, d), generator=g, device="cuda")
    return torch.nn.functional.normalize(x, dim=1).contiguous()


def _scipy_cg(d, q, p, nq):
    import scipy.sparse as sp
    import scipy.sparse.linalg as sla
    g = d.graph
    n = d.n
    S = sp.csr_matrix((g.val.cpu().numpy(), g.col.cpu().numpy(), g.row_ptr.cpu().numpy()), shape=(n, n))
    A = sp.identity(n, format="csr") - p["alpha"] * S
    sc, idx = d.index.search(q[:nq].contiguous(), p["kq"])
    sc, idx = sc.cpu().numpy(), idx.cpu().numpy()
    t = time.perf_counter()
    for i in range(nq):
        y = np.zeros(n)
        ok = idx[i] >= 0
        y[idx[i][ok]] = np.maximum(sc[i][ok], 0) ** p["gamma"]
        sla.cg(A, y, rtol=0.0, atol=0.0, maxiter=p["iters"])
    return (time.perf_counter() - t) / nq


def _rank_count_time(d, q, qb, n, per_query=50):
    """Time of dirb200_diffusion_rank_count over one solved block, per_query flagged targets per query."""
    import ctypes as C
    from dirb200 import lib, ops
    _, f, _, _ = next(d._blocks(q, DEFAULTS["kq"], DEFAULTS["alpha"], DEFAULTS["iters"], DEFAULTS["tol"], qb))
    T = qb * per_query
    off = np.ascontiguousarray(np.arange(qb + 1) * per_query, np.int32)
    rows = np.random.RandomState(qb).randint(0, n, T).astype(np.int64)
    off_d, rows_d = torch.from_numpy(off).cuda(), torch.from_numpy(rows).cuda()
    flags_d = torch.ones(T, dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.raw("dirb200_diffusion_rank_count_workspace_bytes")(qb, T), dtype=torch.uint8, device="cuda")
    sc = torch.empty(T, dtype=torch.float64, device="cuda")
    ab = torch.empty(T, dtype=torch.int64, device="cuda")

    def call():
        lib.call("dirb200_diffusion_rank_count", ops._ptr(f), n, qb, off.ctypes.data_as(C.c_void_p), ops._ptr(off_d),
                 ops._ptr(rows_d), ops._ptr(flags_d), T, ops._ptr(ws), ops._ptr(sc), ops._ptr(ab), ops._stream())
    call()
    _, t = _timed(lambda: [call() for _ in range(10)])
    return t / 10


def run(sizes, queries, dim, out):
    p = dict(DEFAULTS)
    res = dict(card=_card(), params=p, dim=dim, hbm_bytes_per_s=HBM, cpu_count=os.cpu_count(), runs=[])
    for n in sizes:
        db = _rows(n, dim, 1)
        d0 = Diffusion(db[:64], k=p["k"])                   # warm the modules
        d0.solve(db[:2], iters=2)
        (sc, idx), t_knn = _timed(lambda: d0.index.__class__(db).search(db, p["k"] + 1))
        g, t_csr = _timed(lambda: graph_from_knn(idx, sc, p["k"], p["gamma"]))
        d = Diffusion(db, k=p["k"], knn=(sc, idx))
        del sc, idx
        nnz = int(g.row_ptr[-1])
        entry = dict(n=n, knn_s=t_knn, csr_s=t_csr, graph_s=t_knn + t_csr, nnz=nnz, solves=[])
        for nq in queries:
            q = _rows(nq, dim, 2 + nq, centres=max(2, n // 100))
            qb = d.query_block(nq)
            d.solve(q[:qb], q_block=qb)                    # warm-up of this block width
            _, t_solve = _timed(lambda: d.solve(q))
            _, t_one = _timed(lambda: d.solve(q[:qb], q_block=qb, iters=1))
            _, t_full = _timed(lambda: d.solve(q[:qb], q_block=qb))
            per_iter = (t_full - t_one) / (p["iters"] - 1)
            spmm_bytes = nnz * (8 + 4) + (n + 1) * 8 + nnz * qb * 8 + 2 * n * qb * 8
            iter_bytes = spmm_bytes + 6 * n * qb * 8 + 3 * n * qb * 8
            t_rank = _rank_count_time(d, q[:qb], qb, n)
            entry["solves"].append(dict(q=nq, q_block=qb, blocks=-(-nq // qb), solve_s=t_solve,
                                        block_s=t_full, iter_s=per_iter, spmm_bytes_per_iter=spmm_bytes,
                                        iter_bytes=iter_bytes, iter_hbm_fraction=iter_bytes / per_iter / HBM,
                                        rank_count_block_s=t_rank))
            if n <= 100_000 and nq == queries[0]:
                entry["scipy_cg_s_per_query"] = _scipy_cg(d, q, p, min(nq, 10))
        res["runs"].append(entry)
        print(json.dumps(entry), flush=True)
        del d, d0, db, g
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[5063, 100_000, 1_000_000])
    ap.add_argument("--queries", type=int, nargs="+", default=[70, 1000])
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--out", default="results/h100_diffusion.json")
    a = ap.parse_args()
    run(a.sizes, a.queries, a.dim, a.out)
