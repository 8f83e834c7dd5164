"""Timings of the triangular self-join and the range search on one GPU -> results/h100_join.json (or --out).

Data: D = 2048 clustered unit rows generated on the GPU (the clusters of tools/diffusion_profile.py: one centre per 100
rows, per-entry noise 0.6, within-cluster scores ~0.74) with planted near-duplicate groups: 1 % of the rows are
replaced by copies of another row with per-entry noise 0.04 (scores ~0.998), in groups of 2 to 5.  For N = 100k and
1M and tau in {0.95, 0.8}: self_join(tau) with option profile = 1 (CUDA events per stage: filter passes, exact
re-scoring, sort + compaction, summed over the row blocks), then the connected components and groups (events around
ops.join_components / ops.join_groups), then range_search(X, tau) over the full square, whose filter passes run twice
the tensor-core tiles.  Issued TFLOP/s = 2 * 128 * 128 * D * tiles / filter time, against the 989 TFLOP/s of NVIDIA's
H100 SXM data sheet (dense fp16).  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dirb200  # noqa: E402,F401
from dirb200 import ops  # noqa: E402

PEAK_FP16 = 989e12


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
    n_dup = n // 100                                          # planted groups: copies of a source row, 1 to 4 each
    src = torch.randint(0, n, (n_dup // 3,), generator=g, device="cuda")
    reps = torch.randint(1, 5, (src.shape[0],), generator=g, device="cuda")
    src = torch.repeat_interleave(src, reps)[:n_dup]
    dst = torch.randperm(n, generator=g, device="cuda")[:src.shape[0]]
    keep = ~torch.isin(dst, src)
    x[dst[keep]] = x[src[keep]] + 0.04 * torch.randn((int(keep.sum()), d), generator=g, device="cuda")
    del c
    return torch.nn.functional.normalize(x, dim=1).contiguous()


def _events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def _run(idx, kind, x, tau, D):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = idx.self_join(tau) if kind == "self_join" else idx.range_search(x, tau)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = idx.join_stats()
    flops = 2.0 * 128 * 128 * D * st["tiles"]
    rec = dict(wall_s=wall, filter_s=st["filter_ms"] / 1e3, rescore_s=st["rescore_ms"] / 1e3,
               sort_s=st["sort_ms"] / 1e3, tiles=st["tiles"], filter_launches=st["filter_launches"],
               reruns=st["reruns"], candidates=st["candidates"], pairs=st["pairs"],
               issued_tflops=flops / max(st["filter_ms"], 1e-9) / 1e9,
               share_of_fp16_peak=flops / max(st["filter_ms"], 1e-9) * 1e3 / PEAK_FP16)
    rec["candidates_per_pair"] = st["candidates"] / max(st["pairs"], 1)
    return res, rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--taus", type=float, nargs="+", default=[0.95, 0.8])
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "results", "h100_join.json"))
    args = ap.parse_args()
    ops.require_gpu(0)
    out = dict(card=_card(), dim=args.dim, peak_fp16_tflops=PEAK_FP16 / 1e12, runs=[])
    warm = _rows(4096, args.dim, 1)                               # module load, first launches
    wi = ops.Index(warm)
    wi.self_join(0.9)
    wi.range_search(warm, 0.9)
    wi.close()
    for n in args.sizes:
        x = _rows(n, args.dim, 7)
        idx = ops.Index(x)
        idx.set_option("profile", 1)
        for tau in args.taus:
            (off, cols, _), rec = _run(idx, "self_join", x, tau, args.dim)
            labels, cc_ms = _events_ms(lambda: ops.join_components(off, cols, n))
            (goff, mem), gr_ms = _events_ms(lambda: ops.join_groups(labels))
            sizes = (goff[1:] - goff[:-1]).cpu()
            rec.update(components_s=cc_ms / 1e3, groups_s=gr_ms / 1e3, groups=int(sizes.numel()),
                       largest_group=int(sizes.max()) if sizes.numel() else 0)
            del off, cols, labels, goff, mem
            _, sq = _run(idx, "range_search", x, tau, args.dim)
            torch.cuda.empty_cache()
            run = dict(n=n, tau=tau, self_join=rec, range_search_square=sq,
                       triangle_share_of_square_filter_time=rec["filter_s"] / max(sq["filter_s"], 1e-12),
                       triangle_share_of_square_tiles=rec["tiles"] / max(sq["tiles"], 1))
            print(json.dumps(run))
            out["runs"].append(run)
        idx.close()
        del x
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
