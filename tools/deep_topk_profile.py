"""Queries/s and search phase profile of the exact top-k at depths on both sides of the shallow / deep finish
(k = 100, 1024, 1025, 4096, 16384), 1000 and 70 queries on a 1M x 2048 database, one GPU.

    python tools/deep_topk_profile.py OUT.json

Timed: CUDA events around `steps` searches after `warmup` searches of the same shape (profile option off); then one
more search with option "profile" for the phase split.  rescore_gbs = bytes of fp32 rows the exact re-scoring
gathers (survivors x D x 4) over the time of that phase: with the HBM bandwidth it tells whether the gather bounds it."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from dirb200 import ops  # noqa: E402

N, D = 1_000_000, 2048
KS = (100, 1024, 1025, 4096, 16384)
QS = (1000, 70)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    name, power, clock = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main(path, steps=5, warmup=2):
    g = torch.Generator(device="cuda").manual_seed(1)
    db, db16 = ops.l2_normalize(torch.randn((N, D), generator=g, device="cuda"), want_f16=True)
    qall = ops.l2_normalize(torch.randn((max(QS), D), generator=g, device="cuda"))
    idx = ops.Index(db, db16=db16)
    rows = []
    for Q in QS:
        q = qall[:Q].contiguous()
        for k in KS:
            for _ in range(warmup):
                idx.search(q, k)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                idx.search(q, k)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / steps
            idx.set_option("profile", 1)
            idx.search(q, k)
            prof = idx.profile()
            idx.set_option("profile", 0)
            st = idx.stats()
            r = {"Q": Q, "k": k, "ms_per_search": ms, "queries_per_s": Q / (ms * 1e-3), "profile_ms": prof, "stats": st,
                 "q_block": idx.search_max_queries(k)}
            if "finish_rescore" in prof and prof["finish_rescore"] > 0:
                r["rescore_gbs"] = st["survivors"] * D * 4 / (prof["finish_rescore"] * 1e-3) / 1e9
            print(json.dumps(r), flush=True)
            rows.append(r)
    res = {"card": card(), "database": "%d x %d fp32 + fp16, unit-norm Gaussian rows" % (N, D), "steps": steps,
           "warmup": warmup, "runs": rows}
    with open(path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "deep_topk.json")
