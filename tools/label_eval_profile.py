"""Label-dataset evaluation on the GPU: threshold counts (dirb200_index_count_ge) vs the dense-score path.

A seeded class-structured set (Zipf class sizes from 2 to 2000, every image a query, as for Landmarks_clean) at
N = Q = 50k, D = 2048: CUDA-event times of the positives' exact scores, of Index.count_ge (fp64 tensor-core pass +
band + scan) with its achieved fp64 rate 2 Q N D / time against the 67 TFLOP/s of the H100 SXM data sheet, and of
the exact top-100.  Then eval_model end to end on both paths at N = Q = 20k in the same process, with the largest
difference between their APs.  Card name, power limit and SM clock are read in the same run.

    python tools/label_eval_profile.py --out results/
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

FP64_TC_PEAK = 67e12          # H100 SXM data sheet, dense fp64 tensor core


def zipf_classes(n, d, seed, lo=2, hi=2000, a=1.5, sigma=0.6):
    r = np.random.RandomState(seed)
    sizes = np.arange(lo, hi + 1)
    p = sizes ** -a
    p /= p.sum()
    cls = []
    while sum(cls) < n:
        cls.append(int(r.choice(sizes, p=p)))
    cls[-1] -= sum(cls) - n
    if cls[-1] < lo:
        cls[-2] += cls.pop()
    labels = np.repeat(np.arange(len(cls)), cls)
    r.shuffle(labels)
    g = torch.Generator(device="cuda").manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(len(cls), d, generator=g, device="cuda"), dim=1)
    x = centers[torch.from_numpy(labels).cuda()] + sigma * torch.randn(n, d, generator=g, device="cuda") * (8.0 / d ** 0.5)
    return torch.nn.functional.normalize(x, dim=1).contiguous(), ["c%d" % v for v in labels], cls


def timed(fn, reps=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()                                                   # warm-up
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3 / reps, out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default="results/")
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--n-e2e", type=int, default=20000)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from dirb200 import datasets as D
    from dirb200.dist import ShardedIndex, sort_thresholds
    from dirb200.pipeline import eval_model
    out = {"gpu": torch.cuda.get_device_name(0)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out["power_limit_sm_clock_max_clock"] = q.stdout.strip()

    # ---- kernel-level times at N = Q = 50k
    n, d = args.n, args.dim
    x, labels, cls = zipf_classes(n, d, args.seed)
    ds = D.ImageListLabels(imgs=["im%06d.jpg" % i for i in range(n)], labels=labels)
    t_off, t_rows, skip = ds.label_targets()
    T = int(t_off[-1])
    dev = x.device
    off_d = torch.from_numpy(t_off.astype(np.int32)).to(dev)
    rows_d = torch.from_numpy(t_rows).to(dev)
    skip_d = torch.from_numpy(skip).to(dev)
    t_q = torch.repeat_interleave(torch.arange(n, dtype=torch.int32, device=dev), (off_d[1:] - off_d[:-1]).long())
    index = ShardedIndex(x, 0)
    t_sc, sc = timed(lambda: index.local.target_scores(x, t_q, rows_d))
    thr = sort_thresholds(sc.float(), t_q)
    t_cnt, cnt = timed(lambda: index.local.count_ge(x, off_d, thr, skip_d), reps=3)
    stats = index.local.stats()
    t_top, _ = timed(lambda: [index.search(x[c:c + 4096], 100) for c in range(0, n, 4096)])
    flops = 2.0 * n * n * d
    out["kernel"] = dict(N=n, Q=n, D=d, classes=len(cls), class_size_max=max(cls), thresholds=T,
                         target_scores_s=t_sc, count_ge_s=t_cnt, count_ge_fp64_tflops=flops / t_cnt / 1e12,
                         count_ge_share_of_fp64_tc_peak=flops / t_cnt / FP64_TC_PEAK,
                         band_entries=stats["candidates"], fallback_queries=stats["retries"], top100_s=t_top)
    print(json.dumps(out["kernel"]), flush=True)
    del x, index, sc, thr, cnt, rows_d, t_q
    torch.cuda.empty_cache()

    # ---- eval_model end to end, both paths, at N = Q = 20k
    n2 = args.n_e2e
    x2, labels2, _ = zipf_classes(n2, d, args.seed + 1)
    ds2 = D.ImageListLabels(imgs=["im%06d.jpg" % i for i in range(n2)], labels=labels2)
    with tempfile.TemporaryDirectory() as tmp:
        np.save(os.path.join(tmp, "feats.bdescs.npy"), x2.cpu().numpy())
        del x2
        res = {}
        for name, dense in (("counts", False), ("dense", True)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[name] = eval_model(ds2, None, "", detailed=True, load_feats=tmp, dense_scores=dense)
            torch.cuda.synchronize()
            out.setdefault("e2e", {})["eval_model_%s_s" % name] = time.perf_counter() - t0
    out["e2e"]["N"] = out["e2e"]["Q"] = n2
    out["e2e"]["max_abs_AP_diff"] = float(np.max(np.abs(np.array(res["counts"]["APs"]) - np.array(res["dense"]["APs"]))))
    out["e2e"]["tops_equal"] = res["counts"]["tops"] == res["dense"]["tops"]
    out["e2e"]["mAP"] = res["counts"]["mAP"]
    print(json.dumps(out), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_label_eval.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
