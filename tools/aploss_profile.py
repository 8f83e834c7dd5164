"""Kernel times of the AP loss (csrc/aploss.cu) on the GPU, and the reference formulation for comparison.

    python tools/aploss_profile.py --out results/h100_aploss.json

Forward (histogram + finalisation) and backward times from CUDA events over --iters calls after warm-up, at
N = M in {4096, 16384}, nq in {25, 100}, uniform and concentrated scores, bool labels.  Bytes: N M (4 + 1) read by the
forward; N M (4 + 1 + 4) read and written by the backward; plus the histogram and the coefficients.  The reference
formulation (a 1x1 Conv1d over x.unsqueeze(1), loss.py:43-65, restated in plain torch, TF32 off) is timed at
N = M = 4096, nq = 25; at 16384 its Conv1d output alone is given from the shapes, and it is not run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from dirb200 import ops  # noqa: E402
from dirb200.loss import quantizer_table  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters * 1e-3


def scores(N, nq, kind, gen):
    x = torch.rand((N, N), device="cuda", generator=gen)
    if kind == "concentrated":      # 99 % inside one bin
        x = (nq // 3 + 0.3 + 0.2 * (x - 0.5)) / (nq - 1)
        x = 1 - x
        o = torch.rand((N, N), device="cuda", generator=gen) < 0.01
        x[o] = torch.rand(int(o.sum()), device="cuda", generator=gen)
    lab = torch.rand((N, N), device="cuda", generator=gen) < 0.01
    return x.contiguous(), lab


def reference_formulation(x, lab, nq):
    """loss.py:43-65 in plain torch: Conv1d quantiser, min / clamp, sums, cumsum, AP; forward + backward."""
    t = quantizer_table(nq, 0, 1).cuda()
    w, b = t[:2 * nq].view(2 * nq, 1, 1), t[2 * nq:]
    x = x.detach().requires_grad_(True)
    q = F.conv1d(x.unsqueeze(1), w, b)
    q = torch.min(q[:, :nq], q[:, nq:]).clamp(min=0)
    nbs = q.sum(-1)
    rec = (q * lab.view(x.shape[0], 1, -1).float()).sum(-1)
    prec = rec.cumsum(-1) / (1e-16 + nbs.cumsum(-1))
    rec = rec / rec.sum(-1, keepdim=True)
    loss = 1 - (prec * rec).sum(-1).mean()
    loss.backward()
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(REPO, "results", "h100_aploss.json"))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"card": card(), "iters": args.iters, "hbm_bytes_per_s": HBM, "rows": []}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for N in (4096, 16384):
        for nq in (25, 100):
            t = quantizer_table(nq, 0, 1).cuda()
            for kind in ("uniform", "concentrated"):
                x, lab = scores(N, nq, kind, gen)
                lab8 = lab.view(torch.uint8)
                _, G, apv = ops.aploss_forward(x, lab8, nq, t, "ap")
                g = torch.full((N,), -1.0 / N, device="cuda")
                tf = timed(lambda: ops.aploss_forward(x, lab8, nq, t, "ap"), args.iters)
                tb = timed(lambda: ops.aploss_backward(x, lab8, nq, t, G, g), args.iters)
                small = N * (2 * nq + 1) * 8 + N * 2 * nq * 8
                bf = N * N * 5 + small
                bb = N * N * 9 + N * 2 * nq * 8
                res["rows"].append({"N": N, "M": N, "nq": nq, "scores": kind, "fwd_s": tf, "bwd_s": tb,
                                    "fwd_bytes": bf, "bwd_bytes": bb, "fwd_bw": bf / tf, "bwd_bw": bb / tb,
                                    "fwd_hbm_share": bf / tf / HBM, "bwd_hbm_share": bb / tb / HBM})
                print(res["rows"][-1], flush=True)
                del x, lab, lab8, G, apv, g, _
                torch.cuda.empty_cache()
    # the reference formulation at 4096 / 25
    N, nq = 4096, 25
    x, lab = scores(N, nq, "uniform", gen)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    reference_formulation(x, lab, nq)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    tr = timed(lambda: reference_formulation(x, lab, nq), 5, warmup=1)
    # the kernels on the same inputs: everything they allocate (hist, G, ap, dx) is held to the end of the window,
    # and nothing allocated before it is freed inside it
    t = quantizer_table(nq, 0, 1).cuda()
    lab8 = lab.view(torch.uint8)
    grad_ap = torch.ones(N, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    hist, G, apv = ops.aploss_forward(x, lab8, nq, t, "ap")
    dx = ops.aploss_backward(x, lab8, nq, t, G, grad_ap)
    torch.cuda.synchronize()
    peak_k = torch.cuda.max_memory_allocated() - base
    shapes_k = sum(v.numel() * v.element_size() for v in (hist, G, apv, dx))
    assert peak_k >= shapes_k, (peak_k, shapes_k)
    res["reference_formulation"] = {
        "N": N, "M": N, "nq": nq, "fwd_bwd_s": tr, "peak_bytes_above_inputs": peak,
        "kernels_peak_bytes_above_inputs": peak_k, "kernels_output_bytes_from_shapes": shapes_k,
        "conv_output_bytes_at_16384_nq25": 16384 * 2 * 25 * 16384 * 4,
        "conv_output_bytes_at_16384_nq100": 16384 * 2 * 100 * 16384 * 4,
        "note": "at N = M = 16384 the reference formulation is not run: its Conv1d output alone exceeds 80 GB"}
    print(res["reference_formulation"])
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
