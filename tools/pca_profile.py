"""Timing of the GPU PCA fit (whitening.fit_pca) at D = 2048: the Gram kernel, the column sums, the host eigh, the fit
end to end from a device tensor and from a descriptor store, and sklearn's own PCA(whiten=True).fit as the baseline.

    python tools/pca_profile.py OUT.json

Kernel times: CUDA events around `reps` calls after one warm-up call of the same shape (each call = the split-K tile
kernel + the ordered reduction, or the two column-sum kernels).  gram_tflops = the useful flops of the computed
(upper-triangle) 128 x 128 tiles, 2 N x tiles x 128^2, over the Gram time.  The bound is the fp64 tensor-core (DMMA)
rate: 67 TFLOP/s on NVIDIA's H100 SXM data sheet at 700 W.  The card's name, power limit and SM clocks are read in the
same run, after the timings.  fit_pca times are one call each, after one warm-up fit, from the host clock around the
call (which ends with the statistics on the host); they include the host eigh."""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dirb200 import ops, store, whitening  # noqa: E402

D = 2048
NS = (5063, 100000, 1000000)
GT = 128


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    name, power, clock, max_clock = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_after_run": clock, "max_sm_clock": max_clock}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main(path):
    ops.require_gpu(0)
    whitening.fit_pca(torch.randn((4096, D), device="cuda"))      # module load, scratch, sklearn import, eigh warm-up
    g = torch.Generator(device="cuda").manual_seed(5)
    t = -(-D // GT)
    tiles = t * (t + 1) // 2
    rows = []
    for n in NS:
        x = (torch.randn((n, D), generator=g, device="cuda") * 0.05 + 0.01).contiguous()
        reps = 5 if n >= 1000000 else 20
        sums = torch.zeros(D, dtype=torch.float64, device="cuda")
        gram = torch.zeros((D, D), dtype=torch.float64, device="cuda")
        ms_sums = timed(lambda: ops.col_sums_f64(x, sums), reps)
        mean = (ops.col_sums_f64(x) / n).contiguous()
        ms_gram = timed(lambda: ops.gram_f64(x, mean, gram), reps)
        useful = 2.0 * n * tiles * GT * GT
        ms_fit, _ = wall(lambda: whitening.fit_pca(x))
        r = {"N": n, "D": D, "col_sums_ms": ms_sums, "col_sums_gbs": n * D * 4 / (ms_sums * 1e-3) / 1e9,
             "gram_ms": ms_gram, "gram_useful_tflop": useful / 1e12, "gram_tflops": useful / (ms_gram * 1e-3) / 1e12,
             "gram_share_of_dmma_peak_67": useful / (ms_gram * 1e-3) / 67e12, "fit_pca_device_ms": ms_fit}
        if n == 100000:
            xh = x.cpu().numpy()
            with tempfile.TemporaryDirectory() as tmp:
                st = store.write_store(os.path.join(tmp, "st"), xh)
                r["fit_pca_store_ms"], _ = wall(lambda: whitening.fit_pca(st))
            from sklearn.decomposition import PCA
            t0 = time.perf_counter()
            p = PCA(whiten=True).fit(xh)
            r["sklearn_fit_ms"] = (time.perf_counter() - t0) * 1e3
            r["sklearn_solver"] = p._fit_svd_solver
            r["sklearn_host_threads"] = os.cpu_count()
            del xh
        print(json.dumps(r), flush=True)
        rows.append(r)
        del x, gram
    cov = np.cov(np.random.RandomState(0).standard_normal((4 * D, D)), rowvar=False)
    np.linalg.eigh(cov)
    t0 = time.perf_counter()
    for _ in range(3):
        np.linalg.eigh(cov)
    eigh_ms = (time.perf_counter() - t0) / 3 * 1e3
    res = {"card": card(), "data": "N x 2048 fp32 Gaussian rows on the device", "host_eigh_ms_D2048": eigh_ms,
           "host_cpus": os.cpu_count(), "runs": rows}
    print(json.dumps(res["card"]), "eigh %.1f ms" % eigh_ms)
    with open(path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "pca_profile.json")
