"""GPU JPEG decoding (ops.JpegDecoder) against PIL decoding, decode-only and end to end.

Corpus: seeded photo-like images (smooth structure + texture + noise) in the Oxford-like size mix of
tools/ragged_profile.py, written as q90 4:2:0 baseline JPEGs at run time.  Reported, with the card name and power limit
read in the same run:
  - GPU decode-only images/s and MP/s over the corpus in calls of 64 files (host clock around synchronised work, after
    a warm-up pass over every file), and the per-phase kernel times of one pass from torch.profiler (separate pass);
  - the PIL loader's decode-only rate (pipeline._RawImages without a source) with 1, 8 and 16 workers, capped at the
    core count;
  - extract_image_features end to end on ResNet-101 (synthetic weights), chain '', batch 1 and 16, with GPU and with
    PIL decoding (pipeline.GPU_JPEG), the modes alternating over the rounds.

    python tools/jpeg_profile.py --out results/h100_jpeg.json
"""
import argparse
import io
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
sys.path.insert(0, os.path.join(REPO, "tools"))

PHASES = {"unstuff": ("unstuff_kernel",), "sync": ("sync_init_kernel", "sync_round_kernel"),
          "decode": ("count_kernel", "scan_check_kernel", "write_kernel"), "dc_scan": ("dc_kernel",),
          "idct": ("idct_kernel",), "color": ("color_kernel",)}


def photo_like(h, w, rng):
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.zeros((h, w, 3), np.float32)
    for _ in range(6):
        f = rng.uniform(0.5, 12, 2) / np.array([h, w])
        ph = rng.uniform(0, 6.28, 3)
        amp = rng.uniform(10, 50)
        a += amp * np.sin(6.28 * (f[0] * y + f[1] * x)[..., None] + ph)
    a += rng.normal(0, 6, a.shape)
    return np.clip(a + 128, 0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="results/h100_jpeg.json")
    ap.add_argument("--files", type=int, default=192)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    from PIL import Image
    import synthdata as synth
    from ragged_profile import oxford_like_sizes
    from dirb200 import datasets, nets, ops, pipeline
    ops.require_gpu(0)
    out = {}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out["gpu_name_power_limit_max_sm_clock"] = q.stdout.strip()
    out["cpu_cores"] = os.cpu_count()
    rng = np.random.default_rng(args.seed)
    sizes = oxford_like_sizes(args.files, args.seed)
    files = []
    for h, w in sizes:
        b = io.BytesIO()
        Image.fromarray(photo_like(h, w, rng)).save(b, "JPEG", quality=90, subsampling=2)
        files.append(b.getvalue())
    mp = sum(h * w for h, w in sizes) / 1e6
    out["corpus"] = dict(files=args.files, megapixels=mp, mean_kib=float(np.mean([len(f) for f in files]) / 1024),
                         quality=90, subsampling="4:2:0")

    # ---- GPU decode only
    dec = ops.JpegDecoder(0)
    batches = [files[i:i + 64] for i in range(0, len(files), 64)]

    def gpu_pass():
        for b in batches:
            imgs, ok = dec.decode(b)
            assert all(ok)
        torch.cuda.synchronize()

    gpu_pass()
    t = []
    for _ in range(3):
        t0 = time.perf_counter()
        gpu_pass()
        t.append(time.perf_counter() - t0)
    tm = float(np.median(t))
    out["gpu_decode"] = dict(batch=64, seconds_all=t, images_per_s=args.files / tm, megapixels_per_s=mp / tm,
                             sync_rounds_last_call=dec.last_rounds)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gpu_pass()
    phase_ms = {k: 0.0 for k in PHASES}
    for e in prof.key_averages():
        for k, names in PHASES.items():
            if any(n in e.key for n in names):
                phase_ms[k] += e.device_time_total / 1000.0
    out["gpu_decode"]["kernel_ms_per_pass"] = phase_ms

    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, "jpg"))
        names = []
        for i, f in enumerate(files):
            names.append("im%04d.jpg" % i)
            with open(os.path.join(root, "jpg", names[-1]), "wb") as fh:
                fh.write(f)
        ds = datasets.ImageList(imgs=names, root=os.path.join(root, "jpg"))
        # ---- PIL loader, decode only
        loader_rates = {}
        for nw in sorted({min(1, os.cpu_count()), min(8, os.cpu_count()), min(16, os.cpu_count())}):
            loader = torch.utils.data.DataLoader(pipeline._RawImages(ds), batch_size=None, shuffle=False,
                                                 num_workers=nw if nw > 1 else 0, pin_memory=True)
            for _ in loader:
                pass
            t0 = time.perf_counter()
            for _ in loader:
                pass
            loader_rates["workers_%d" % nw] = args.files / (time.perf_counter() - t0)
        out["pil_loader_decode_images_per_s"] = loader_rates
        # ---- end to end
        net = nets.create_model("resnet101_rmac")
        net.load_state_dict(synth.make_state_dict("resnet101_rmac", seed=0))
        net.eval()
        threads = min(16, os.cpu_count() or 1)
        e2e = {"loader_threads": threads}
        for gpu in (True, False):                                   # warm-up of every mode
            pipeline.GPU_JPEG = gpu
            for bs in (1, 16):
                pipeline.extract_image_features(ds, "", net, threads=threads, batch_size=bs, desc="warm")
        ref = None
        for _ in range(args.rounds):
            for gpu in (True, False):
                pipeline.GPU_JPEG = gpu
                for bs in (1, 16):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    d = pipeline.extract_image_features(ds, "", net, threads=threads, batch_size=bs, desc="e2e")
                    torch.cuda.synchronize()
                    key = "%s_decode_batch_%d_images_per_s" % ("gpu" if gpu else "pil", bs)
                    e2e.setdefault(key, []).append(args.files / (time.perf_counter() - t0))
                    if ref is None:
                        ref = d
                    assert torch.equal(d, ref)
        pipeline.GPU_JPEG = True
        out["extract_image_features_r101"] = e2e
        out["descriptors_identical_across_modes"] = True
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
