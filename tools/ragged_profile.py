"""Mixed-size extraction: one image per network call vs ragged batches (dirb200_net_forward_ragged_u8).

About 512 seeded uint8 images with an Oxford-like size mix (mostly 1024x768 and 768x1024, random aspect ratios with a
1024 long side, cropped queries), pre-decoded in pinned host memory, through ResNet-101 (synthetic weights).  Per mode
the timed pass is H2D copy + (slot packing) + forward for every image, host clock around work ending in a device
synchronise; the modes alternate over several rounds after a warm-up of each.  Reported: images/s, the padded-area
overhead of the ragged groups (sum B*H*W / sum h*w), "useful" TFLOP/s from the images' true sizes beside the FLOPs the
network counts over the slots.  Then extract_image_features end to end from PNG files (batch_size 1 vs 16) next to
the rate at which the loader alone decodes them.  Card name and power limit are read in the same run.

    python tools/ragged_profile.py --out results/h100_ragged.json
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


def oxford_like_sizes(n, seed):
    r = np.random.RandomState(seed)
    sizes = []
    for _ in range(n):
        u = r.rand()
        if u < 0.45:
            sizes.append((768, 1024))
        elif u < 0.7:
            sizes.append((1024, 768))
        elif u < 0.85:
            a = int(r.randint(500, 1024))
            sizes.append((a, 1024) if r.rand() < 0.5 else (1024, a))
        else:                                                   # query crops (bounding boxes)
            sizes.append((int(r.randint(150, 800)), int(r.randint(150, 800))))
    return sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="results/h100_ragged.json")
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--files", type=int, default=192, help="images written as PNG for the end-to-end extraction")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import synthdata as synth
    from dirb200 import datasets, nets, ops, pipeline
    ops.require_gpu(0)
    out = {}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out["gpu_name_power_limit_max_sm_clock"] = q.stdout.strip()

    net = nets.create_model("resnet101_rmac")
    net.load_state_dict(synth.make_state_dict("resnet101_rmac", seed=0))
    net.eval()
    sizes = oxford_like_sizes(args.n, args.seed)
    g = torch.Generator().manual_seed(args.seed)
    pool = torch.randint(0, 256, (1024 * 1024 * 3 + 4096,), dtype=torch.uint8, generator=g)
    imgs = []
    for i, (h, w) in enumerate(sizes):                          # seeded content, pinned host memory
        off = (i * 7919) % 4096
        imgs.append(pool[off:off + h * w * 3].view(h, w, 3).clone().pin_memory())
    true_px = sum(h * w for h, w in sizes)
    out["images"] = args.n
    out["size_mix"] = {"768x1024": sizes.count((768, 1024)), "1024x768": sizes.count((1024, 768)),
                       "other": args.n - sizes.count((768, 1024)) - sizes.count((1024, 768))}

    def per_image(subset):
        flops = 0.0
        for i in subset:
            d = net.forward_u8(imgs[i].cuda(non_blocking=True)[None])
            flops += net.last_launch_stats()[1]
        return flops

    def ragged(subset, bs):
        flops, slot_px = 0.0, 0
        win = pipeline.RAGGED_WINDOW * bs
        for w0 in range(0, len(subset), win):
            part = [imgs[i].cuda(non_blocking=True) for i in subset[w0:w0 + win]]
            hw = [(int(x.shape[0]), int(x.shape[1])) for x in part]
            for grp in pipeline.ragged_groups(hw, bs):
                hh, ww = max(hw[k][0] for k in grp), max(hw[k][1] for k in grp)
                slots = part[grp[0]].new_empty((len(grp), hh, ww, 3))
                for j, k in enumerate(grp):
                    slots[j, :hw[k][0], :hw[k][1]] = part[k]
                net.forward_ragged_slots(slots, [hw[k] for k in grp])
                flops += net.last_launch_stats()[1]
                slot_px += len(grp) * hh * ww
        return flops, slot_px

    modes = {"per_image": lambda s: (per_image(s), true_px)}
    for bs in (8, 16, 64):
        modes["ragged_%d" % bs] = (lambda b: (lambda s: ragged(s, b)))(bs)
    allidx = list(range(args.n))
    for name, fn in modes.items():                              # warm-up: every mode once over 64 images
        fn(allidx[:64])
    torch.cuda.synchronize()
    times = {k: [] for k in modes}
    stats = {}
    for _ in range(args.rounds):
        for name, fn in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn(allidx)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            stats[name] = res
    per_img_flops = stats["per_image"][0]                       # FLOPs of the images at their true sizes
    out["modes"] = {}
    for name in modes:
        t = float(np.median(times[name]))
        flops, px = stats[name]
        out["modes"][name] = dict(seconds_median=t, seconds_all=times[name], images_per_s=args.n / t,
                                  padded_area_overhead=px / true_px, useful_tflops=per_img_flops / t / 1e12,
                                  counted_tflops=flops / t / 1e12)
    out["speedup_ragged_16_vs_per_image"] = out["modes"]["ragged_16"]["images_per_s"] / out["modes"]["per_image"]["images_per_s"]

    # end to end from image files: decode (CPU loader workers) + GPU, '' chain
    from PIL import Image
    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, "jpg"))
        names = []
        for i in range(args.files):
            names.append("im%04d.png" % i)
            Image.fromarray(imgs[i].numpy()).save(os.path.join(root, "jpg", names[-1]), compress_level=1)
        ds = datasets.ImageList(imgs=names, root=os.path.join(root, "jpg"))
        threads = min(16, os.cpu_count() or 1)
        loader = torch.utils.data.DataLoader(pipeline._RawImages(ds), batch_size=None, shuffle=False,
                                             num_workers=threads, pin_memory=True)
        for _ in loader:                                        # warm the page cache and the workers' imports
            pass
        t0 = time.perf_counter()
        for _ in loader:
            pass
        decode = time.perf_counter() - t0
        e2e = {"files": args.files, "loader_threads": threads, "decode_only_images_per_s": args.files / decode}
        for bs in (1, 16, 1, 16):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipeline.extract_image_features(ds, "", net, threads=threads, batch_size=bs, desc="bs%d" % bs)
            torch.cuda.synchronize()
            e2e.setdefault("batch_size_%d_images_per_s" % bs, []).append(args.files / (time.perf_counter() - t0))
        out["extract_image_features"] = e2e
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
