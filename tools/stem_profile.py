"""Stem timing: the fused stem (one kernel: space-to-depth, 7x7/s2 convolution, BN + ReLU, 3x3/s2 max-pool) against the
three-launch path (s2d_kernel, the wgmma convolution, maxpool_kernel), for fp32 NCHW and uint8 HWC input.

Both are timed inside a ResNet-50 forward (synthetic weights) with the network's per-launch CUDA events (option
"profile" 2, accumulated over --reps forwards after --warmup untimed ones), so they run at the batch and chunk sizes
the network gives them and after the same predecessor kernels.  Reported per shape and input: ms per forward of the
stem launches, the rate over the stem's real 7x7x3 FLOPs, the bytes the fused kernel needs (images in, pooled map out)
over its time.  Card name and power limit are read in the same run.

    python tools/stem_profile.py --out results/h100_stem.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

SHAPES = [(64, 1024, 1024), (16, 1434, 1434), (1, 1024, 1024)]


def stem_ms(net, x, u8, warmup, reps):
    """ms per forward of the launches up to and including the max-pool (the fused one, or s2d + conv + maxpool)."""
    fwd = net.forward_u8 if u8 else net.forward
    for _ in range(warmup):
        fwd(x)
    torch.cuda.synchronize()
    net.set_backend_option_live("profile", 2)
    for _ in range(reps):
        fwd(x)
    torch.cuda.synchronize()
    rows = [r for r in net.profile_table() if r["tag"].startswith("stem") or r["tag"].startswith("maxpool")]
    net.set_backend_option_live("profile", 0)
    return sum(r["ms"] for r in rows) / reps, [(r["tag"], round(r["ms"] / reps, 4)) for r in rows]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="results/h100_stem.json")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import synthdata as synth
    from dirb200 import nets, ops
    ops.require_gpu(0)
    out = {}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out["gpu_name_power_limit_max_sm_clock"] = q.stdout.strip()
    sd = synth.make_state_dict("resnet50_rmac", seed=0)
    handles = {}
    for fuse in (1, 0):
        net = nets.create_model("resnet50_rmac")
        net.load_state_dict(sd)
        net.set_backend_option("fuse_stem", fuse)
        handles[fuse] = net.eval()
    res = []
    for (b, h, w) in SHAPES:
        for u8 in (False, True):
            if u8:
                x = torch.from_numpy(synth.make_images_u8(b, h, w, seed=1)).cuda()
            else:
                x = synth.make_images(b, h, w, seed=1).cuda()
            ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            hp, wp = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
            flops = 2.0 * b * ho * wo * 64 * 147
            need = b * ((3.0 if u8 else 12.0) * h * w + 128.0 * hp * wp)
            row = {"B": b, "H": h, "W": w, "input": "uint8 HWC" if u8 else "fp32 NCHW"}
            for fuse in (1, 0):
                ms, tags = stem_ms(handles[fuse], x, u8, args.warmup, args.reps)
                key = "fused" if fuse else "unfused"
                row[key] = {"ms": round(ms, 4), "tflops_real_k147": round(flops / ms / 1e9, 1),
                            "needed_bytes_tb_s": round(need / ms / 1e9, 3), "launches": tags}
            row["speedup"] = round(row["unfused"]["ms"] / row["fused"]["ms"], 2)
            print(json.dumps(row), flush=True)
            res.append(row)
            del x
            torch.cuda.empty_cache()
    out["rows"] = res
    out["note"] = ("per-launch CUDA events inside ResNet-50 forwards (option profile 2); fused = stem_pool_kernel, "
                   "unfused = s2d_kernel + conv_pers_kernel<64> + maxpool_kernel; tflops over the real K = 147, "
                   "needed bytes = images once + pooled map once")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu_name_power_limit_max_sm_clock"]}))


if __name__ == "__main__":
    main()
