"""Teacher-forced fp64 reference of every layer of the extraction network, and the per-element error bound its fp16
outputs are held to.

Every check reads the GPU's own fp16 input of a launch (a debug tap, see ``dirb200_net_debug_stage``) and never its
own earlier outputs, so errors cannot compound and a failure names exactly one launch.  The parameters are rebuilt
bit for bit as the host code packs them (``net.cu``, ``pack_conv`` and the fused-shortcut fold): fp16 weights
``fl16(W)``, BatchNorm folded in fp32, ``s = fl32(g / sqrtf(fl32(v + 1e-5f)))``, ``t = fl32(b - fl32(m * s))``.

For a convolution with exact value ``e = sum a*w`` (fp64), magnitude ``m = sum |a|*|w|`` and epilogue
``y = relu(s*e + t (+ res))`` the GPU's fp16 output must satisfy, element by element::

    |y_gpu - y_ref| <= 1/2 ulp16(max(|y_gpu|, |y_ref|)) + KAPPA * 2^-23 * |s| * m + 2^-22 * (|s*e| + |t| + |res|)

The middle term is the fp32 tensor-core accumulation (it truncates, DESIGN section 2), the last one the epilogue's fp32
FMA and residual add.  KAPPA comes from the H100 (DESIGN section 2).  Every k16 step of the accumulation loses less
than 2^-23 * m, so a launch with S steps is held to min(KAPPA, S): the rigorous bound where it is the tighter one.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

import synthdata as synth
from oracle import dir_oracle as O

F64 = torch.float64
KAPPA = 18.2    # 2 x the largest accumulation-error ratio measured on the H100 over the whole matrix (DESIGN section 2)
OLD_REL_TOL = 2e-3   # the operator tests' former global tolerance: 2e-3 * max(1, max|y|)


# --------------------------------------------------------------------------- rounding helpers
def fl16(x: torch.Tensor) -> torch.Tensor:
    """Round fp32-exact values to fp16 (round to nearest even) and back to x's dtype."""
    return x.float().half().to(x.dtype)


def ulp16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of the fp16 numbers at |v|: 2^(floor(log2|v|) - 10), and 2^-24 in the subnormal range."""
    a = v.abs().to(F64)
    _, ex = torch.frexp(a)
    u = torch.ldexp(torch.ones_like(a), (ex - 11).to(torch.int32))
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), u)


def bn_fold(sd, bn, cout):
    """(scale, shift) fp32 numpy arrays exactly as pack_conv folds eval-mode BatchNorm; bn None -> (1, 0)."""
    if bn is None:
        return np.ones(cout, np.float32), np.zeros(cout, np.float32)
    g, b, m, v = (np.asarray(sd[bn + k], dtype=np.float32) for k in (".weight", ".bias", ".running_mean", ".running_var"))
    s = (g / np.sqrt(v + np.float32(1e-5))).astype(np.float32)
    t = (b - (m * s).astype(np.float32)).astype(np.float32)
    return s, t


def w16(w) -> torch.Tensor:
    """fl16 of an OIHW fp32 weight, as fp64."""
    return torch.as_tensor(np.asarray(w, dtype=np.float32)).half().to(F64)


def fused_shortcut_params(sd, prefix):
    """Block 0's fused conv3 + projection shortcut as the host folds it: fl16(fl32(s3*W3)), fl16(fl32(sd*Wd)), scale 1,
    shift fl32(t3 + td)."""
    w3 = np.asarray(sd[prefix + "conv3.weight"], np.float32)
    wd = np.asarray(sd[prefix + "downsample.0.weight"], np.float32)
    s3, t3 = bn_fold(sd, prefix + "bn3", w3.shape[0])
    sdn, tdn = bn_fold(sd, prefix + "downsample.1", wd.shape[0])
    a = torch.from_numpy((s3[:, None, None, None] * w3).astype(np.float32)).half().to(F64)
    b = torch.from_numpy((sdn[:, None, None, None] * wd).astype(np.float32)).half().to(F64)
    return a, b, np.ones_like(s3), (t3 + tdn).astype(np.float32)


def stem_input_u8(u8: np.ndarray, mean=synth.RGB_MEANS, std=synth.RGB_STDS) -> torch.Tensor:
    """(B,H,W,3) uint8 -> NCHW fp16 values of s2d_u8_kernel: fl16(fl32(fl32(fl32(px / 255) - mean) / std))."""
    x = u8.astype(np.float32).transpose(0, 3, 1, 2)
    m = np.asarray(mean, np.float32).reshape(1, 3, 1, 1)
    s = np.asarray(std, np.float32).reshape(1, 3, 1, 1)
    v = ((x / np.float32(255.0)).astype(np.float32) - m).astype(np.float32) / s
    return torch.from_numpy(np.ascontiguousarray(v.astype(np.float32))).half()


# --------------------------------------------------------------------------- reference values and the bound
def conv_em(a_nhwc: torch.Tensor, w: torch.Tensor, stride: int, pad: int):
    """Exact value e = sum a*w and magnitude m = sum |a|*|w| of a convolution in fp64, NHWC in and out."""
    x = a_nhwc.to(device=w.device, dtype=F64).permute(0, 3, 1, 2)
    e = F.conv2d(x, w, None, stride=stride, padding=pad)
    m = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=pad)
    return e.permute(0, 2, 3, 1), m.permute(0, 2, 3, 1)


@dataclass
class Report:
    """Outcome of one element-bound check: elements, failures, the largest accumulation-error ratio
    (|d| - 1/2 ulp16 - epilogue term) / (2^-23 |s| m), elements equal to fl16(y_ref), and where the worst element sits."""
    name: str
    n: int
    n_fail: int
    kappa_max: float
    exact: int
    worst: str = ""
    fail_tiles: list = field(default_factory=list)

    @property
    def ok(self):
        return self.n_fail == 0


def _where(idx, shape):
    """(n, y, x, c) of a flat NHWC index, with the 128-row tile of the flat pixel index and the 64-channel block."""
    n_, h, w, c = shape
    ci = idx % c
    p = idx // c
    x = p % w
    y = (p // w) % h
    n = p // (w * h)
    return (int(n), int(y), int(x), int(ci)), int(p // 128), int(ci // 64)


def k16_steps(cin, kh=1, kw=1):
    """k16 steps of a convolution's K loop: K = kh * kw * Cin (Cin padded to 8) padded to 32, as pack_conv lays it out."""
    return -(-kh * kw * (-(-cin // 8) * 8) // 32) * 2


def check_elements(name, y_gpu, e, m, s, t, res=None, relu=True, kappa=None, mask=None, steps=None) -> Report:
    """Hold y_gpu (NHWC, any float dtype) to the element bound against relu(s*e + t (+ res)); s, t per channel (fp32
    values); kappa None = KAPPA, capped at the launch's k16 steps when given.  mask (N,H,W bool): inside it the bound,
    outside it y_gpu must be exactly 0."""
    kappa = KAPPA if kappa is None else kappa
    if steps is not None:
        kappa = min(kappa, steps)
    dev = e.device
    yg = y_gpu.to(device=dev, dtype=F64)
    s_ = torch.as_tensor(np.asarray(s, np.float32)).to(dev, F64)
    t_ = torch.as_tensor(np.asarray(t, np.float32)).to(dev, F64)
    se = e * s_
    z = se + t_
    last = se.abs() + t_.abs()
    if res is not None:
        r = res.to(device=dev, dtype=F64)
        z = z + r
        last = last + r.abs()
        del r
    yr = torch.relu(z) if relu else z
    del z
    d = (yg - yr).abs()
    half = 0.5 * ulp16(torch.maximum(yg.abs(), yr.abs()))
    last = last * 2.0 ** -22
    acc = (2.0 ** -23) * s_.abs() * m
    slack = d - half - last
    bad = ~(slack <= kappa * acc)            # NaN / inf fail too
    exact = (yg == fl16(yr))
    ratio = torch.where(acc > 0, slack / torch.where(acc > 0, acc, torch.ones_like(acc)),
                        torch.where(slack > 0, torch.full_like(acc, math.inf), torch.full_like(acc, -math.inf)))
    if mask is not None:
        mk = mask.to(dev)[..., None].expand_as(yg)
        bad = torch.where(mk, bad, yg != 0)
        exact = exact & mk
        ratio = torch.where(mk, ratio, torch.full_like(ratio, -math.inf))
        n = int(mk.sum())
    else:
        n = yg.numel()
    n_fail = int(bad.sum())
    kmax = float(ratio.max()) if ratio.numel() else -math.inf
    worst, tiles = "", []
    if n_fail:
        flat = torch.nonzero(bad.reshape(-1)).reshape(-1)
        i = int(flat[torch.argmax(d.reshape(-1)[flat])])
        (nn, yy, xx, cc), tile, cb = _where(i, yg.shape)
        worst = ("worst failing element n=%d y=%d x=%d c=%d (pixel tile %d of 128 rows, channel block %d): gpu %.8g ref %.8g "
                 "bound %.3g" % (nn, yy, xx, cc, tile, cb, float(yg.reshape(-1)[i]), float(yr.reshape(-1)[i]),
                                 float((half + last + kappa * acc).reshape(-1)[i])))
        per_pix = bad.reshape(-1, yg.shape[-1])
        rows = torch.nonzero(per_pix.any(1)).reshape(-1)
        tiles = sorted(set(int(v) // 128 for v in rows.tolist()))
        worst += "; %d failing pixel tiles, first %s" % (len(tiles), tiles[:8])
    return Report(name, n, n_fail, kmax, int(exact.sum()), worst, tiles)


def old_tolerance_passes(y_gpu, y_ref) -> bool:
    """The operator tests' former check: max |y_gpu - y_ref| < 2e-3 * max(1, max |y_ref|)."""
    y_gpu = y_gpu.to(F64)
    y_ref = y_ref.to(device=y_gpu.device, dtype=F64)
    return float((y_gpu - y_ref).abs().max()) < OLD_REL_TOL * max(1.0, float(y_ref.abs().max()))


def check_conv(name, y_gpu, a, w, stride, pad, s, t, res=None, relu=True, kappa=None, mask=None, device=None) -> Report:
    """One convolution launch: fp16 input a (NHWC), fp32 OIHW weight w (fl16 here), folded BN (s, t)."""
    dev = device or (y_gpu.device if y_gpu.is_cuda else torch.device("cpu"))
    e, m = conv_em(a, w16(w).to(dev), stride, pad)
    steps = k16_steps(w.shape[1], w.shape[2], w.shape[3])
    return check_elements(name, y_gpu, e, m, s, t, res=res, relu=relu, kappa=kappa, mask=mask, steps=steps)


# --------------------------------------------------------------------------- exact operators
def maxpool_ref(stem_conv: torch.Tensor) -> torch.Tensor:
    """3x3/s2/p1 max of the fp16 stem output (NHWC), -inf padding: exact."""
    x = stem_conv.float().permute(0, 3, 1, 2)
    return F.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1).half()


def upsample_add_ref(x4: torch.Tensor, lat: torch.Tensor) -> torch.Tensor:
    """fl16(fp32(x4) + fp32(lat[nearest])), nearest index as F.interpolate(mode='nearest') computes it."""
    n, h, w, c = lat.shape
    idx = torch.arange(h * w, dtype=torch.float32, device=lat.device).view(1, 1, h, w)
    up = F.interpolate(idx, size=x4.shape[1:3], mode="nearest").long().view(-1)
    g = lat.reshape(n, h * w, c)[:, up].reshape(x4.shape)
    return (x4.float() + g.float()).half()


# --------------------------------------------------------------------------- the network, launch by launch
def _blocks(arch):
    from dirb200 import nets
    trunk, fpn, mode = nets._ARCH[arch]
    blocks, exp = nets._TRUNKS[trunk]
    return blocks, exp, fpn, mode


def expected_launches(arch, fuse_ds=True, conv_impl=0, fpn_mode=None):
    """Every convolution launch of one forward (fuse_c23 0) as the output tap it writes, from the block structure of
    nets._TRUNKS: 'stem_conv', per block conv1 / conv2 / down (unless fused) / the block output, the FPN convolutions."""
    blocks, exp, fpn, mode = _blocks(arch)
    mode = mode if fpn_mode is None else fpn_mode
    fused = exp == 4 and fuse_ds and conv_impl == 0
    names = ["stem_conv"]
    inplanes = 64
    for li, nb in enumerate(blocks, start=1):
        planes = 64 << (li - 1)
        for b in range(nb):
            p = "layer%d.%d" % (li, b)
            stride = 2 if (li > 1 and b == 0) else 1
            has_down = b == 0 and (stride != 1 or inplanes != planes * exp)
            names.append(p + ".conv1")
            if exp == 4:
                names.append(p + ".conv2")
            if has_down and not fused:
                names.append(p + ".down")
            names.append(p)
            inplanes = planes * exp
    if fpn and mode == 1:
        names += ["fpn_lat", "fpn_c4"]
    return names


def check_network(tap, sd, arch, x16, *, fuse_ds=True, conv_impl=0, kappa=None, device="cuda", masks=None):
    """Check every launch of the last forward from its taps.  tap(name) -> NHWC fp16 tensor; x16: the stem's fp16
    input (NCHW); masks: {(H, W): (N,H,W) bool} extents of a ragged batch per map size.  -> (reports, exact_ok) where
    exact_ok lists the exact operators (maxpool, upsample-add) that matched."""
    blocks, exp, fpn, mode = _blocks(arch)
    fused = exp == 4 and fuse_ds and conv_impl == 0
    dev = torch.device(device)
    reps, exact = [], []

    def mk(y):
        return None if masks is None else masks[tuple(y.shape[1:3])]

    def conv(name, a, wname, stride, pad, bn, res=None, relu=True):
        y = tap(name)
        w = sd[wname]
        s, t = bn_fold(sd, bn, w.shape[0])
        reps.append(check_conv(name, y, a, w, stride, pad, s, t, res=res, relu=relu, kappa=kappa, mask=mk(y), device=dev))
        return y

    conv("stem_conv", x16.permute(0, 2, 3, 1), "conv1.weight", 2, 3, "bn1")
    sc = tap("stem_conv")
    pooled = tap("stem")
    ref = maxpool_ref(sc)
    if masks is not None:
        ref = torch.where(mk(pooled).to(ref.device)[..., None], ref, torch.zeros_like(ref))
    assert torch.equal(pooled, ref.to(pooled.device)), "maxpool != max of the stem_conv tap"
    exact.append("stem")
    x = pooled
    inplanes = 64
    for li, nb in enumerate(blocks, start=1):
        planes = 64 << (li - 1)
        for b in range(nb):
            p = "layer%d.%d" % (li, b)
            q = p + "."
            stride = 2 if (li > 1 and b == 0) else 1
            has_down = b == 0 and (stride != 1 or inplanes != planes * exp)
            if exp == 1:
                t1 = conv(p + ".conv1", x, q + "conv1.weight", stride, 1, q + "bn1")
                res = conv(p + ".down", x, q + "downsample.0.weight", stride, 0, q + "downsample.1", relu=False) if has_down else x
                y = conv(p, t1, q + "conv2.weight", 1, 1, q + "bn2", res=res)
            else:
                t1 = conv(p + ".conv1", x, q + "conv1.weight", 1, 0, q + "bn1")
                t2 = conv(p + ".conv2", t1, q + "conv2.weight", stride, 1, q + "bn2")
                if has_down and fused:
                    y = tap(p)
                    wa, wb, s1, sh = fused_shortcut_params(sd, q)
                    e, m = conv_em(t2, wa.to(dev), 1, 0)
                    e2, m2 = conv_em(x, wb.to(dev), stride, 0)
                    e += e2
                    m += m2
                    del e2, m2
                    reps.append(check_elements(p, y, e, m, s1, sh, kappa=kappa, mask=mk(y),
                                               steps=k16_steps(wa.shape[1]) + k16_steps(wb.shape[1])))
                    del e, m
                else:
                    res = conv(p + ".down", x, q + "downsample.0.weight", stride, 0, q + "downsample.1", relu=False) if has_down else x
                    y = conv(p, t2, q + "conv3.weight", 1, 0, q + "bn3", res=res)
            x = y
            inplanes = planes * exp
        if li < 4:
            assert torch.equal(tap("layer%d" % li), x), "stage tap layer%d != its last block" % li
    assert torch.equal(tap("layer4"), x)
    if fpn and mode == 1:
        lat = conv("fpn_lat", x, "conv1x5.weight", 1, 0, None)
        merged = tap("fpn_merge")
        assert torch.equal(merged, upsample_add_ref(tap("layer3"), lat).to(merged.device)), "fpn_merge != upsample-add"
        exact.append("fpn_merge")
        conv("fpn_c4", merged, "conv3c4.weight", 1, 1, None)
    return reps, exact


def fused_shortcut_ulps(tap, sd, prefix, stride, device="cuda"):
    """Block-0 output vs the unfolded arithmetic in fp64 - fp16 W3 and Wd, fp32 (s3, sd) applied after the sums,
    relu(s3*e3 + t3 + sd*ed + td) - from the block's own conv2 tap and input tap: max |y - y_exact| in units of
    ulp16(max(|y|, |y_exact|))."""
    dev = torch.device(device)
    L, B = prefix.split(".")[0], int(prefix.split(".")[1])
    li = int(L[5:])
    inp = tap("stem" if li == 1 else "layer%d" % (li - 1)) if B == 0 else tap("%s.%d" % (L, B - 1))
    q = prefix + "."
    e3, _ = conv_em(tap(prefix + ".conv2"), w16(sd[q + "conv3.weight"]).to(dev), 1, 0)
    ed, _ = conv_em(inp, w16(sd[q + "downsample.0.weight"]).to(dev), stride, 0)
    s3, t3 = bn_fold(sd, q + "bn3", e3.shape[-1])
    sdn, tdn = bn_fold(sd, q + "downsample.1", e3.shape[-1])
    c = lambda v: torch.as_tensor(v).to(dev, F64)
    ye = torch.relu(c(s3) * e3 + c(t3) + c(sdn) * ed + c(tdn))
    y = tap(prefix).to(dev, F64)
    return float(((y - ye).abs() / ulp16(torch.maximum(y.abs(), ye.abs()))).max())


# --------------------------------------------------------------------------- trained-like weights
def trunk_walk(x, sd, arch, hook=None):
    """The oracle's trunk (oracle.dir_oracle.bottleneck / basic_block) launch by launch: hook(tap, bn, conv_in,
    conv_out) may replace each convolution's output before its BatchNorm.  -> (layer4 map, {'layer1'..'layer4': maps})."""
    blocks, exp, _, _ = _blocks(arch)

    def cbn(tapname, wname, bn, a, stride, pad, relu=True):
        y = F.conv2d(a, sd[wname], None, stride=stride, padding=pad)
        if hook is not None:
            y = hook(tapname, bn, a, y)
        y = O._bn(y, sd, bn)
        return F.relu(y) if relu else y

    x = F.max_pool2d(cbn("stem_conv", "conv1.weight", "bn1", x, 2, 3), 3, 2, 1)
    stages = {}
    inplanes = 64
    for li, nb in enumerate(blocks, start=1):
        planes = 64 << (li - 1)
        for b in range(nb):
            p = "layer%d.%d" % (li, b)
            q = p + "."
            stride = 2 if (li > 1 and b == 0) else 1
            has_down = b == 0 and (stride != 1 or inplanes != planes * exp)
            if exp == 1:
                out = cbn(p + ".conv1", q + "conv1.weight", q + "bn1", x, stride, 1)
                out = cbn(p + ".conv2", q + "conv2.weight", q + "bn2", out, 1, 1, relu=False)
            else:
                out = cbn(p + ".conv1", q + "conv1.weight", q + "bn1", x, 1, 0)
                out = cbn(p + ".conv2", q + "conv2.weight", q + "bn2", out, stride, 1)
                out = cbn(p + ".conv3", q + "conv3.weight", q + "bn3", out, 1, 0, relu=False)
            if has_down:
                x = cbn(p + ".down", q + "downsample.0.weight", q + "downsample.1", x, stride, 0, relu=False)
            x = F.relu(out + x)
            inplanes = planes * exp
        stages["layer%d" % li] = x
    return x, stages


@functools.lru_cache(maxsize=4)
def _trained_like(arch, seed):
    sd = synth.make_state_dict(arch, seed=seed)
    for k in sorted(sd):
        if k.endswith(".weight") and sd[k].dim() == 4:
            r = synth._rs(seed + 1, k + ".scale")
            sc = np.exp(r.uniform(math.log(0.1), math.log(10.0), sd[k].shape[0])).astype(np.float32)
            sd[k] = sd[k] * torch.from_numpy(sc).view(-1, 1, 1, 1)

    def calibrate(tapname, bn, a, y):
        # running statistics = the batch statistics of this convolution's output, as a trained BatchNorm holds them
        c = y.shape[1]
        r = synth._rs(seed + 1, bn + ".affine")
        g = np.exp(r.uniform(math.log(1e-4), math.log(2.0), c))
        g[r.uniform(0, 1, c) < 0.05] = 0.0
        sd[bn + ".running_mean"] = y.mean(dim=(0, 2, 3)).float()
        sd[bn + ".running_var"] = y.var(dim=(0, 2, 3), unbiased=False).float()
        sd[bn + ".weight"] = torch.from_numpy(g.astype(np.float32))
        sd[bn + ".bias"] = torch.from_numpy((0.5 * r.standard_normal(c)).astype(np.float32))
        return y

    with torch.no_grad():
        trunk_walk(synth.make_images(2, 160, 160, seed=seed + 2), sd, arch, hook=calibrate)
    return sd


def make_trained_like_state_dict(arch="resnet50_rmac", seed=0) -> dict:
    """State dict with a trained network's dynamic range: per-output-channel conv weight scales log-uniform over
    [0.1, 10]; every BatchNorm's running mean / variance calibrated to the batch statistics of its convolution's output
    on seeded images (the oracle's own activations, layer by layer); gamma log-uniform over [1e-4, 2] with ~5 % exact
    zeros; beta ~ N(0, 0.5).  Deterministic from the seed."""
    return {k: v.clone() for k, v in _trained_like(arch, seed).items()}
