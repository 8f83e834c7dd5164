"""CPU tests of the per-layer element bound of tests/layer_model.py: an emulated correct kernel passes it, each of a
list of plausible kernel bugs fails it (several of which the former 2e-3 * max tolerance accepts), and a localized bug
in one layer3 convolution that moves the descriptor by less than the 1e-3 descriptor bar is flagged per layer."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_model as LM
import synthdata as synth
from oracle import dir_oracle as O
from conftest import rel_l2


# --------------------------------------------------------------------------- a numpy model of the tensor-core kernel
def _trunc32(v):
    """fp64 -> fp32 rounded toward zero (the tensor cores' accumulation)."""
    r = v.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(v)
    r[over] = np.nextafter(r[over], np.float32(0))
    return r


def _f16(v):
    return v.astype(np.float32).astype(np.float16).astype(np.float64)


def emulate(A, W, s, t, res=None, relu=True, drop=None, f16_kblock=None, s_f16=None):
    """Implicit GEMM of fp16 operands A (P x K) and W (Cout x K): fp32 accumulation in k16 steps with truncation toward
    zero, epilogue fl32(fma(acc, s, t)) (+ res) (relu) -> fp16.  Mutations: drop = (k16 step, pixel tile, channel block)
    skipped for one 128 x 64 tile; f16_kblock = a 64-wide K block accumulated in fp16; s_f16 = a channel whose BN scale
    is rounded to fp16."""
    P, K = A.shape
    acc = np.zeros((P, W.shape[0]), np.float32)
    for k in range(K // 16):
        part = A[:, 16 * k:16 * k + 16] @ W[:, 16 * k:16 * k + 16].T
        if drop is not None and drop[0] == k:
            part[128 * drop[1]:128 * drop[1] + 128, 64 * drop[2]:64 * drop[2] + 64] = 0.0
        if f16_kblock is not None and k // 4 == f16_kblock:
            acc = _f16(acc.astype(np.float64) + part).astype(np.float32)
        else:
            acc = _trunc32(acc.astype(np.float64) + part)
    s = np.asarray(s, np.float32).copy()
    if s_f16 is not None:
        s[s_f16] = np.float32(np.float16(s[s_f16]))
    z = (acc.astype(np.float64) * s + np.asarray(t, np.float64)).astype(np.float32)
    if res is not None:
        z = (z.astype(np.float64) + res).astype(np.float32)
    if relu:
        z = np.maximum(z, np.float32(0))
    return z.astype(np.float16)


def _layer(kind, seed=0):
    """A real layer shape on a few hundred pixels: conv3 of layer4 (1x1, K = 2048, residual) or conv2 of layer4
    (3x3, K = 4608).  -> dict with the fp16 input map, fp32 weight, (s, t), residual, im2col operands."""
    r = np.random.RandomState(seed)
    h, w, cout = 15, 20, 128
    if kind == "1x1_k2048":
        cin, k = 2048, 1
    else:
        cin, k = 512, 3
    a = torch.from_numpy(np.maximum(r.standard_normal((1, h, w, cin)), 0).astype(np.float32)).half()
    wt = (r.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    s = r.uniform(0.2, 1.5, cout).astype(np.float32)
    t = (0.3 * r.standard_normal(cout)).astype(np.float32)
    res = torch.from_numpy(r.standard_normal((1, h, w, cout)).astype(np.float32)).half() if k == 1 else None
    cols = F.unfold(a.double().permute(0, 3, 1, 2), k, padding=k // 2)[0].T.numpy()     # (P, cin*k*k), OIHW order
    W16 = LM.w16(wt).reshape(cout, -1).numpy()
    return dict(a=a, w=wt, s=s, t=t, res=res, A=cols, W=W16, k=k, shape=(1, h, w, cout))


def _run(L, **mut):
    res = None if L["res"] is None else L["res"].double().reshape(-1, L["shape"][3]).numpy()
    y = emulate(L["A"], L["W"], L["s"], L["t"], res=res, **mut)
    return torch.from_numpy(y.reshape(L["shape"]))


def _check(L, y, kappa=None):
    return LM.check_conv("emulated", y, L["a"], L["w"], 1, L["k"] // 2, L["s"], L["t"], res=L["res"], kappa=kappa,
                         device=torch.device("cpu"))


def _yref(L):
    e, _ = LM.conv_em(L["a"], LM.w16(L["w"]), 1, L["k"] // 2)
    z = e * torch.from_numpy(L["s"]).double() + torch.from_numpy(L["t"]).double()
    if L["res"] is not None:
        z = z + L["res"].double()
    return torch.relu(z)


LAYERS = ["1x1_k2048", "3x3_k4608"]


@pytest.fixture(scope="module", params=LAYERS)
def layer(request):
    return request.param, _layer(request.param)


def test_emulated_correct_kernel_passes(layer):
    name, L = layer
    rep = _check(L, _run(L))
    print("%s: emulated kernel kappa_max %.3f, exact %.4f" % (name, rep.kappa_max, rep.exact / rep.n))
    assert rep.ok, rep.worst
    assert rep.kappa_max <= LM.KAPPA
    K = L["A"].shape[1]
    assert LM.KAPPA <= K / 16 / 5           # far below one full truncation per k16 step


def _mutations(L):
    """name -> mutated fp16 output of the emulated kernel."""
    good = _run(L)
    yref = _yref(L)
    out = {}
    # one element moved by 1 ulp16 away from the exact value, where the half-ulp term dominates the bound
    g = good.double()
    acc = 2.0 ** -23 * torch.from_numpy(L["s"]).double().abs() * LM.conv_em(L["a"], LM.w16(L["w"]), 1, L["k"] // 2)[1]
    margin = 0.5 * LM.ulp16(g) - LM.KAPPA * acc - 2.0 ** -22 * (g.abs() + 2.0)
    margin[g == 0] = -1
    i = int(torch.argmax(margin.reshape(-1)))
    y = good.clone().reshape(-1)
    v = float(y[i])
    step = float(LM.ulp16(torch.tensor(v)))
    y[i] = v + step if v >= float(yref.reshape(-1)[i]) else v - step
    out["one_ulp"] = y.reshape(good.shape)
    out["k16_step_dropped_in_one_tile"] = _run(L, drop=(5, 1, 1))
    sc = L["s"]
    c = int(np.argmax(np.abs(sc.astype(np.float16).astype(np.float64) - sc) / sc))
    out["bn_scale_in_fp16_one_channel"] = _run(L, s_f16=c)
    if L["res"] is not None:
        Lr = dict(L)
        r = L["res"].clone().reshape(-1, L["shape"][3])
        r[:128] = torch.cat([r[1:129]])                   # tile 0 reads the next pixel's residual
        Lr["res"] = r.reshape(L["res"].shape)
        out["residual_from_neighbour_pixel"] = _run(Lr)
    y = good.clone().reshape(-1, L["shape"][3])
    P = y.shape[0]
    t0 = (P - 1) // 128 * 128                             # the ragged last tile
    y[t0 + 1:] = y[t0:P - 1].clone()
    out["edge_tile_shifted_one_pixel"] = y.reshape(good.shape)
    out["k_block_accumulated_in_fp16"] = _run(L, f16_kblock=3)
    return out, yref


@pytest.fixture(scope="module")
def mutated(layer):
    name, L = layer
    return name, L, _mutations(L)


def test_each_mutation_fails_the_bound(mutated):
    name, L, (muts, _) = mutated
    for mname, y in muts.items():
        rep = _check(L, y)
        print("%s / %s: %d elements fail, %s" % (name, mname, rep.n_fail, rep.worst))
        assert not rep.ok, mname
    rep = _check(L, muts["k16_step_dropped_in_one_tile"])
    assert rep.fail_tiles == [1]                           # the report names the tile


def test_old_tolerance_misses_mutations_the_bound_catches(mutated):
    """Blind spot of the former operator tolerance 2e-3 * max(1, max|y|): these bugs pass it."""
    name, L, (muts, yref) = mutated
    passed_old = sorted(m for m, y in muts.items() if LM.old_tolerance_passes(y, yref))
    print("%s: mutations the old tolerance accepts: %s" % (name, passed_old))
    assert {"one_ulp", "bn_scale_in_fp16_one_channel", "k_block_accumulated_in_fp16"} <= set(passed_old)


# --------------------------------------------------------------------------- the descriptor bar's blind spot
def _tile_mutation(a, w, kind):
    """Change of a 1x1 convolution's output (NCHW, fp64) by a bug confined to pixel tile 0 (pixels 0..127) and channel
    block 0: 'k16_step_dropped' (K channels 0..15 left out) or 'k_block_accumulated_in_fp16' (the accumulator held in
    fp16 through the last 64-channel K block, four k16 steps)."""
    a, w = a.double(), w.double()
    if kind == "k16_step_dropped":
        d = -F.conv2d(a[:, :16], w[:64, :16])
    else:
        k0 = a.shape[1] - 64
        full = F.conv2d(a, w[:64])
        parts = [F.conv2d(a[:, k0 + 16 * i:k0 + 16 * i + 16], w[:64, k0 + 16 * i:k0 + 16 * i + 16]) for i in range(4)]
        acc = full - sum(parts)
        for p in parts:
            acc = LM.fl16(acc + p)
        d = acc - full
    n, _, h, wd = d.shape
    mask = torch.zeros(h * wd, dtype=d.dtype)
    mask[:128] = 1
    out = torch.zeros(n, w.shape[0], h, wd, dtype=d.dtype)
    out[:, :64] = d * mask.view(1, 1, h, wd)
    return out


@pytest.mark.parametrize("kind", ["k16_step_dropped", "k_block_accumulated_in_fp16"])
def test_descriptor_bar_vs_a_localized_layer3_bug(kind):
    """On the oracle (R50, 224^2, one image: layer3 maps of 14 x 14): a bug in one 128-pixel x 64-channel tile of
    layer3.1.conv1 (1x1, K = 1024).  The per-layer check of that launch fails and names the tile.  A dropped k16 step
    moves the descriptor by several times the 1e-3 bar, so the descriptor check catches it too; a 64-wide K block
    accumulated in fp16 moves it by less than 1e-3: only the per-layer check sees it."""
    sd = synth.make_state_dict("resnet50_rmac", seed=0)
    x = synth.make_images(1, 224, 224, seed=77)
    target = "layer3.1.conv1"
    w = sd[target + ".weight"]
    seen = {}

    def hook(tap, bn, a, y):
        if tap == target:
            seen["a"] = a.clone()
            return y + _tile_mutation(a, w, kind).to(y.dtype)
        return y

    with torch.no_grad():
        ref = O.head(LM.trunk_walk(x, sd, "resnet50_rmac")[0], sd)
        mut = O.head(LM.trunk_walk(x, sd, "resnet50_rmac", hook=hook)[0], sd)
    moved = rel_l2(mut.numpy(), ref.numpy())
    print("%s in one tile of %s: descriptor moved by %.3e" % (kind, target, moved))
    if kind == "k16_step_dropped":
        assert moved > 1e-3
    else:
        assert 0 < moved < 1e-3
    # the same bug as that launch's tap would show it, against the teacher-forced reference
    a16 = seen["a"].half().permute(0, 2, 3, 1)
    s, t = LM.bn_fold(sd, "layer3.1.bn1", w.shape[0])
    e, m = LM.conv_em(a16, LM.w16(w), 1, 0)
    d = _tile_mutation(a16.permute(0, 3, 1, 2), LM.w16(w), kind).permute(0, 2, 3, 1)
    st = lambda v: torch.from_numpy(v).double()
    good = LM.check_elements(target, LM.fl16(torch.relu(e * st(s) + st(t))), e, m, s, t)
    bad = LM.check_elements(target, LM.fl16(torch.relu((e + d) * st(s) + st(t))), e, m, s, t)
    print("  per-layer check: %d elements fail; %s" % (bad.n_fail, bad.worst))
    assert good.ok and not bad.ok and bad.fail_tiles == [0]


# --------------------------------------------------------------------------- the network walk itself
def _emulated_taps(sd, arch, x16, fuse_ds=True, bad=None):
    """Taps of a forward whose every launch is exact up to the final fp16 rounding (fp64 arithmetic); bad = a tap name
    whose pixel tile 0 is off by 1 %."""
    blocks, exp, fpn, mode = LM._blocks(arch)
    taps = {}

    def conv(name, a, wname, stride, pad, bn, res=None, relu=True, w=None, st=None):
        e, _ = LM.conv_em(a, LM.w16(sd[wname]) if w is None else w, stride, pad)
        s, t = LM.bn_fold(sd, bn, e.shape[-1]) if st is None else st
        z = e * torch.from_numpy(s).double() + torch.from_numpy(t).double()
        if res is not None:
            z = z + res.double()
        y = LM.fl16(torch.relu(z) if relu else z).half()
        if name == bad:
            y.reshape(-1, y.shape[-1])[:128] *= 1.01
        taps[name] = y
        return y

    sc = conv("stem_conv", x16.permute(0, 2, 3, 1), "conv1.weight", 2, 3, "bn1")
    x = taps["stem"] = LM.maxpool_ref(sc)
    inplanes = 64
    for li, nb in enumerate(blocks, start=1):
        planes = 64 << (li - 1)
        for b in range(nb):
            p, q = "layer%d.%d" % (li, b), "layer%d.%d." % (li, b)
            stride = 2 if (li > 1 and b == 0) else 1
            has_down = b == 0 and (stride != 1 or inplanes != planes * exp)
            if exp == 1:
                t1 = conv(p + ".conv1", x, q + "conv1.weight", stride, 1, q + "bn1")
                r = conv(p + ".down", x, q + "downsample.0.weight", stride, 0, q + "downsample.1", relu=False) if has_down else x
                x = conv(p, t1, q + "conv2.weight", 1, 1, q + "bn2", res=r)
            else:
                t1 = conv(p + ".conv1", x, q + "conv1.weight", 1, 0, q + "bn1")
                t2 = conv(p + ".conv2", t1, q + "conv2.weight", stride, 1, q + "bn2")
                if has_down and fuse_ds:
                    wa, wb, s1, sh = LM.fused_shortcut_params(sd, q)
                    e1, _ = LM.conv_em(t2, wa, 1, 0)
                    e2, _ = LM.conv_em(x, wb, stride, 0)
                    x = taps[p] = LM.fl16(torch.relu(e1 + e2 + torch.from_numpy(sh).double())).half()
                else:
                    r = conv(p + ".down", x, q + "downsample.0.weight", stride, 0, q + "downsample.1", relu=False) if has_down else x
                    x = conv(p, t2, q + "conv3.weight", 1, 0, q + "bn3", res=r)
            inplanes = planes * exp
        taps["layer%d" % li] = x
    if fpn and mode == 1:
        lat = conv("fpn_lat", x, "conv1x5.weight", 1, 0, None)
        taps["fpn_merge"] = LM.upsample_add_ref(taps["layer3"], lat)
        conv("fpn_c4", taps["fpn_merge"], "conv3c4.weight", 1, 1, None)
    return taps


@pytest.mark.parametrize("arch,fuse_ds", [("resnet50_rmac", True), ("resnet50_rmac", False), ("resnet18_rmac", True),
                                          ("resnet50_fpn_rmac", True)])
def test_walk_checks_every_launch(arch, fuse_ds):
    """check_network visits every launch expected_launches lists (from nets._TRUNKS), passes an exact forward and names
    the one launch and tile that is off."""
    sd = synth.make_state_dict(arch, seed=1)
    x16 = synth.make_images(1, 64, 96, seed=3).half()
    taps = _emulated_taps(sd, arch, x16, fuse_ds)
    reps, exact = LM.check_network(taps.__getitem__, sd, arch, x16, fuse_ds=fuse_ds, device="cpu")
    assert [r.name for r in reps] == LM.expected_launches(arch, fuse_ds=fuse_ds)
    assert all(r.ok for r in reps)
    nb = sum(LM._blocks(arch)[0])
    n_down = 4 if arch.startswith("resnet50") else 3
    per_block = 2 if arch.startswith("resnet18") else 3
    assert len(reps) == 1 + per_block * nb + (0 if fuse_ds and per_block == 3 else n_down) + (2 if "_fpn" in arch else 0)
    bad = "layer2.1.conv1"
    reps, _ = LM.check_network(_emulated_taps(sd, arch, x16, fuse_ds, bad=bad).__getitem__, sd, arch, x16,
                               fuse_ds=fuse_ds, device="cpu")
    assert [r.name for r in reps if not r.ok] == [bad]


def test_trained_like_state_dict():
    """Deterministic; gammas over [1e-4, 2] with exact zeros; running statistics calibrated to the conv outputs (the
    oracle's BN output of the calibration images has per-channel mean beta)."""
    a = LM.make_trained_like_state_dict("resnet50_rmac", seed=3)
    b = LM.make_trained_like_state_dict("resnet50_rmac", seed=3)
    assert all(torch.equal(a[k], b[k]) for k in a)
    g = torch.cat([v for k, v in a.items() if k.endswith(".weight") and v.dim() == 1])
    assert float(g.max()) <= 2.0 and float(g[g > 0].min()) >= 1e-4
    assert 0.02 < float((g == 0).float().mean()) < 0.08
    assert float(g[g > 0].min()) < 1e-3
    assert torch.isfinite(torch.stack([v.float().abs().max() for v in a.values() if v.is_floating_point()])).all()
