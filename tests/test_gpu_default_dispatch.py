"""Which kernel each launch of the default forward runs, and an element-by-element check of the forwards where every
stage takes the fused conv3 + residual + next conv1 kernel (conv_c31).

The kernel of a launch depends on the batch, the map size and the SM count (net.cu: c31_taken, c23_taken,
halo_order_plain and the fused-shortcut condition; conv.cu: the tile width of conv_pers_any and the ping-pong rule of
launch_conv_pers).  `plan` mirrors those rules launch by launch.  Every GPU case runs with option "profile" 1 and asserts
that the tags and launch counts of profile_table() equal the plan before it checks a single element, so a changed
threshold cannot quietly move a case off the kernel it was written for.  A tag names the operation and its shape but
not the instantiation: ping-pong vs cooperative, the 64- or 128-channel tile, HALO vs tap-by-tap K order, the RAGGED
instantiation and the per-image K order are derived from the sizes and the device's SM count, as
test_gpu_conv_pingpong.py does.

The CPU tests (no marker) check the plan against the block structure and show that each check fails when it should:
an element just past its own bound, a nonzero element outside a picture, a census one launch off."""
import math
import time
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import layer_model as LM
import synthdata as synth
from test_gpu_layers import _head_check, _levels, _net, _report, _taps

DEV = "cuda:0"
gpu = pytest.mark.gpu


# --------------------------------------------------------------------------- the selection rules, mirrored
def _cdiv(a, b):
    return -(-a // b)


def level_sizes(H, W):
    """(h, w) of the resolution levels 0..6 (input, stem conv, maxpool, layer1..4), net.cu level_sizes."""
    out = [(H, W)]
    for lvl in range(1, 7):
        h, w = out[-1]
        if lvl != 3:                                    # layer1 keeps the maxpool's size
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out.append((h, w))
    return out


def pick_patch(B, Ho, Wo):
    """(tw, th, nb) output patch of a spatial conv_pers tile, conv.cu pick_patch."""
    best, bt, bh, bb, bscore = -1, 16, 8, 1, 1 << 30
    w = 1
    while w <= 128:
        h = 1
        while w * h <= 128:
            b = 128 // (w * h)
            if w <= 64 and h <= 64:
                tiles = _cdiv(Wo, w) * _cdiv(Ho, h) * _cdiv(B, b)
                pen = (w // h if w > h else h // w) + (1 if b > 1 else 0) + (4 if w < 8 else 0)
                if best < 0 or tiles < best or (tiles == best and pen < bscore):
                    best, bscore, bt, bh, bb = tiles, pen, w, h, b
            h *= 2
        w *= 2
    return bt, bh, bb


@dataclass(frozen=True)
class Launch:
    """One launch: its profile tag, the debug taps it writes, the kernel (instantiation) and its tile count.
    pp: ping-pong (True) or cooperative (False) consumer mode of the persistent convolution, None for other kernels."""
    tag: str
    writes: tuple
    kernel: str
    tiles: int = 0
    pp: bool = None
    ragged: bool = False
    last_rows: int = 0      # conv_c31: rows of the last 128-row tile

    def families(self):
        k = self.kernel
        if k.startswith("conv_c31") or k.startswith("conv_c23"):
            return {k[:-1] + (",RAGGED>" if self.ragged else ">")}
        out = {k}
        if self.pp is not None:
            out.add("ping-pong" if self.pp else "cooperative")
        if self.ragged and k.startswith("conv_pers"):
            out.add("conv_pers RAGGED")
        return out


# The kernel families the default configuration (fuse_c23 0, halo 1, fuse_ds 1, fused stem) can select for a
# Bottleneck network; each must run in at least one case checked element by element.
REQUIRED = {"stem_pool", "conv_pers flat", "conv_pers spatial", "conv_pers HALO", "conv_pers per-image K order",
            "conv_pers RAGGED", "ping-pong", "cooperative", "fused shortcut",
            "conv_c31<64>", "conv_c31<128>", "conv_c31<256>",
            "conv_c31<64,RAGGED>", "conv_c31<128,RAGGED>", "conv_c31<256,RAGGED>"}


def plan(arch, B, H, W, *, sms, hw=None, halo=1, fuse_ds=1, fuse_c23=0):
    """Every launch of one pass (chunk = B, conv_impl 0, fused stem) of a Bottleneck network without FPN over B
    images of H x W, or over B pictures of sizes hw in H x W slots (ragged), on a device with `sms` SMs."""
    blocks, exp, fpn, _ = LM._blocks(arch)
    assert exp == 4 and not fpn, "the mirror covers the Bottleneck networks without FPN"
    rag = hw is not None
    lv = level_sizes(H, W)
    pics = [level_sizes(h, w) for h, w in hw] if rag else []
    out = []

    def plain(h, w):                                    # halo_order_plain
        return bool(halo) and h >= 16 and w >= 8

    def c23_taken(b, h, w, cm):
        if not fuse_c23:
            return False
        sup = cm in (64, 128, 256) and h >= 16 and w >= 8
        return sup if fuse_c23 == 2 else sup and _cdiv(w, 8) * _cdiv(h, 16) * b >= 2 * sms

    def per_image_order(lvl, col, slot_order):
        """ext3: the pictures of a ragged pass disagree with the slot's K order (table column col at level lvl)."""
        if not rag:
            return False
        cm = 64 << max(0, lvl - 3)
        want = [plain(*p[lvl]) if col == 2 else (c23_taken(1, p[lvl][0], p[lvl][1], cm) or plain(*p[lvl])) for p in pics]
        return any(v != slot_order for v in want)

    def pers(tiles):
        return tiles >= 3 * min(tiles, sms)             # launch_conv_pers

    def conv(tap, k, stride, cin, cout, h, w, res, per_image=False):
        pad = (k - 1) // 2
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        m_tiles = _cdiv(B * ho * wo, 128)
        bn = 128 if cout % 128 == 0 and m_tiles * (cout // 128) >= sms else 64      # conv_pers_any
        if halo and not per_image and k == 3 and stride == 1 and h >= 16 and w >= 8:
            kind, tiles = "HALO", _cdiv(w, 8) * _cdiv(h, 16) * B
        elif k == 1 and stride == 1:
            kind, tiles = "flat", m_tiles
        else:
            tw, th, nb = (8, 16, 1) if per_image else pick_patch(B, ho, wo)
            kind, tiles = "per-image K order" if per_image else "spatial", _cdiv(wo, tw) * _cdiv(ho, th) * _cdiv(B, nb)
        tiles *= cout // bn
        tag = "%dx%d%s %d->%d%s @%dx%d" % (k, k, "/s2" if stride == 2 else "", cin, cout, " +res" if res else "", ho, wo)
        out.append(Launch(tag, (tap,), "conv_pers " + kind, tiles, pers(tiles), rag))

    out.append(Launch("stem 7x7/s2 3->64 + maxpool 3x3/s2 fused", ("stem_conv",), "stem_pool", ragged=rag))
    inplanes, t1_ready = 64, False
    for s, nb in enumerate(blocks, start=1):
        planes = 64 << (s - 1)
        cm, cout = planes, planes * 4
        lvl = 1 + s
        for j in range(nb):
            st = 2 if (s > 1 and j == 0) else 1
            has_down = j == 0
            lvl_in = lvl
            if st == 2:
                lvl = 2 + s
            (h, w), (h2, w2) = lv[lvl_in], lv[lvl]
            tp = "layer%d.%d" % (s, j)
            if not t1_ready:
                conv(tp + ".conv1", 1, 1, inplanes, cm, h, w, False)
            t1_ready = False
            c23 = not has_down and st == 1 and c23_taken(B, h, w, cm)
            per_image = st == 1 and per_image_order(lvl, 2 if has_down else 3, c23 or plain(h, w))
            if c23 and not per_image:
                tiles = _cdiv(w, 8) * _cdiv(h, 16) * B
                out.append(Launch("3x3 %d->%d + 1x1 ->%d +res fused @%dx%d" % (cm, cm, cout, h, w), (tp,),
                                  "conv_c23<%d>" % cm, tiles, ragged=rag))
                inplanes = cout
                continue
            conv(tp + ".conv2", 3, st, cm, cm, h, w, False, per_image)
            if has_down and fuse_ds and cout % 256 == 0:
                tw, th, nbt = pick_patch(B, h2, w2)
                tiles = _cdiv(w2, tw) * _cdiv(h2, th) * _cdiv(B, nbt) * (cout // 128)
                out.append(Launch("1x1 [%d|%d%s]->%d fused-shortcut @%dx%d" % (cm, inplanes, "/s2" if st == 2 else "", cout, h2, w2),
                                  (tp,), "fused shortcut", tiles, pers(tiles), rag))
                inplanes = cout
                continue
            m = B * h * w
            if not has_down and st == 1 and j + 1 < nb and cm in (64, 128, 256) and _cdiv(m, 128) >= sms:   # c31_taken
                out.append(Launch("1x1 %d->%d +res + 1x1 ->%d fused @%dx%d" % (cm, cout, cm, h, w),
                                  (tp, "layer%d.%d.conv1" % (s, j + 1)), "conv_c31<%d>" % cm, _cdiv(m, 128),
                                  ragged=rag, last_rows=m - 128 * (_cdiv(m, 128) - 1)))
                t1_ready = True
                inplanes = cout
                continue
            if has_down:
                conv(tp + ".down", 1, st, inplanes, cout, h, w, False)
            conv(tp, 1, 1, cm, cout, h2, w2, True)
            inplanes = cout
    out.append(Launch("head pool+fc+l2", (), "head"))
    return out


def census(launches):
    """[(tag, launches)] in first-launch order: what profile_table() reports for one profiled forward."""
    rows = {}
    for ln in launches:
        rows[ln.tag] = rows.get(ln.tag, 0) + 1
    return list(rows.items())


def census_errors(launches, table):
    """Differences between the planned launches and a profile_table(); empty when they agree."""
    want = census(launches)
    got = [(r["tag"], int(r["launches"])) for r in table]
    if got == want:
        return []
    errs = ["planned %s x%d, ran %s" % (w[0], w[1], "x%d" % dict(got)[w[0]] if w[0] in dict(got) else "never")
            for w in want if w not in got]
    errs += ["ran %s x%d, not planned" % g for g in got if g[0] not in dict(want)]
    return errs or ["same launches in another order: %s" % [g[0] for g in got]]


def summary(launches):
    """Launches per kernel and consumer mode, with the tile counts of the conv_c31 launches."""
    n = {}
    for ln in launches:
        key = ln.kernel + ("" if ln.pp is None else " pp" if ln.pp else " coop") + (" RAGGED" if ln.ragged and ln.kernel != "head" else "")
        n[key] = n.get(key, 0) + 1
    c31 = sorted({(ln.kernel, ln.tiles, ln.last_rows) for ln in launches if ln.kernel.startswith("conv_c31")})
    return "; ".join("%s x%d" % kv for kv in n.items()) + "".join(
        "; %s: %d tiles, last tile %d rows" % c for c in c31)


# --------------------------------------------------------------------------- the cases
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _r152_batch(sms):
    """Smallest batch of 512^2 images whose layer3 (32^2 maps) has a 128-pixel tile for every SM."""
    return _cdiv(sms * 128, 32 * 32)


RAGGED_SIZES = [(1023, 513), (513, 1023), (1024, 1024), (333, 517), (64, 900)]


def network_cases(sms):
    """name -> (arch, B, H, W, picture sizes or None, seed) of the element-checked forwards."""
    b152 = _r152_batch(sms)
    return {
        "r101_9x717": ("resnet101_rmac", 9, 717, 717, None, 11),
        "r101_6x1024_trained": ("resnet101_rmac", 6, 1024, 1024, None, 12),
        "r152_%dx512" % b152: ("resnet152_rmac", b152, 512, 512, None, 13),
        "r50_ragged_1024_trained": ("resnet50_rmac", len(RAGGED_SIZES), 1024, 1024, RAGGED_SIZES, 14),
    }


def _case_plan(case, sms, **opts):
    arch, B, H, W, hw, _ = network_cases(sms)[case]
    return plan(arch, B, H, W, sms=sms, hw=hw, **opts)


def _covered(sms):
    fam = {}
    for case in network_cases(sms):
        for ln in _case_plan(case, sms):
            for f in ln.families():
                fam.setdefault(f, case)
    return fam


def _stage_fuses(launches, cm):
    return any(ln.kernel == "conv_c31<%d>" % cm for ln in launches)


# --------------------------------------------------------------------------- CPU: the plan itself
@pytest.mark.parametrize("case", list(network_cases(132)))
def test_plan_writes_every_checked_tap_once(case):
    """The plan's launches write, in order, exactly the taps check_network visits; every stage fuses at 132 SMs."""
    arch = network_cases(132)[case][0]
    launches = _case_plan(case, 132)
    writes = [t for ln in launches for t in ln.writes]
    assert writes == LM.expected_launches(arch)
    assert all(_stage_fuses(launches, cm) for cm in (64, 128, 256))


def test_plan_reproduces_the_selection_at_132_sms():
    """The existing matrix on a 132-SM H100: which stages take conv_c31 and which run two launches."""
    def fused(arch, B, H, W):
        return [_stage_fuses(plan(arch, B, H, W, sms=132), cm) for cm in (64, 128, 256)]
    assert fused("resnet101_rmac", 1, 1024, 1024) == [True, False, False]
    assert fused("resnet101_rmac", 1, 717, 717) == [True, False, False]
    assert fused("resnet101_rmac", 2, 1024, 1024) == [True, True, False]
    assert fused("resnet50_rmac", 8, 333, 517) == [True, True, False]
    assert fused("resnet50_rmac", 4, 224, 224) == [False, False, False]
    assert fused("resnet101_rmac", 9, 717, 717) == [True, True, True]
    # R101 9 x 717^2: layer3 is 45^2 x 9 = 143 tiles, its last tile 49 rows (warpgroup 1 has none)
    c31 = [ln for ln in plan("resnet101_rmac", 9, 717, 717, sms=132) if ln.kernel == "conv_c31<256>"]
    assert len(c31) == 21 and {(ln.tiles, ln.last_rows) for ln in c31} == {(143, 49)}
    # one 717^2 image: layer3 is 16 tiles, fused only where that is a tile for every SM
    assert not _stage_fuses(plan("resnet101_rmac", 1, 717, 717, sms=132), 256)
    assert _stage_fuses(plan("resnet101_rmac", 1, 717, 717, sms=16), 256)


def test_planned_cases_cover_every_family_at_132_sms():
    fam = _covered(132)
    assert REQUIRED <= set(fam), sorted(REQUIRED - set(fam))


# --------------------------------------------------------------------------- CPU: the checks fail when they should
def test_element_just_past_its_bound_fails_and_names_the_launch():
    """R50 forward emulated exactly (fp64, one fp16 rounding per launch): one element of the layer3 tap that conv_c31
    writes as the next block's conv1 output is set to the largest fp16 value within its bound (passes), then to the
    next one (fails, and the report names that launch alone)."""
    from test_layer_model import _emulated_taps
    arch, target = "resnet50_rmac", "layer3.2.conv1"
    sd = synth.make_state_dict(arch, seed=1)
    x16 = synth.make_images(1, 64, 96, seed=3).half()
    taps = _emulated_taps(sd, arch, x16)
    w = sd[target + ".weight"]
    s, t = LM.bn_fold(sd, "layer3.2.bn1", w.shape[0])
    e, m = LM.conv_em(taps["layer3.1"], LM.w16(w), 1, 0)
    sd64, td64 = (torch.from_numpy(v).double() for v in (s, t))
    yr = torch.relu(e * sd64 + td64)
    kappa = min(LM.KAPPA, LM.k16_steps(w.shape[1]))
    bound = 0.5 * LM.ulp16(yr) + 2.0 ** -22 * ((e * sd64).abs() + td64.abs()) + kappa * 2.0 ** -23 * sd64.abs() * m
    u = LM.ulp16(yr)
    frac = yr / (1024 * u) - 1                          # position inside the binade
    ok = (yr > 2.0 ** -13) & (frac > 0.2) & (frac < 0.8) & (bound < 0.1 * 1024 * u)
    i = int(torch.nonzero(ok.reshape(-1))[0])
    v, ui = float((yr + bound).reshape(-1)[i]), float(u.reshape(-1)[i])
    inside = math.floor(v / ui) * ui
    for val, passes in ((inside, True), (inside + ui, False)):
        y = taps[target].contiguous().clone()
        y.reshape(-1)[i] = val
        assert float(y.reshape(-1)[i]) == val
        bad = dict(taps, **{target: y})
        reps, _ = LM.check_network(bad.__getitem__, sd, arch, x16, device="cpu")
        assert [r.name for r in reps if not r.ok] == ([] if passes else [target])
        if not passes:
            with pytest.raises(AssertionError, match=r"layer3\.2\.conv1: 1 / \d+ elements outside the bound"):
                _report("planted", reps, LM.expected_launches(arch))


def test_nonzero_outside_an_extent_fails_the_mask_check():
    """Inside the mask the bound; outside it exactly 0: relu(shift) or the smallest fp16 subnormal there fails."""
    g = torch.Generator().manual_seed(0)
    e = torch.randn(2, 6, 10, 64, generator=g, dtype=torch.float64)
    m = e.abs() * 3
    s = np.full(64, 0.5, np.float32)
    t = np.linspace(-1, 1, 64).astype(np.float32)
    mask = torch.zeros(2, 6, 10, dtype=torch.bool)
    mask[0, :4, :7] = True
    mask[1, :6, :3] = True
    y = LM.fl16(torch.relu(e * 0.5 + torch.from_numpy(t).double()))
    y[~mask] = 0
    assert LM.check_elements("t1", y, e, m, s, t, mask=mask).ok
    for val in (float(t[-1]), 2.0 ** -24):
        z = y.clone()
        z[1, 5, 9, 63] = val
        r = LM.check_elements("t1", z, e, m, s, t, mask=mask)
        assert r.n_fail == 1 and "n=1 y=5 x=9 c=63" in r.worst


def test_census_one_launch_off_fails():
    """A profile table that ran one launch more, one fewer or another kernel than planned does not pass."""
    launches = _case_plan("r101_9x717", 132)
    table = [dict(tag=tg, launches=n) for tg, n in census(launches)]
    assert census_errors(launches, table) == []
    for i in (0, len(table) // 2, len(table) - 1):
        for d in (1, -1):
            off = [dict(r) for r in table]
            off[i]["launches"] += d
            assert census_errors(launches, off), (i, d)
    # one conv_c31 launch replaced by the two single launches it fuses
    k = next(j for j, ln in enumerate(launches) if ln.kernel == "conv_c31<256>")
    c = launches[k]
    split = launches[:k] + [Launch("1x1 256->1024 +res @45x45", (c.writes[0],), "conv_pers flat"),
                            Launch("1x1 1024->256 @45x45", (c.writes[1],), "conv_pers flat")] + launches[k + 1:]
    errs = census_errors(launches, [dict(tag=tg, launches=n) for tg, n in census(split)])
    assert any("fused" in e_ for e_ in errs), errs


# --------------------------------------------------------------------------- GPU: census + every element
def _run_network(case):
    """Profiled forward with taps, census against the plan, every launch against the fp64 bound, profile 0 forward
    bit-identical."""
    sms = _sms()
    arch, B, H, W, hw, seed = network_cases(sms)[case]
    trained = "trained" in case
    sd = LM.make_trained_like_state_dict(arch, seed=seed) if trained else synth.make_state_dict(arch, seed=seed)
    from dirb200 import ops
    launches = plan(arch, B, H, W, sms=sms, hw=hw, halo=int(ops.get_global_option("halo")))
    assert all(_stage_fuses(launches, cm) for cm in (64, 128, 256)), "%s: a stage does not fuse at %d SMs" % (case, sms)
    t0 = time.time()
    net = _net(arch, sd, B, profile=1)
    if hw is None:
        x = synth.make_images(B, H, W, seed=seed + 1)
        x16 = x.half()
        run = lambda: net(x.to(DEV))
    else:
        imgs = [synth.make_images(1, h, w, seed=seed + 1 + i)[0].to(DEV) for i, (h, w) in enumerate(hw)]
        x16 = torch.zeros(B, 3, H, W, dtype=torch.float16)
        for i, im in enumerate(imgs):
            x16[i, :, : im.shape[1], : im.shape[2]] = im.half().cpu()
        run = lambda: net.forward_ragged(imgs)
    d = run()
    torch.cuda.synchronize()
    table = net.profile_table()
    errs = census_errors(launches, table)
    print("CENSUS %s (%d SMs): %d launches: %s" % (case, sms, len(launches), summary(launches)))
    assert not errs, "%s: the forward did not run the planned kernels:\n%s" % (case, "\n".join(errs[:20]))
    tap = _taps(net)
    masks = None
    if hw is not None:
        masks = {}
        for lv, (Hs, Ws) in enumerate(_levels(H, W)):
            mk = torch.zeros(B, Hs, Ws, dtype=torch.bool)
            for i, (h, w) in enumerate(hw):
                hh, ww = _levels(h, w)[lv]
                mk[i, :hh, :ww] = True
            masks[(Hs, Ws)] = mk
    reps, _ = LM.check_network(tap, sd, arch, x16.to(DEV), device=DEV, masks=masks)
    _report(case, reps, LM.expected_launches(arch))
    if hw is None:
        _head_check(arch, sd, tap, d)
    if trained:
        for name in LM.expected_launches(arch) + ["stem", "layer4"]:
            assert torch.isfinite(tap(name)).all(), name
    del tap
    net.set_backend_option_live("profile", 0)
    d0 = run()
    torch.cuda.synchronize()
    assert torch.equal(d, d0), "%s: profile 1 changed the descriptors" % case
    print("TIME %s: %.1f s" % (case, time.time() - t0))


@gpu
def test_r101_9x717_every_stage_fused():
    """Layer3 is 45^2 x 9 = 143 tiles on 132 SMs; its last tile holds 49 rows, so warpgroup 1 has none."""
    _run_network("r101_9x717")


@gpu
def test_r101_6x1024_trained_like_every_stage_fused():
    """The bench's layer3 kernel (conv_c31<256>) with gammas down to 1e-4 and 0 and weight scales over two decades;
    every tap finite."""
    _run_network("r101_6x1024_trained")


@gpu
def test_r152_every_stage_fused():
    """34 conv_c31<256> launches in a row at layer3, at the smallest batch of 512^2 images that fuses it."""
    _run_network("r152_%dx512" % _r152_batch(_sms()))


@gpu
def test_r50_ragged_trained_like_every_stage_fused():
    """The RAGGED instantiations at all three stages: five pictures in 1024^2 slots (layer3 160 tiles); the conv1
    outputs conv_c31 writes for the next block are within the bound inside each picture and exactly 0 outside,
    where a missing zeroing would leave relu(shift1) (trained-like BatchNorm: shifts often positive)."""
    _run_network("r50_ragged_1024_trained")


@gpu
def test_every_family_is_checked_element_by_element():
    """Every kernel family the default configuration can select runs in one of the cases above on this device."""
    fam = _covered(_sms())
    print("FAMILIES (%d SMs): %s" % (_sms(), "; ".join("%s <- %s" % (f, fam[f]) for f in sorted(fam))))
    assert REQUIRED <= set(fam), sorted(REQUIRED - set(fam))


CENSUS_ONLY = [("fuse_c23_1", dict(fuse_c23=1)), ("fuse_c23_2", dict(fuse_c23=2)), ("halo_0", dict(halo=0)),
               ("fuse_ds_0", dict(fuse_ds=0))]


@gpu
@pytest.mark.parametrize("name,opts", CENSUS_ONLY, ids=[c[0] for c in CENSUS_ONLY])
def test_census_under_other_options(name, opts):
    """The mirror of the rules the default configuration does not take: R50 at 8 x 333 x 517 (layer1 c23-profitable,
    layer1 / layer2 c31) under fuse_c23 1 / 2, halo 0 and fuse_ds 0, tags and launch counts only."""
    from dirb200 import ops
    sms, arch, B, H, W = _sms(), "resnet50_rmac", 8, 333, 517
    saved = ops.get_global_option("halo")
    try:
        ops.set_global_option("halo", opts.get("halo", 1))
        launches = plan(arch, B, H, W, sms=sms, **opts)
        from dirb200 import nets
        net = nets.create_model(arch)
        net.load_state_dict(synth.make_state_dict(arch, seed=4))
        net.eval()
        for k, v in dict(chunk=B, profile=1, **{k: v for k, v in opts.items() if k != "halo"}).items():
            net.set_backend_option(k, v)
        net(synth.make_images(B, H, W, seed=9).to(DEV))
        torch.cuda.synchronize()
        errs = census_errors(launches, net.profile_table())
    finally:
        ops.set_global_option("halo", saved)
    print("CENSUS r50_8x333x517_%s (%d SMs): %s" % (name, sms, summary(launches)))
    assert not errs, "\n".join(errs[:20])


# --------------------------------------------------------------------------- GPU: the conv_c31 op against fp64
def _loguniform(r, n, lo, hi, zeros=0.0):
    v = np.exp(r.uniform(math.log(lo), math.log(hi), n))
    v[r.uniform(0, 1, n) < zeros] = 0.0
    return v.astype(np.float32)


# (Cm, B, H, W): full tiles at the ResNet-101 1024^2 stage shapes; the network's layer3 at 9 x 717^2 (143 tiles, the
# last one 49 rows); partial last tiles of 7, 49 and 3 rows, where only warpgroup 0 has rows
OP_CASES = [(64, 3, 256, 256), (128, 3, 128, 128), (256, 3, 64, 64), (256, 9, 45, 45), (256, 1, 17, 23),
            (128, 3, 7, 45), (64, 1, 33, 35)]


@gpu
@pytest.mark.parametrize("cm,b,h,w", OP_CASES, ids=["cm%d_%dx%dx%d" % c for c in OP_CASES])
def test_conv_c31_trained_like_against_fp64(cm, b, h, w):
    """ops.conv_c31 with a trained network's epilogue ranges - s3, s1 log-uniform over [1e-4, 10] with 5 % zeros,
    shifts of both signs, residual channels up to ~1e3, weight scales over two decades: y against the fp64 conv3 of t2
    plus x, t1 against the fp64 conv1 of the y the kernel wrote (teacher-forced), both bit-identical to the two single
    launches."""
    from dirb200 import ops
    ops.require_gpu(0)
    r = np.random.RandomState(cm * 7 + b * h * w)
    c4 = 4 * cm
    t2 = np.maximum(r.standard_normal((b, h, w, cm)), 0) * _loguniform(r, cm, 0.1, 10.0)
    x = np.maximum(r.standard_normal((b, h, w, c4)), 0) * _loguniform(r, c4, 1e-2, 1e3)
    w3 = r.standard_normal((c4, cm, 1, 1)) * np.sqrt(2.0 / cm) * _loguniform(r, c4, 0.1, 10.0)[:, None, None, None]
    w1 = r.standard_normal((cm, c4, 1, 1)) * np.sqrt(2.0 / c4) * _loguniform(r, cm, 0.03, 0.3)[:, None, None, None]
    s3, s1 = _loguniform(r, c4, 1e-4, 10.0, 0.05), _loguniform(r, cm, 1e-4, 10.0, 0.05)
    h3, h1 = (r.standard_normal(c4) * 2).astype(np.float32), (r.standard_normal(cm) * 2).astype(np.float32)
    t2g = torch.from_numpy(t2.astype(np.float16)).to(DEV)
    xg = torch.from_numpy(x.astype(np.float16)).to(DEV)
    w3t, w1t = torch.from_numpy(w3.astype(np.float32)), torch.from_numpy(w1.astype(np.float32))
    w3p, w1p = ops.pack_conv_weight(w3t).to(DEV), ops.pack_conv_weight(w1t).to(DEV)
    dev = lambda v: torch.from_numpy(v).to(DEV)
    y, t1 = ops.conv_c31(t2g, w3p, dev(s3), dev(h3), xg, w1p, dev(s1), dev(h1))
    y2 = ops.conv_bn_act(t2g, w3p, c4, 1, 1, 1, 0, dev(s3), dev(h3), xg, True)
    t12 = ops.conv_bn_act(y2, w1p, cm, 1, 1, 1, 0, dev(s1), dev(h1), None, True)
    torch.cuda.synchronize()
    m = b * h * w
    last = m - 128 * (_cdiv(m, 128) - 1)
    assert torch.isfinite(y).all() and torch.isfinite(t1).all()
    ry = LM.check_conv("y", y, t2g, w3t, 1, 0, s3, h3, res=xg, device=DEV)
    rt = LM.check_conv("t1", t1, y, w1t, 1, 0, s1, h1, device=DEV)
    print("C31 cm %d %dx%dx%d: %d tiles, last %d rows; y kappa_max %.4f exact %.4f, max %.4g; t1 kappa_max %.4f exact %.4f"
          % (cm, b, h, w, _cdiv(m, 128), last, ry.kappa_max, ry.exact / ry.n, float(y.float().max()), rt.kappa_max,
             rt.exact / rt.n))
    for rep in (ry, rt):
        assert rep.ok, "%s: %d / %d elements outside the bound; %s" % (rep.name, rep.n_fail, rep.n, rep.worst)
    assert torch.equal(y, y2)
    assert torch.equal(t1, t12)
