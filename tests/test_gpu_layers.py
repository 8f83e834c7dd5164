"""Every convolution launch of the network against the teacher-forced fp64 reference of tests/layer_model.py, element
by element, at the network's real shapes: R101 at 1024^2 and 717^2, R50 under every kernel choice, BasicBlock, FPN,
uint8 input, trained-like weights and a ragged batch.  Needs an H100: -m gpu."""
import pytest
import torch

import layer_model as LM
import post_model as PM
import synthdata as synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _net(arch, sd, chunk, model_kw=None, **opts):
    from dirb200 import nets, ops
    ops.require_gpu(0)
    net = nets.create_model(arch, **(model_kw or {}))
    net.load_state_dict(sd)
    net.eval()
    for k, v in dict(debug_taps=1, fuse_c23=0, chunk=chunk, **opts).items():
        net.set_backend_option(k, v)
    return net


def _taps(net):
    cache = {}

    def tap(name):
        if name not in cache:
            cache[name] = net.debug_stage(name)
        return cache[name]
    return tap


def _head_check(arch, sd, tap, d, center_bias=0.0):
    """The head from the layer4 (and FPN fpn_c4) taps against the end-to-end bound of tests/post_model.py: every phase's
    bound propagated to the descriptor.  center_bias > 0: the taps precede it, so the head input is the fp64 x * m with
    the fp16 rounding of the center-bias output (one fp16 ulp plus its own bound) as input uncertainty."""
    w, b = sd["fc.weight"].to(DEV), sd["fc.bias"].to(DEV)

    def flat(t):
        return t.reshape(t.shape[0], -1, t.shape[-1])

    x5 = tap("layer4")
    if "_fpn" in arch:
        parts = [PM.head_partial_ref(flat(tap(n)), "gem", sd[k].item(), 1e-6) for n, k in (("fpn_c4", "adpoolc4.p"),
                                                                                         ("layer4", "adpoolx5.p"))]
        hw = [flat(tap("fpn_c4")).shape[1], flat(x5).shape[1]]
        pooled = [PM.head_pool_final_ref(P, n, "gem", sd[k].item(), False, eP)
                  for (P, eP), n, k in zip(parts, hw, ("adpoolc4.p", "adpoolx5.p"))]
        g, eg = torch.cat([v[0] for v in pooled], 1), torch.cat([v[1] for v in pooled], 1)
        y, ey = PM.head_fc_ref(g, w, b, eg)
        ref, bound = PM.l2_ref(y, ey, eps=1e-12)
    else:
        e_in = None
        x = x5
        if center_bias > 0:
            x, e_cb = PM.center_bias_ref(x5, center_bias)
            e_in = flat(e_cb + PM.ulp16(x * (1 + 2.0 ** -10)))
        ref, bound = PM.head_e2e(flat(x), "gem", sd["adpool.p"].item(), 1e-6, False, w, b, e_in)
    c = PM.check("head", d.reshape(ref.shape), ref, bound)
    print("HEAD %s: ratio %.4f" % (arch, c.ratio))
    assert c.ok, c.worst


def _report(case, reps, expected):
    n = sum(r.n for r in reps)
    kmax = max(r.kappa_max for r in reps)
    worst = max(reps, key=lambda r: r.kappa_max)
    print("LAYERS %s: %d launches, %d elements, kappa_max %.4f (%s), exact %.4f" %
          (case, len(reps), n, kmax, worst.name, sum(r.exact for r in reps) / n))
    assert [r.name for r in reps] == expected, "a convolution launch went unchecked"
    bad = [r for r in reps if not r.ok]
    assert not bad, "\n".join("%s: %d / %d elements outside the bound; %s" % (r.name, r.n_fail, r.n, r.worst) for r in bad[:12])


def _case(case, arch, sd, x, *, u8=None, head=True, center_bias=0.0, **opts):
    """Forward x (NCHW fp32) or u8 (B,H,W,3) with taps on, check every launch, the exact operators and the head."""
    B = (u8 if u8 is not None else x).shape[0]
    net = _net(arch, sd, B, model_kw=dict(center_bias=center_bias) if center_bias else None, **opts)
    if u8 is not None:
        d = net.forward_u8(torch.from_numpy(u8).to(DEV))
        x16 = LM.stem_input_u8(u8)
    else:
        d = net(x.to(DEV))
        x16 = x.half()
    torch.cuda.synchronize()
    tap = _taps(net)
    fuse_ds, impl = bool(opts.get("fuse_ds", 1)), int(opts.get("conv_impl", 0))
    reps, _ = LM.check_network(tap, sd, arch, x16.to(DEV), fuse_ds=fuse_ds, conv_impl=impl, device=DEV)
    _report(case, reps, LM.expected_launches(arch, fuse_ds=fuse_ds, conv_impl=impl))
    if head:
        _head_check(arch, sd, tap, d, center_bias)
    return net, tap


def _with_halo(halo, fn):
    from dirb200 import ops
    saved = ops.get_global_option("halo")
    try:
        ops.set_global_option("halo", halo)
        return fn()
    finally:
        ops.set_global_option("halo", saved)


def test_r101_1024_every_launch():
    """Bench geometry: 256^2 ... 32^2 maps, BN 64 and 128 tiles in one forward, HALO order at layer4 32^2."""
    _case("r101_1024", "resnet101_rmac", synth.make_state_dict("resnet101_rmac", seed=0), synth.make_images(1, 1024, 1024, seed=5))


def test_r101_717_every_launch():
    """Odd maps at every level (180 / 90 / 45 / 23): ragged tiles everywhere."""
    _case("r101_717", "resnet101_rmac", synth.make_state_dict("resnet101_rmac", seed=1), synth.make_images(1, 717, 717, seed=6))


@pytest.mark.parametrize("impl", [0, 1, 2], ids=["pers", "mma", "pers_1tile"])
def test_r50_224_every_launch(impl):
    """Golden geometry; layer4 7^2 runs tap by tap; the mma.sync path; one tile per CTA."""
    _case("r50_224_impl%d" % impl, "resnet50_rmac", synth.make_state_dict("resnet50_rmac", seed=2),
          synth.make_images(4, 224, 224, seed=7), conv_impl=impl)


@pytest.mark.parametrize("halo", [0, 1], ids=["tap_by_tap", "patch_once"])
def test_r50_333x517_many_tiles(halo):
    """8 images of 333 x 517: many tiles per CTA, both K orders of the 3x3 convolutions."""
    _with_halo(halo, lambda: _case("r50_333x517_halo%d" % halo, "resnet50_rmac", synth.make_state_dict("resnet50_rmac", seed=3),
                                   synth.make_images(8, 333, 517, seed=8)))


def test_r50_unfused_shortcut():
    """fuse_ds 0: the projection shortcut as its own launch (tap 'down') and conv3 with that residual."""
    _case("r50_fuse_ds0", "resnet50_rmac", synth.make_state_dict("resnet50_rmac", seed=4), synth.make_images(2, 160, 192, seed=9),
          fuse_ds=0)


def test_r50_center_bias_head():
    """center_bias > 0 runs on the layer4 map after its tap: the head is checked against center_bias applied to it."""
    _case("r50_center_bias", "resnet50_rmac", synth.make_state_dict("resnet50_rmac", seed=10), synth.make_images(2, 250, 190, seed=16),
          center_bias=1.5)


def test_r18_basic_block():
    """BasicBlock trunk: 3x3 convolutions with a residual, stride-2 3x3."""
    _case("r18", "resnet18_rmac", synth.make_state_dict("resnet18_rmac", seed=5), synth.make_images(3, 400, 300, seed=10))


def test_r50_fpn_head():
    """FPN mode 1: conv1x5, the nearest upsample-add (exact), the 3x3 smoothing convolution."""
    _, tap = _case("r50_fpn", "resnet50_fpn_rmac", synth.make_state_dict("resnet50_fpn_rmac", seed=6, out_dim=3072),
                   synth.make_images(2, 400, 300, seed=11))
    assert tap("fpn_c4").shape[1:3] == tap("layer3").shape[1:3]


def test_r50_uint8_stem():
    """uint8 input: the stem input is s2d_u8_kernel's normalisation, mirrored division by division."""
    _case("r50_u8", "resnet50_rmac", synth.make_state_dict("resnet50_rmac", seed=7), None,
          u8=synth.make_images_u8(3, 130, 174, seed=12))


@pytest.mark.parametrize("arch,b,size", [("resnet50_rmac", 2, 224), ("resnet101_rmac", 1, 1024)], ids=["r50_224", "r101_1024"])
def test_trained_like_weights(arch, b, size):
    """fp16 dynamic range of a trained network: gammas down to 1e-4 and 0, weight scales over two decades, calibrated
    BatchNorm statistics.  No inf or NaN anywhere."""
    sd = LM.make_trained_like_state_dict(arch, seed=0)
    _, tap = _case("trained_%s_%d" % (arch.split("_")[0], size), arch, sd, synth.make_images(b, size, size, seed=13))
    for name in LM.expected_launches(arch) + ["stem", "layer4"]:
        assert torch.isfinite(tap(name)).all(), name


def _levels(h, w):
    """Map sizes of the resolution levels 1..6 (stem conv, maxpool, layer1..4) of an h x w input."""
    out = []
    for lvl in range(1, 7):
        if lvl != 3:                                      # layer1 keeps the maxpool's size
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out.append((h, w))
    return out


def test_ragged_batch_absolute():
    """One ragged batch of three sizes: inside each picture's extent the convolution of its own cropped input with
    zero padding (by induction: every input tap is asserted exactly 0 outside), exactly 0 outside."""
    sizes = [(224, 224), (161, 97), (97, 161)]
    imgs = [synth.make_images(1, h, w, seed=20 + i)[0] for i, (h, w) in enumerate(sizes)]
    sd = synth.make_state_dict("resnet50_rmac", seed=8)
    net = _net("resnet50_rmac", sd, len(sizes))
    net.forward_ragged([x.to(DEV) for x in imgs])
    torch.cuda.synchronize()
    slots = torch.zeros(len(sizes), 3, 224, 224)
    for i, x in enumerate(imgs):
        slots[i, :, : x.shape[1], : x.shape[2]] = x
    masks = {}
    slot_lv = _levels(224, 224)
    for lv, (H, W) in enumerate(slot_lv):
        m = torch.zeros(len(sizes), H, W, dtype=torch.bool)
        for i, (h, w) in enumerate(sizes):
            hh, ww = _levels(h, w)[lv]
            m[i, :hh, :ww] = True
        masks[(H, W)] = m
    reps, _ = LM.check_network(_taps(net), sd, "resnet50_rmac", slots.half().to(DEV), device=DEV, masks=masks)
    _report("r50_ragged", reps, LM.expected_launches("resnet50_rmac"))


def test_fused_shortcut_fold_trained_like():
    """The fold fl16(s*W) of block 0's fused conv3 + projection shortcut, with trained-like BatchNorm: every block-0
    output against the unfolded arithmetic in fp64 (fp16 W, fp32 scale after the sum) from the same taps; the fused
    path's largest error in ulps of the output is at most twice the unfused path's."""
    arch = "resnet50_rmac"
    sd = LM.make_trained_like_state_dict(arch, seed=1)
    x = synth.make_images(2, 224, 224, seed=14).to(DEV)
    ulps = {}
    for fuse in (1, 0):
        net = _net(arch, sd, 2, fuse_ds=fuse)
        net(x)
        torch.cuda.synchronize()
        tap = _taps(net)
        for li in range(1, 5):
            ulps[(fuse, li)] = LM.fused_shortcut_ulps(tap, sd, "layer%d.0" % li, 1 if li == 1 else 2, device=DEV)
    print("FUSED_DS ulps: " + ", ".join("layer%d.0 fused %.2f unfused %.2f" % (li, ulps[(1, li)], ulps[(0, li)]) for li in range(1, 5)))
    for li in range(1, 5):
        assert ulps[(1, li)] <= 2.0 * max(ulps[(0, li)], 0.5), (li, ulps[(1, li)], ulps[(0, li)])


@pytest.mark.parametrize("arch", ["resnet50_rmac", "resnet50_fpn_rmac", "resnet18_rmac"])
def test_debug_taps_do_not_change_results(arch):
    """Descriptors (fp32 and fp16) are bit-identical with debug_taps 1 and 0."""
    net = _net(arch, synth.make_state_dict(arch, seed=9, out_dim=3072 if "_fpn" in arch else 2048), 3)
    x = synth.make_images(3, 200, 168, seed=15).to(DEV)
    on = net.forward(x, want_f16=True)
    net.set_backend_option_live("debug_taps", 0)
    off = net.forward(x, want_f16=True)
    torch.cuda.synchronize()
    assert torch.equal(on[0], off[0]) and torch.equal(on[1], off[1])
