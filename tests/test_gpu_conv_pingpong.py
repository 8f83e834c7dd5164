"""Ping-pong consumer mode of the persistent convolution (conv_pers.cuh, PP): launches where every CTA gets at least three
tiles.  Each case is checked against the fp64 element bound of tests/layer_model.py, bit for bit against the same images
run in sub-batches small enough for the cooperative mode, and for determinism over three launches.  Batches are derived
from the SM count, so the mode of every launch is known.  Needs an H100: -m gpu."""
import math

import pytest
import torch

import layer_model as LM
import synthdata as synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ping_pong(total_tiles):
    """The selection rule of launch_conv_pers: ping-pong when every CTA of the persistent grid gets three tiles."""
    return total_tiles >= 3 * min(total_tiles, _sms())


def _bn_params(cout, seed):
    g = torch.Generator().manual_seed(seed)
    s = (0.5 + torch.rand(cout, generator=g)).float()
    t = (0.2 * torch.randn(cout, generator=g)).float()
    return s, t


def _conv(x, wp, cout, k, stride, pad, s, t, res, relu):
    from dirb200 import ops
    return ops.conv_bn_act(x, wp, cout, k, k, stride, pad, s.to(DEV), t.to(DEV), res=res, relu=relu)


def _run_case(name, cin, cout, k, stride, pad, H, W, B, b, res, relu=True, seed=0):
    """B images in one launch (ping-pong) against sub-batches of b (cooperative), the bound and three repeats."""
    from dirb200 import ops
    ops.require_gpu(0)
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, W, cin, generator=g) * 0.5).half().to(DEV)
    w = torch.randn(cout, cin, k, k, generator=g) * (1.0 / math.sqrt(cin * k * k))
    wp = ops.pack_conv_weight(w).to(DEV)
    s, t = _bn_params(cout, seed + 1)
    Ho = (H + 2 * pad - k) // stride + 1
    Wo = (W + 2 * pad - k) // stride + 1
    r = (torch.randn(B, Ho, Wo, cout, generator=g) * 0.5).half().to(DEV) if res else None
    y = _conv(x, wp, cout, k, stride, pad, s, t, r, relu)
    reps = [_conv(x, wp, cout, k, stride, pad, s, t, r, relu) for _ in range(3)]
    parts = [_conv(x[i:i + b].contiguous(), wp, cout, k, stride, pad, s, t,
                   None if r is None else r[i:i + b].contiguous(), relu) for i in range(0, B, b)]
    torch.cuda.synchronize()
    for i, yr in enumerate(reps):
        assert torch.equal(y, yr), "%s: launch %d differs from the first" % (name, i + 1)
    coop = torch.cat(parts, 0)
    assert torch.equal(y, coop), "%s: %d of %d elements differ from the cooperative sub-batches" % (
        name, int((y != coop).sum()), y.numel())
    rep = LM.check_conv(name, y, x, w, stride, pad, s.numpy(), t.numpy(), res=r, relu=relu, device=DEV)
    print("PINGPONG %s: B=%d b=%d kappa_max %.4f exact %.4f" % (name, B, b, rep.kappa_max, rep.exact / rep.n))
    assert rep.ok, "%s: %d / %d elements outside the bound; %s" % (name, rep.n_fail, rep.n, rep.worst)


def _batches(tiles_per_image):
    """(B, b): B images give >= 3 tiles per CTA; b images give >= SMs tiles (so a 128-channel tile stays 128 wide) and
    < 2 SMs tiles (so the launch is cooperative)."""
    S = _sms()
    b = -(-S // tiles_per_image)
    B = 3 * b
    assert _ping_pong(B * tiles_per_image) and not _ping_pong(b * tiles_per_image)
    return B, b


# name, cin, cout, kernel, stride, pad, H, W, residual; tiles per image = output pixels / 128 * cout / BN
CASES = [
    ("flat_bn128_res", 256, 1024, 1, 1, 0, 32, 32, True),        # the layer3 +res launch
    ("flat_bn128", 256, 1024, 1, 1, 0, 32, 32, False),
    ("flat_bn64_res", 64, 64, 1, 1, 0, 64, 64, True),
    ("flat_bn64", 128, 64, 1, 1, 0, 64, 64, False),
    ("strided_bn128", 256, 256, 1, 2, 0, 64, 64, False),         # 1x1 / stride 2: spatial TMA boxes, element stride 2
    ("halo_bn64_cin1", 64, 64, 3, 1, 1, 64, 64, False),
    ("halo_bn64_cin4", 256, 64, 3, 1, 1, 32, 32, True),
    ("halo_bn128_cin1", 64, 128, 3, 1, 1, 32, 32, True),
    ("halo_bn128_cin4", 256, 256, 3, 1, 1, 32, 32, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_pingpong_matches_cooperative(case):
    name, cin, cout, k, stride, pad, H, W, res = case
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    bn = 128 if cout % 128 == 0 else 64
    B, b = _batches(Ho * Wo // 128 * cout // bn)
    _run_case(name, cin, cout, k, stride, pad, H, W, B, b, res, seed=len(name))


TILE_COUNTS = [(2, -1), (2, 0), (2, 1), (3, 0), (3, -1), (3, 1), (5, 0)]


@pytest.mark.parametrize("mult_extra", TILE_COUNTS, ids=["2sms-1", "2sms", "2sms+1", "3sms", "3sms-1", "3sms+1", "5sms"])
def test_tile_counts_around_the_threshold(mult_extra):
    """1 x 128-pixel images, 64 channels: one tile each.  Up to 3 SMs - 1 tiles the launch stays cooperative (two tiles
    per CTA, and a third for some); 3 SMs gives every CTA three tiles (warpgroup 0 one more than warpgroup 1); 3 SMs + 1
    gives one CTA a fourth; 5 SMs gives every CTA an odd count again."""
    S = _sms()
    mult, extra = mult_extra
    B = mult * S + extra
    assert _ping_pong(B) == (B >= 3 * S)
    _run_case("tiles_%d" % B, 64, 64, 1, 1, 0, 1, 128, B, S - 1, True, seed=B)


def _net(arch, sd, chunk, **opts):
    from dirb200 import nets, ops
    ops.require_gpu(0)
    net = nets.create_model(arch)
    net.load_state_dict(sd)
    net.eval()
    for k, v in dict(debug_taps=1, fuse_c23=0, chunk=chunk, **opts).items():
        net.set_backend_option(k, v)
    return net


def test_network_fused_shortcut_and_every_launch_match_one_image_at_a_time():
    """R50 at 24 x 224^2: layer1 and layer2 (fused projection shortcut, k_split) ping-pong, layer3/4 stay cooperative.
    Every convolution's output and the descriptors equal those of each image alone (all cooperative)."""
    arch, B = "resnet50_rmac", 24
    sd = synth.make_state_dict(arch, seed=3)
    x = synth.make_images(B, 224, 224, seed=31).to(DEV)
    assert _ping_pong(B * 56 * 56 // 128 * 2) and _ping_pong(B * 28 * 28 // 128 * 4)
    names = LM.expected_launches(arch)
    net = _net(arch, sd, B)
    d, d16 = net.forward(x, want_f16=True)
    torch.cuda.synchronize()
    taps = {n: net.debug_stage(n) for n in names}
    one = _net(arch, sd, 1)
    for i in range(B):
        di, di16 = one.forward(x[i:i + 1], want_f16=True)
        torch.cuda.synchronize()
        assert torch.equal(d[i], di[0]) and torch.equal(d16[i], di16[0]), i
        if i % 5 == 0:
            for n in names:
                assert torch.equal(taps[n][i], one.debug_stage(n)[0]), (n, i)


def test_ragged_batch_pingpong_matches_one_image_at_a_time():
    """The RAGGED instantiation in ping-pong mode: 24 pictures of mixed sizes in one pass padded to 224^2 (layer1 and
    layer2 ping-pong) give the descriptors of each picture alone."""
    arch = "resnet50_rmac"
    sd = synth.make_state_dict(arch, seed=4)
    net = _net(arch, sd, 24)
    sizes = [(224 - 7 * i, 224 - 5 * ((3 * i) % 11)) for i in range(24)]
    imgs = [synth.make_images(1, h, w, seed=40 + i)[0] for i, (h, w) in enumerate(sizes)]
    assert _ping_pong(24 * 56 * 56 // 128 * 2)
    d = net.forward_ragged([im.to(DEV) for im in imgs])
    torch.cuda.synchronize()
    one = _net(arch, sd, 1)
    for i, im in enumerate(imgs):
        di = one(im[None].to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(d[i], di), (i, sizes[i])


def test_r101_2x1024_every_launch():
    """R101 at 2 x 1024^2: the layer3 +res launches (512 tiles of 128 x 128) take the ping-pong mode; every launch against
    the fp64 element bound."""
    from test_gpu_layers import _case
    assert _ping_pong(2 * 64 * 64 // 128 * 8)
    _case("r101_2x1024", "resnet101_rmac", synth.make_state_dict("resnet101_rmac", seed=2), synth.make_images(2, 1024, 1024, seed=7))
