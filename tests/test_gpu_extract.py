"""End-to-end descriptor extraction on the GPU vs the golden vectors of the unmodified reference and the
CPU oracle.  Tolerance: 1e-3 relative L2 on the unit-norm descriptor (BASELINE.json north_star).  -m gpu."""
import numpy as np
import pytest
import torch

import synthdata as synth
from oracle import dir_oracle as O
from conftest import rel_l2

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _net(arch, seed, **kw):
    from dirb200 import nets, ops
    ops.require_gpu(0)
    net = nets.create_model(arch, **kw)
    sd = synth.make_state_dict(arch, seed=seed, gemp=kw.get("gemp", 3))
    if not kw.get("pooling", "gem").startswith("gem"):
        sd.pop("adpool.p")
    net.load_state_dict(sd)
    net.eval()
    return net, sd


@pytest.mark.parametrize("impl", [0, 1, 2], ids=["tcgen05", "mma", "tcgen05np"])
def test_extract_r50_golden(golden, impl):
    g = golden("extract_r50.npz")
    net, sd = _net("resnet50_rmac", int(g["seed"]))
    net.set_backend_option("conv_impl", impl)
    net.set_backend_option("debug_taps", 1)
    x = synth.make_images(4, 224, 224, seed=int(g["img_seed"]))
    d = net(x.cuda()).cpu().numpy()
    # stage-by-stage diagnostics against the reference's activations (one pixel, all channels)
    for stage, key in (("stem", "maxpool"), ("layer1", "layer1"), ("layer2", "layer2"), ("layer3", "layer3"), ("layer4", "layer4")):
        a = net.debug_stage(stage).float().cpu()
        sl = a[0, a.shape[1] // 2, a.shape[2] // 3, :].numpy()
        assert rel_l2(sl, g["slice_" + key]) < 5e-3, stage
    assert d.shape == (4, 2048)
    assert rel_l2(d, g["desc"]) < TOL
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-5)
    d1 = net(x[:1].cuda())
    assert tuple(d1.shape) == (2048,)                     # squeeze at B=1, rmac_resnet.py:64
    assert rel_l2(d1.cpu().numpy(), g["desc_b1"]) < TOL
    xr = synth.make_images(2, 160, 224, seed=int(g["img_seed_rect"]))
    assert rel_l2(net(xr.cuda()).cpu().numpy(), g["desc_rect"]) < TOL
    # chunking must not change anything: same descriptors with 1 image per pass
    net.set_backend_option("chunk", 1)
    net.set_backend_option("conv_impl", impl)
    assert np.array_equal(net(x.cuda()).cpu().numpy(), d)
    # host-buffer entry point (H2D + forward + D2H inside the C call)
    assert np.array_equal(net.forward_host(x.numpy()), d)


def test_extract_r50_options(golden):
    g = golden("extract_r50_options.npz")
    b, h, w = [int(v) for v in g["img_shape"]]
    x = synth.make_images(b, h, w, seed=int(g["img_seed"])).cuda()
    for tag, kw in [("max", dict(pooling="max")), ("avg", dict(pooling="avg")), ("normfeat", dict(norm_features=True)),
                    ("nofc", dict(without_fc=True)), ("gemp2", dict(gemp=2))]:
        net, _ = _net("resnet50_rmac", int(g["seed"]), **kw)
        assert rel_l2(net(x).cpu().numpy(), g["desc_" + tag]) < TOL, tag


def test_extract_r101_golden(golden):
    g = golden("extract_r101.npz")
    net, _ = _net("resnet101_rmac", int(g["seed"]))
    x = synth.make_images(2, 224, 224, seed=int(g["img_seed"]))
    assert rel_l2(net(x.cuda()).cpu().numpy(), g["desc"]) < TOL


def test_extract_r152_and_center_bias_golden(golden):
    g = golden("extract_extra.npz")
    net, _ = _net("resnet152_rmac", int(g["r152_seed"]))
    b, h, w = [int(v) for v in g["r152_img_shape"]]
    d = net(synth.make_images(b, h, w, seed=int(g["r152_img_seed"])).cuda())
    assert tuple(d.shape) == (2048,) and rel_l2(d.cpu().numpy(), g["desc_r152"]) < TOL
    b, h, w = [int(v) for v in g["cb_img_shape"]]
    x = synth.make_images(b, h, w, seed=int(g["cb_img_seed"])).cuda()
    for tag, cb in (("cb05", 0.5), ("cb2", 2.0)):                      # rmac_resnet.py:52-56
        net, _ = _net("resnet50_rmac", int(g["cb_seed"]), center_bias=cb)
        assert rel_l2(net(x).cpu().numpy(), g["desc_" + tag]) < TOL, tag


def _variant_net(arch, seed, **kw):
    from dirb200 import nets, ops
    ops.require_gpu(0)
    net = nets.create_model(arch, **kw)
    sd = synth.make_state_dict(arch, seed=seed, out_dim=net.out_dim)
    if net.fpn and net.mode == 0:
        sd.pop("conv1x5.weight")
        sd.pop("conv3c4.weight")
    net.load_state_dict(sd)
    return net.eval(), sd


def test_extract_variants_golden(golden):
    """SURVEY 8f-4: BasicBlock trunk (resnet18_rmac, resnet.py:15-44) and the FPN head (rmac_resnet_fpn.py:52-90,
    modes 1 and 0) against the unmodified reference's descriptors."""
    g = golden("extract_variants.npz")
    b, h, w = [int(v) for v in g["img_shape"]]
    x = synth.make_images(b, h, w, seed=int(g["img_seed"])).cuda()
    net, _ = _variant_net("resnet18_rmac", int(g["r18_seed"]))
    assert rel_l2(net(x).cpu().numpy(), g["desc_r18"]) < TOL
    d1 = net(x[:1])
    assert tuple(d1.shape) == (2048,) and rel_l2(d1.cpu().numpy(), g["desc_r18_b1"]) < TOL
    net, _ = _variant_net("resnet50_fpn_rmac", int(g["fpn_seed"]), out_dim=2048)
    assert rel_l2(net(x).cpu().numpy(), g["desc_r50_fpn"]) < TOL
    net, _ = _variant_net("resnet50_fpn_rmac", int(g["fpn_seed"]), out_dim=2048, mode=0)
    assert rel_l2(net(x).cpu().numpy(), g["desc_r50_fpn0"]) < TOL
    net, _ = _variant_net("resnet18_fpn_rmac", int(g["r18_fpn_seed"]), out_dim=512)
    d = net(x)
    assert tuple(d.shape) == (2, 512) and rel_l2(d.cpu().numpy(), g["desc_r18_fpn"]) < TOL


@pytest.mark.parametrize("arch,kw", [("resnet18_rmac", {}), ("resnet18_fpn_rmac", {}), ("resnet50_fpn_rmac", {}),
                                      ("resnet101_fpn0_rmac", {}), ("resnet50_fpn_rmac", dict(norm_features=True, without_fc=True))],
                         ids=["r18", "r18_fpn", "r50_fpn", "r101_fpn0", "r50_fpn_nofc_norm"])
def test_variants_larger_images_vs_oracle(arch, kw):
    """Same variants at sizes that reach the 3x3 convolution with a residual (BasicBlock conv2), the stride-2 3x3
    convolutions, odd map sizes in the nearest upsampling (layer3 25x19 <- layer4 13x10) and batch / chunk invariance."""
    net, sd = _variant_net(arch, 9, **kw)
    x = synth.make_images(3, 400, 300, seed=17)
    d = net(x.cuda())
    if "_fpn" in arch:
        ref = O.extract_fpn(x, sd, arch, mode=net.mode, norm_features=bool(kw.get("norm_features")),
                            without_fc=bool(kw.get("without_fc"))).numpy()
    else:
        ref = O.extract(x, sd, arch).numpy()
    assert d.shape == ref.shape and rel_l2(d.cpu().numpy(), ref) < TOL
    one = net(x[1:2].cuda())
    assert torch.equal(one, d[1])                                       # batch invariance, B=1 squeeze
    net.set_backend_option("chunk", 2)
    assert torch.equal(net(x.cuda()), d)


def test_fused_c23_network_equals_two_kernel_path():
    """Option fuse_c23 (conv2 + conv3 + residual of the identity blocks as one kernel) does not change a single bit
    of the descriptors."""
    net, sd = _net("resnet101_rmac", 3)
    x = synth.make_images(3, 320, 272, seed=8).cuda()
    net.set_backend_option("fuse_c23", 2)
    a = net(x)
    n_fused = net.last_launch_stats()[0]
    net.set_backend_option("fuse_c23", 0)
    b = net(x)
    assert net.last_launch_stats()[0] > n_fused          # fewer launches with the fused blocks
    assert torch.equal(a, b)
    assert rel_l2(a.cpu().numpy(), O.extract(x.cpu(), sd, "resnet101_rmac").numpy()) < TOL


def test_extract_r101_large_image_vs_oracle():
    # one 512x384 image against the CPU oracle, plus batch-composition invariance at that size
    net, sd = _net("resnet101_rmac", 2)
    x = synth.make_images(3, 384, 512, seed=9)
    d = net(x.cuda()).cpu().numpy()
    ref = O.extract(x[:1], sd, "resnet101_rmac", squeeze=False).numpy()
    assert rel_l2(d[:1], ref) < TOL
    d_alone = net(x[1:2].cuda()).cpu().numpy()
    assert np.array_equal(d_alone, d[1])


def test_full_size_1024_vs_oracle_and_batch_properties():
    """BASELINE configs[1] geometry (ResNet-101, 1024x1024): one image against the CPU oracle, and the
    size-independent properties at batch level: batch-composition invariance, unit norm, determinism."""
    net, sd = _net("resnet101_rmac", 0)
    x = synth.make_images(6, 1024, 1024, seed=21)
    xc = x.cuda()
    d = net(xc).cpu().numpy()
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-5)
    ref = O.extract(x[2:3], sd, "resnet101_rmac", squeeze=False).numpy()
    assert rel_l2(d[2:3], ref) < TOL
    assert np.array_equal(net(xc[2:3]).cpu().numpy(), d[2])              # alone == inside the batch
    assert np.array_equal(net(xc[[4, 2, 0]]).cpu().numpy(), d[[4, 2, 0]])  # order / neighbours do not matter
    assert np.array_equal(net(xc).cpu().numpy(), d)                      # run-to-run deterministic
    launches, flops = net.last_launch_stats()
    assert abs(flops / 6 / 325.99e9 - 1.0) < 0.01                        # SURVEY 8d: 325.99 GFLOP per image


def test_multiscale_pool_matches_oracle():
    """BASELINE configs[4] structure at reduced size: Scale(0.7), identity, Scale(1.4) chains -> gem pool -> L2."""
    from dirb200 import ops
    net, sd = _net("resnet50_rmac", 0)
    base = synth.make_images(3, 160, 192, seed=8)
    sizes = [(int(0.5 + 0.7 * 160), int(0.5 + 0.7 * 192)), (160, 192), (int(0.5 + 1.4 * 160), int(0.5 + 1.4 * 192))]
    descs_gpu, descs_ref = [], []
    for (h, w) in sizes:
        xs = torch.nn.functional.interpolate(base, size=(h, w), mode="bilinear", align_corners=False)
        descs_gpu.append(net(xs.cuda()))
        descs_ref.append(O.extract(xs, sd, "resnet50_rmac").numpy())
    pooled = ops.pool_scales(descs_gpu, "gem", 3, l2=True).cpu().numpy()
    ref = O.l2n(O.pool_scales(descs_ref, "gem", 3))
    assert rel_l2(pooled, ref) < TOL


def test_uint8_input_is_bit_identical_to_fp32_input():
    """ToTensor + Normalize fused into the stem input stage (uint8 HWC in): same descriptors, bit for bit."""
    net, sd = _net("resnet50_rmac", 0)
    u8 = synth.make_images_u8(3, 130, 174, seed=12)
    x = synth.normalise_images(u8)
    d_f32 = net(x.cuda()).cpu().numpy()
    d_u8 = net.forward_u8(torch.from_numpy(u8).cuda()).cpu().numpy()
    assert np.array_equal(d_u8, d_f32)
    assert np.array_equal(net.forward_host_u8(u8), d_f32)
    ref = O.extract(x, sd, "resnet50_rmac").numpy()
    assert rel_l2(d_u8, ref) < TOL


def test_host_pipeline_over_several_chunks_is_bit_identical():
    """The host-buffer entry points copy chunk i+1 while chunk i runs, in doubling chunks: host_chunk 4 over 23 images
    runs chunks of 2, 2, 4, 8 and 7 images.  They give the device entry points' descriptors bit for bit.  The removed
    sub-chunk schedule options are unknown keys."""
    from dirb200 import lib
    net, _ = _net("resnet50_rmac", 0)
    u8 = synth.make_images_u8(23, 64, 96, seed=5)
    x = synth.normalise_images(u8)
    d = net(x.cuda()).cpu().numpy()
    d_u8 = net.forward_u8(torch.from_numpy(u8).cuda()).cpu().numpy()
    net.set_backend_option("host_chunk", 4)
    assert np.array_equal(net.forward_host(x.numpy()), d)
    assert np.array_equal(net.forward_host_u8(u8), d_u8)
    for key, value in (("stage_sched", 1), ("sub0", 8)):
        net, _ = _net("resnet50_rmac", 0)
        net.set_backend_option(key, value)
        with pytest.raises(lib.DirbError):
            net(x[:1].cuda())


@pytest.mark.parametrize("size", [(717, 717), (1434, 1434), (64, 48), (333, 517)], ids=lambda s: "%dx%d" % s)
def test_odd_and_multiscale_sizes_vs_oracle(size):
    """BASELINE configs[4] scales of a 1024^2 image (Scale(0.7) -> 717, Scale(1.4) -> 1434, transforms.py:168) plus tiny
    and odd rectangular inputs: every stage has ragged tiles; one image against the CPU oracle."""
    net, sd = _net("resnet101_rmac", 3)
    h, w = size
    x = synth.make_images(2, h, w, seed=31)
    d = net(x.cuda()).cpu().numpy()
    ref = O.extract(x[:1], sd, "resnet101_rmac", squeeze=False).numpy()
    assert rel_l2(d[:1], ref) < TOL
    assert np.array_equal(net(x[:1].cuda()).cpu().numpy(), d[0])


def test_gpu_multiscale_equals_pil_resize_path():
    """Scale(0.7) / identity / Scale(1.4) with the resize on the GPU == the same chains with PIL's resize on the CPU
    (bit-identical pixels -> bit-identical descriptors), and the pooled result matches the oracle."""
    from PIL import Image
    from dirb200 import ops
    net, sd = _net("resnet50_rmac", 0)
    u8 = synth.make_images_u8(2, 150, 210, seed=14)
    pooled = net.forward_u8_multiscale(torch.from_numpy(u8).cuda(), scales=(0.7, 1.0, 1.4), pooling="gem", gemp=3).cpu().numpy()
    per_scale_gpu, per_scale_ref = [], []
    for s in (0.7, 1.0, 1.4):
        wo, ho = int(0.5 + s * 210), int(0.5 + s * 150)
        res = np.stack([np.array(Image.fromarray(u8[i]).resize((wo, ho), Image.BILINEAR)) if s != 1.0 else u8[i] for i in range(2)])
        per_scale_gpu.append(net.forward_u8(torch.from_numpy(res).cuda()))
        per_scale_ref.append(O.extract(synth.normalise_images(res), sd, "resnet50_rmac").numpy())
    same = ops.pool_scales(per_scale_gpu, "gem", 3, l2=True).cpu().numpy()
    assert np.array_equal(pooled, same)
    assert rel_l2(pooled, O.l2n(O.pool_scales(per_scale_ref, "gem", 3))) < TOL
