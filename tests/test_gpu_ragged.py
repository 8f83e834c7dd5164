"""Ragged batches: images of different sizes in one network pass (dirb200_net_forward_ragged{,_u8}).  Every descriptor
must equal, bit for bit, the one of a B = 1 forward of the image alone, so everything here compares with ==.  -m gpu."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import synthdata as synth

pytestmark = pytest.mark.gpu

# odd sizes that round differently at every stage, portrait and landscape, the slot itself, the smallest legal size
SIZES = [(1023, 513), (513, 1023), (1023, 1023), (32, 32), (33, 65), (65, 33), (97, 97), (97, 33), (200, 150),
         (333, 517), (64, 48), (129, 257)]


def _net(arch, seed=1, **kw):
    from dirb200 import nets, ops
    ops.require_gpu(0)
    net = nets.create_model(arch, **kw)
    sd = synth.make_state_dict(arch, seed=seed)
    if not kw.get("pooling", "gem").startswith("gem"):
        sd.pop("adpool.p")
    net.load_state_dict(sd)
    return net.eval()


def _images(sizes, seed=5):
    return [torch.from_numpy(synth.make_images_u8(1, h, w, seed=seed + i)[0]).cuda() for i, (h, w) in enumerate(sizes)]


def _alone_u8(net, x):
    """B = 1 forward_u8 of one (h,w,3) image -> (fp32, fp16) descriptors."""
    from dirb200 import lib
    h = net._ensure_with_preprocess(0)
    d = torch.empty((1, net.descriptor_dim), dtype=torch.float32, device="cuda")
    d16 = torch.empty((1, net.descriptor_dim), dtype=torch.float16, device="cuda")
    lib.call("dirb200_net_forward_u8", h, C.c_void_p(x.data_ptr()), 1, int(x.shape[0]), int(x.shape[1]),
             C.c_void_p(d.data_ptr()), C.c_void_p(d16.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return d[0], d16[0]


def _slots_u8(imgs, fill=None):
    hh, ww = max(int(x.shape[0]) for x in imgs), max(int(x.shape[1]) for x in imgs)
    slots = torch.zeros((len(imgs), hh, ww, 3), dtype=torch.uint8, device="cuda")
    if fill is not None:
        slots.copy_(torch.from_numpy(np.random.RandomState(fill).randint(0, 256, slots.shape, dtype=np.uint8)))
    for i, x in enumerate(imgs):
        slots[i, :x.shape[0], :x.shape[1]] = x
    return slots, [(int(x.shape[0]), int(x.shape[1])) for x in imgs]


CASES = [
    ("resnet50_rmac", {}, {}),
    ("resnet50_rmac", {}, dict(fuse_c23=2, head_fused=0, chunk=5)),
    ("resnet50_rmac", {}, dict(fuse_c23=1, halo=0)),
    ("resnet50_rmac", dict(pooling="max", norm_features=True), dict(fuse_c23=2)),
    ("resnet50_rmac", dict(pooling="avg", without_fc=True, center_bias=0.5), {}),
    ("resnet50_rmac", dict(center_bias=1.0, norm_features=True), dict(head_fused=0, chunk=7)),
    ("resnet18_rmac", {}, {}),
    ("resnet18_rmac", dict(center_bias=0.5, pooling="max"), dict(chunk=3, halo=0)),
    ("resnet101_rmac", {}, dict(fuse_c23=1)),
]


@pytest.mark.parametrize("arch,model_kw,opts", CASES,
                         ids=["r50", "r50_c23_2_phases_chunk5", "r50_c23_1_tapbytap", "r50_max_normfeat_c23",
                              "r50_avg_nofc_cbias", "r50_cbias_normfeat_phases_chunk7", "r18", "r18_cbias_max_chunk3_tap",
                              "r101_c23_1"])
def test_ragged_equals_one_image_at_a_time(arch, model_kw, opts):
    from dirb200 import ops
    net = _net(arch, **model_kw)
    glob = {k: v for k, v in opts.items() if k in ("halo", "head_fused")}
    saved = {k: ops.get_global_option(k) for k in glob}
    try:
        for k, v in glob.items():
            ops.set_global_option(k, v)
        for k, v in opts.items():
            if k not in glob:
                net.set_backend_option(k, v)
        sizes = SIZES if arch != "resnet101_rmac" else SIZES[2:]
        imgs = _images(sizes)
        slots, hw = _slots_u8(imgs)
        d, d16 = net.forward_ragged_slots(slots, hw, want_f16=True)
        alone = [_alone_u8(net, x) for x in imgs]
        for i in range(len(imgs)):
            assert torch.equal(d[i], alone[i][0]), (i, hw[i])
            assert torch.equal(d16[i], alone[i][1]), (i, hw[i])
        assert torch.equal(net.forward_ragged_u8(imgs), d)
    finally:
        for k, v in saved.items():
            ops.set_global_option(k, v)


def test_content_outside_the_extents_is_ignored_and_taps_are_zero_there():
    net = _net("resnet50_rmac")
    net.set_backend_option("fuse_c23", 2)
    imgs = _images(SIZES[3:])
    clean, hw = _slots_u8(imgs)
    d = net.forward_ragged_slots(clean, hw)
    noisy, _ = _slots_u8(imgs, fill=17)
    assert not torch.equal(noisy, clean)
    net.set_backend_option_live("debug_taps", 1)
    assert torch.equal(net.forward_ragged_slots(noisy, hw), d)

    def ext(h, w, n):               # stem conv (7x7/s2/p3), then n halvings of 3x3/s2/p1
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        for _ in range(n):
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        return h, w

    for stage, n in (("stem", 1), ("layer1", 1), ("layer2", 2), ("layer3", 3), ("layer4", 4)):
        a = net.debug_stage(stage)
        assert a.shape[0] == len(imgs)
        for i, (h, w) in enumerate(hw):
            eh, ew = ext(h, w, n)
            assert a[i, eh:].abs().max().item() == 0 if eh < a.shape[1] else True, (stage, i)
            assert a[i, :, ew:].abs().max().item() == 0 if ew < a.shape[2] else True, (stage, i)
            assert a[i, :eh, :ew].abs().max().item() > 0, (stage, i)
    # fp32 slots: NaN outside the images changes nothing either
    xs = [synth.normalise_images(x.cpu().numpy()[None])[0] for x in imgs]
    slots = torch.full((len(xs), 3, clean.shape[1], clean.shape[2]), float("nan"), device="cuda")
    for i, x in enumerate(xs):
        slots[i, :, :x.shape[1], :x.shape[2]] = x.cuda()
    assert torch.equal(net.forward_ragged_slots(slots, hw), d)


def test_fp32_entry_agrees_with_u8_and_with_forward():
    net = _net("resnet50_rmac")
    imgs = _images(SIZES[2:9], seed=40)
    d = net.forward_ragged_u8(imgs)
    xs = [synth.normalise_images(x.cpu().numpy()[None])[0].cuda() for x in imgs]
    assert torch.equal(net.forward_ragged(xs), d)
    for i, x in enumerate(xs):
        assert torch.equal(net(x[None]), d[i])


def test_rejections():
    from dirb200 import lib
    net = _net("resnet50_rmac")
    slots, hw = _slots_u8(_images([(64, 64), (48, 40)]))
    with pytest.raises(lib.DirbError) as e:
        net.forward_ragged_slots(slots, [(64, 64), (31, 40)])
    assert e.value.status == -1
    with pytest.raises(lib.DirbError) as e:
        net.forward_ragged_slots(slots, [(64, 65), (48, 40)])
    assert e.value.status == -1
    net.set_backend_option("conv_impl", 1)
    with pytest.raises(lib.DirbError) as e:
        net.forward_ragged_slots(slots, hw)
    assert e.value.status == -2
    fpn = _net("resnet50_fpn_rmac", out_dim=2048)
    with pytest.raises(lib.DirbError) as e:
        fpn.forward_ragged_slots(slots, hw)
    assert e.value.status == -2


def _write_images(root, sizes, seed=3):
    from PIL import Image
    os.makedirs(os.path.join(root, "jpg"), exist_ok=True)
    names = []
    for i, (h, w) in enumerate(sizes):
        names.append("im%03d.png" % i)
        Image.fromarray(synth.make_images_u8(1, h, w, seed=seed + i)[0]).save(os.path.join(root, "jpg", names[-1]))
    return names


def test_driver_batches_mixed_sizes_like_one_at_a_time(tmp_path):
    """extract_image_features(batch_size=16) == batch_size=1 on mixed sizes: GPU preprocessing ('', Scale(0.7)) with
    flips, the PIL branch, and an ImageListROIs query set cropped to per-query boxes."""
    from dirb200 import datasets, pipeline
    root = str(tmp_path)
    rs = np.random.RandomState(0)
    sizes = [(int(rs.randint(60, 300)), int(rs.randint(60, 300))) for _ in range(37)] + [(160, 192)] * 5
    names = _write_images(root, sizes)
    ds = datasets.ImageList(imgs=names, root=os.path.join(root, "jpg"))
    net = _net("resnet50_rmac")
    flips = [bool(v) for v in rs.randint(0, 2, len(names))]
    for chain in ("", "Scale(0.7)"):
        a = pipeline.extract_image_features(ds, chain, net, threads=2, batch_size=16, flip=list(flips))
        b = pipeline.extract_image_features(ds, chain, net, threads=2, batch_size=1, flip=list(flips))
        assert a.shape == (len(names), 2048) and torch.equal(a, b), chain
    a = pipeline.extract_image_features(ds, "Scale(0.7)", net, threads=2, batch_size=5, gpu_preprocess=False)
    b = pipeline.extract_image_features(ds, "Scale(0.7)", net, threads=2, batch_size=1, gpu_preprocess=False)
    assert torch.equal(a, b)
    rois = [(int(rs.randint(0, 20)), int(rs.randint(0, 20)), w - int(rs.randint(0, 20)), h - int(rs.randint(0, 20)))
            for (h, w) in sizes[:12]]
    q = datasets.ImageListROIs(root, "jpg", names[:12], rois)
    a = pipeline.extract_image_features(q, "", net, threads=2, batch_size=16)
    b = pipeline.extract_image_features(q, "", net, threads=2, batch_size=1)
    assert torch.equal(a, b)
