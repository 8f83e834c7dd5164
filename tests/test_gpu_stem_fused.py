"""The fused stem (stem convolution + BN + ReLU + maxpool in one kernel, net option fuse_stem 1) against the three-launch
path (fuse_stem 0) in the same process: the pooled map and the fp32 / fp16 descriptors must be bit-identical, for fp32
and uint8 input, dense and ragged batches and every forward entry point.  -m gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

import layer_model as LM
import synthdata as synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ARCH = "resnet50_rmac"
SHAPES = [(2, 64, 96), (1, 63, 65), (3, 224, 224), (2, 130, 70), (1, 717, 717), (1, 1024, 1024)]
SD = {}


def _sd():
    if not SD:
        SD["sd"] = synth.make_state_dict(ARCH, seed=2)
    return SD["sd"]


def _nets(**opts):
    """(fused, unfused) networks with the same weights and options."""
    from dirb200 import nets, ops
    ops.require_gpu(0)
    out = []
    for fuse in (1, 0):
        net = nets.create_model(ARCH)
        net.load_state_dict(_sd())
        for k, v in dict(opts, fuse_stem=fuse).items():
            net.set_backend_option(k, v)
        out.append(net.eval())
    return out


def _forward_dev(net, x, u8):
    """(fp32, fp16) descriptors of a dense device batch: NCHW fp32 or HWC uint8."""
    from dirb200 import lib
    h = net._ensure_with_preprocess(0) if u8 else net._ensure(0)
    b, hh, ww = int(x.shape[0]), int(x.shape[1] if u8 else x.shape[2]), int(x.shape[2] if u8 else x.shape[3])
    d = torch.empty((b, net.descriptor_dim), dtype=torch.float32, device=DEV)
    d16 = torch.empty((b, net.descriptor_dim), dtype=torch.float16, device=DEV)
    lib.call("dirb200_net_forward_u8" if u8 else "dirb200_net_forward", h, C.c_void_p(x.data_ptr()), b, hh, ww,
             C.c_void_p(d.data_ptr()), C.c_void_p(d16.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return d, d16


def _same(a, b):
    """Bit-identical (torch.equal alone takes -0 == +0)."""
    def bits(t):
        return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def _input(shape, u8, seed=7):
    b, h, w = shape
    if u8:
        return torch.from_numpy(synth.make_images_u8(b, h, w, seed=seed)).to(DEV).contiguous()
    return synth.make_images(b, h, w, seed=seed).to(DEV).contiguous()


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_network_fused_stem_is_bit_identical(shape, u8):
    fused, plain = _nets()
    x = _input(shape, u8)
    d1, h1 = _forward_dev(fused, x, u8)
    d0, h0 = _forward_dev(plain, x, u8)
    assert _same(d1, d0) and _same(h1, h0)
    assert fused.last_launch_stats()[0] == plain.last_launch_stats()[0] - 2
    # the stem taps: the fused kernel also writes the stem map it computes when taps are on
    for net in (fused, plain):
        net.set_backend_option_live("debug_taps", 1)
    t1 = _forward_dev(fused, x, u8)
    t0 = _forward_dev(plain, x, u8)
    assert _same(t1[0], d0) and _same(t0[0], d0)
    assert _same(fused.debug_stage("stem"), plain.debug_stage("stem"))
    assert _same(fused.debug_stage("stem_conv"), plain.debug_stage("stem_conv"))


def _normalised(x_u8, mean=synth.RGB_MEANS, std=synth.RGB_STDS):
    """uint8 HWC -> NCHW fp32 with ToTensor + Normalize in fp32 true divisions (the stem's uint8 input stage)."""
    x = x_u8.cpu().permute(0, 3, 1, 2).float()
    m = torch.tensor(mean, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(std, dtype=torch.float32).view(1, 3, 1, 1)
    return ((x / 255.0) - m) / s


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 2, 3), (2, 17, 9), (1, 9, 30), (2, 64, 96), (1, 63, 65)],
                         ids=lambda s: "x".join(map(str, s)))
def test_stem_pool_op(shape, u8):
    """dirb200_stem_pool on tiny and odd shapes: equal to dirb200_stem_conv + dirb200_maxpool_3x3s2 where that accepts
    the shape (H, W >= 7), otherwise its stem map is checked per element against the fp64 reference and the pooled
    map must be its exact max."""
    from dirb200 import ops
    ops.require_gpu(0)
    sd = _sd()
    w = sd["conv1.weight"]
    s, sh = LM.bn_fold(sd, "bn1", 64)
    s_d, sh_d = torch.from_numpy(s).to(DEV), torch.from_numpy(sh).to(DEV)
    x = _input(shape, u8, seed=11)
    xf = _normalised(x).to(DEV).contiguous() if u8 else x
    ms = list(synth.RGB_MEANS) + list(synth.RGB_STDS)
    pooled, stem = ops.stem_pool(x, w, s_d, sh_d, mean_std=ms if u8 else None, stem_map=True)
    torch.cuda.synchronize()
    b, h, wd = shape
    ho, wo = (h - 1) // 2 + 1, (wd - 1) // 2 + 1
    assert tuple(stem.shape) == (b, ho, wo, 64) and tuple(pooled.shape) == (b, (ho - 1) // 2 + 1, (wo - 1) // 2 + 1, 64)
    assert torch.equal(pooled.cpu(), LM.maxpool_ref(stem.cpu()).to(pooled.dtype))
    if h >= 7 and wd >= 7:
        ref = ops.stem_conv(xf, w, s_d, sh_d)
        assert _same(stem, ref)
        assert _same(pooled, ops.maxpool_3x3s2(ref))
    else:
        rep = LM.check_conv("stem", stem, xf.half().permute(0, 2, 3, 1), w, 2, 3, s, sh, device=torch.device(DEV))
        assert rep.ok, rep.worst


def _level_ext(h, w, n):
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1        # stem conv 7x7/s2/p3
    for _ in range(n):                                # maxpool 3x3/s2/p1
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return h, w


@pytest.mark.parametrize("u8", [False, True], ids=["f32_nan_outside", "u8_bytes_outside"])
def test_ragged_batch(u8):
    sizes = [(300, 517), (33, 65), (517, 300), (97, 97), (300, 32)]
    hh, ww = max(h for h, _ in sizes), max(w for _, w in sizes)
    r = np.random.RandomState(3)
    if u8:
        slots = torch.from_numpy(r.randint(0, 256, (len(sizes), hh, ww, 3)).astype(np.uint8)).to(DEV)
        for i, (h, w) in enumerate(sizes):
            slots[i, :h, :w] = torch.from_numpy(synth.make_images_u8(1, h, w, seed=20 + i)[0]).to(DEV)
    else:
        slots = torch.full((len(sizes), 3, hh, ww), float("nan"), dtype=torch.float32, device=DEV)
        for i, (h, w) in enumerate(sizes):
            slots[i, :, :h, :w] = synth.make_images(1, h, w, seed=20 + i)[0].to(DEV)
    fused, plain = _nets(chunk=2)
    for net in (fused, plain):
        net.set_backend_option("debug_taps", 1)
    d1, h1 = fused.forward_ragged_slots(slots, sizes, want_f16=True)
    p1 = fused.debug_stage("stem")
    d0, h0 = plain.forward_ragged_slots(slots, sizes, want_f16=True)
    p0 = plain.debug_stage("stem")
    assert torch.isfinite(d1).all()
    assert _same(d1, d0) and _same(h1, h0)
    assert _same(p1, p0)
    # the taps hold the last pass (chunk 2): slots 4.. of the batch
    for j, i in enumerate(range(4, len(sizes))):
        eh, ew = _level_ext(*sizes[i], 1)
        assert not p1[j, eh:].view(torch.int16).any() and not p1[j, :, ew:].view(torch.int16).any()


def test_chunk_smaller_than_batch():
    fused, plain = _nets(chunk=2)
    x = _input((5, 130, 97), False, seed=9)
    assert _same(_forward_dev(fused, x, False)[0], _forward_dev(plain, x, False)[0])


def test_host_entry_points():
    fused, plain = _nets(host_chunk=2)
    x = synth.make_images(5, 96, 128, seed=12).numpy()
    assert np.array_equal(fused.forward_host(x), plain.forward_host(x))
    xu = synth.make_images_u8(5, 96, 128, seed=13)
    assert np.array_equal(fused.forward_host_u8(xu), plain.forward_host_u8(xu))


def test_u8_multiscale():
    fused, plain = _nets()
    x = torch.from_numpy(synth.make_images_u8(2, 160, 192, seed=14)).to(DEV)
    assert _same(fused.forward_u8_multiscale(x), plain.forward_u8_multiscale(x))
