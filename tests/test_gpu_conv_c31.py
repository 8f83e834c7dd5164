"""conv3 + residual of an identity Bottleneck and conv1 of the next one in one kernel (ops.conv_c31, conv_c31.cuh): the
block output and the next conv1 output equal the two single launches bit for bit, at the ResNet-101 stage shapes, on
tile counts that do not fill the last wave and on partial last tiles; in the network, ragged batches that take the
fused kernel equal one image at a time.  Needs an H100: -m gpu."""
import numpy as np
import pytest
import torch

from test_gpu_ragged import _alone_u8, _images, _net, _slots_u8

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _pair(ops, cm, b, h, w, seed):
    r = np.random.RandomState(seed)
    t2 = torch.from_numpy(np.maximum(r.standard_normal((b, h, w, cm)), 0).astype(np.float16)).to(DEV)
    x = torch.from_numpy(np.maximum(r.standard_normal((b, h, w, 4 * cm)), 0).astype(np.float16)).to(DEV)
    w3 = torch.from_numpy((r.standard_normal((4 * cm, cm, 1, 1)) * np.sqrt(2.0 / cm)).astype(np.float32))
    w1 = torch.from_numpy((r.standard_normal((cm, 4 * cm, 1, 1)) * np.sqrt(2.0 / (4 * cm))).astype(np.float32))
    s3 = torch.from_numpy(r.uniform(0.2, 0.4, 4 * cm).astype(np.float32)).to(DEV)
    h3 = torch.from_numpy((0.1 * r.standard_normal(4 * cm)).astype(np.float32)).to(DEV)
    s1 = torch.from_numpy(r.uniform(0.7, 1.3, cm).astype(np.float32)).to(DEV)
    h1 = torch.from_numpy((0.1 * r.standard_normal(cm)).astype(np.float32)).to(DEV)
    w3p, w1p = ops.pack_conv_weight(w3).to(DEV), ops.pack_conv_weight(w1).to(DEV)
    y, t1 = ops.conv_c31(t2, w3p, s3, h3, x, w1p, s1, h1)
    y2 = ops.conv_bn_act(t2, w3p, 4 * cm, 1, 1, 1, 0, s3, h3, x, True)
    t12 = ops.conv_bn_act(y2, w1p, cm, 1, 1, 1, 0, s1, h1, None, True)
    torch.cuda.synchronize()
    return y, t1, y2, t12


# ResNet-101 at 1024 x 1024: layer1 (Cm 64) at 256^2, layer2 (128) at 128^2, layer3 (256) at 64^2; B = 3 gives 1536 /
# 384 / 96 tiles (none a multiple of 132), B = 64 many tiles per CTA; 17 x 23 leaves a partial last tile.
@pytest.mark.parametrize("cm,hw", [(64, 256), (128, 128), (256, 64)])
@pytest.mark.parametrize("b", [1, 3, 64])
def test_conv_c31_equals_two_launches(cm, hw, b):
    ops = _ops()
    y, t1, y2, t12 = _pair(ops, cm, b, hw, hw, seed=cm + b)
    assert torch.equal(y, y2)
    assert torch.equal(t1, t12)


@pytest.mark.parametrize("cm,b,h,w", [(256, 1, 17, 23), (128, 5, 9, 31), (64, 2, 40, 3)])
def test_conv_c31_partial_tiles(cm, b, h, w):
    ops = _ops()
    y, t1, y2, t12 = _pair(ops, cm, b, h, w, seed=h * w)
    assert torch.equal(y, y2)
    assert torch.equal(t1, t12)


def test_ragged_batch_through_the_fused_kernel_equals_one_image_at_a_time():
    """Twelve pictures in 256 x 256-class slots: layer1 of the pass has 384 tiles and takes the fused kernel, a picture
    alone (32 tiles) takes the two launches; the fused epilogues zero every row outside a picture as the unfused ones."""
    net = _net("resnet50_rmac")
    rng = np.random.RandomState(5)
    sizes = [(int(rng.randint(160, 257)), int(rng.randint(160, 257))) for _ in range(12)]
    imgs = _images(sizes)
    slots, hw = _slots_u8(imgs)
    d, d16 = net.forward_ragged_slots(slots, hw, want_f16=True)
    for i, x in enumerate(imgs):
        a, a16 = _alone_u8(net, x)
        assert torch.equal(d[i], a), (i, hw[i])
        assert torch.equal(d16[i], a16), (i, hw[i])
