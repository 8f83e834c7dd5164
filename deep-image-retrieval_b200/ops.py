"""Torch-tensor front-end of the single operators of the C ABI (device memory + streams come from torch).

Every function takes CUDA tensors, hands raw pointers to libdirb200.so and launches on torch's
current stream.  Nothing here computes with torch.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import lib
from .inputs import check_norm_at_most_1


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def workspace(nbytes, device):
    """A device scratch buffer of nbytes (at least one, so that its pointer is never null)."""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def _chk(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise TypeError("%s must be a contiguous CUDA tensor of dtype %s" % (name, dtype))
    return t


def require_gpu(device=0):
    lib.call("dirb200_device_check", int(device))


def set_global_option(key, value):
    """Process-wide kernel selectors ('halo', 'pdl', 'head_fused'); include/dirb200.h."""
    lib.call("dirb200_set_global_option", key.encode(), float(value))


def get_global_option(key):
    v = C.c_double()
    lib.call("dirb200_get_global_option", key.encode(), C.byref(v))
    return v.value


def nchw_to_nhwc8(x):
    _chk(x, torch.float32, "x")
    b, c, h, w = x.shape
    assert c == 3
    out = torch.empty((b, h, w, 8), dtype=torch.float16, device=x.device)
    lib.call("dirb200_nchw_to_nhwc8", _ptr(x), b, h, w, _ptr(out), _stream())
    return out


def pack_conv_weight(w_oihw: torch.Tensor, cin_pad=None) -> torch.Tensor:
    """OIHW fp32 -> [Cout][KH][KW][CinPad] fp16, rows zero-padded to a multiple of 32 (the layout
    dirb200_conv_bn_act expects).  Host-side repack (weights are packed once)."""
    o, i, kh, kw = w_oihw.shape
    cp = cin_pad or i
    w = torch.zeros((o, kh, kw, cp), dtype=torch.float32)
    w[..., :i] = w_oihw.detach().float().cpu().permute(0, 2, 3, 1)
    k = kh * kw * cp
    kpad = (k + 31) // 32 * 32
    out = torch.zeros((o, kpad), dtype=torch.float16)
    out[:, :k] = w.reshape(o, k).half()
    return out


def conv_bn_act(x, w_packed, cout, kh, kw, stride, pad, scale, shift, res=None, relu=True, impl=0):
    """x NHWC fp16 (B,H,W,Cin) -> NHWC fp16 (B,Ho,Wo,Cout)."""
    _chk(x, torch.float16, "x")
    _chk(w_packed, torch.float16, "w_packed")
    _chk(scale, torch.float32, "scale")
    _chk(shift, torch.float32, "shift")
    b, h, w, cin = x.shape
    ho = (h + 2 * pad - kh) // stride + 1
    wo = (w + 2 * pad - kw) // stride + 1
    out = torch.empty((b, ho, wo, cout), dtype=torch.float16, device=x.device)
    if res is not None:
        _chk(res, torch.float16, "res")
        assert res.shape == out.shape
    lib.call("dirb200_conv_bn_act", _ptr(x), b, h, w, cin, _ptr(w_packed), cout, kh, kw, stride, pad, _ptr(scale),
             _ptr(shift), _ptr(res), int(bool(relu)), int(impl), _ptr(out), _stream())
    return out


def conv_c23(t1, w2_packed, scale2, shift2, w3_packed, scale3, shift3, res, variant=1):
    """Fused Bottleneck tail: relu(bn3(conv1x1(relu(bn2(conv3x3(t1))))) + res).  t1 NHWC fp16 (B,H,W,Cm) -> (B,H,W,4Cm)."""
    _chk(t1, torch.float16, "t1")
    _chk(res, torch.float16, "res")
    b, h, w, cm = t1.shape
    assert tuple(res.shape) == (b, h, w, 4 * cm)
    out = torch.empty_like(res)
    lib.call("dirb200_conv_c23", _ptr(t1), b, h, w, cm, _ptr(_chk(w2_packed, torch.float16, "w2")), _ptr(scale2), _ptr(shift2),
             _ptr(_chk(w3_packed, torch.float16, "w3")), _ptr(scale3), _ptr(shift3), _ptr(res), _ptr(out), int(variant), _stream())
    return out


def conv_c31(t2, w3_packed, scale3, shift3, x, w1_packed, scale1, shift1):
    """Identity Bottleneck b's conv3 and block b+1's conv1 in one kernel: y = relu(bn3(conv1x1(t2)) + x),
    t1 = relu(bn1(conv1x1(y))).  t2 NHWC fp16 (B,H,W,Cm), x (B,H,W,4Cm) -> (y, t1)."""
    _chk(t2, torch.float16, "t2")
    _chk(x, torch.float16, "x")
    b, h, w, cm = t2.shape
    assert tuple(x.shape) == (b, h, w, 4 * cm)
    y = torch.empty_like(x)
    t1 = torch.empty_like(t2)
    lib.call("dirb200_conv_c31", _ptr(t2), b, h, w, cm, _ptr(_chk(w3_packed, torch.float16, "w3")),
             _ptr(_chk(scale3, torch.float32, "scale3")), _ptr(_chk(shift3, torch.float32, "shift3")), _ptr(x), _ptr(y),
             _ptr(_chk(w1_packed, torch.float16, "w1")), _ptr(_chk(scale1, torch.float32, "scale1")),
             _ptr(_chk(shift1, torch.float32, "shift1")), _ptr(t1), _stream())
    return y, t1


def stem_conv(x_nchw, w_oihw, scale, shift):
    """Conv 7x7/s2/p3 (3->64) + BN + ReLU on tensor cores: NCHW fp32 (B,3,H,W) -> NHWC fp16 (B,Ho,Wo,64)."""
    _chk(x_nchw, torch.float32, "x_nchw")
    b, c, h, w = x_nchw.shape
    assert c == 3 and tuple(w_oihw.shape) == (64, 3, 7, 7)
    wh = np.ascontiguousarray(w_oihw.detach().cpu().numpy().astype(np.float32))
    w2 = np.empty((64, 256), dtype=np.float16)
    lib.call("dirb200_stem_pack_weight", wh.ctypes.data_as(C.c_void_p), w2.ctypes.data_as(C.c_void_p))
    w2d = torch.from_numpy(w2).to(x_nchw.device)
    ws = torch.empty(lib.raw("dirb200_stem_workspace_bytes")(b, h, w), dtype=torch.uint8, device=x_nchw.device)
    ho, wo = (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
    out = torch.empty((b, ho, wo, 64), dtype=torch.float16, device=x_nchw.device)
    lib.call("dirb200_stem_conv", _ptr(x_nchw), b, h, w, _ptr(w2d), _ptr(_chk(scale, torch.float32, "scale")),
             _ptr(_chk(shift, torch.float32, "shift")), _ptr(ws), _ptr(out), _stream())
    return out


def stem_pool(x, w_oihw, scale, shift, mean_std=None, stem_map=False):
    """Stem conv 7x7/s2/p3 + BN + ReLU + maxpool 3x3/s2 as one kernel: NCHW fp32 (B,3,H,W), or HWC uint8 (B,H,W,3)
    with mean_std = (mean[3], std[3]), -> NHWC fp16 (B,Hp,Wp,64); with stem_map also the stem map (B,Ho,Wo,64)."""
    u8 = x.dtype == torch.uint8
    _chk(x, torch.uint8 if u8 else torch.float32, "x")
    if u8:
        b, h, w, c = x.shape
        ms = np.ascontiguousarray(np.asarray(mean_std, dtype=np.float32).reshape(6))
    else:
        b, c, h, w = x.shape
        ms = None
    assert c == 3 and tuple(w_oihw.shape) == (64, 3, 7, 7)
    wh = np.ascontiguousarray(w_oihw.detach().cpu().numpy().astype(np.float32))
    w2 = np.empty((64, 256), dtype=np.float16)
    lib.call("dirb200_stem_pack_weight", wh.ctypes.data_as(C.c_void_p), w2.ctypes.data_as(C.c_void_p))
    w2d = torch.from_numpy(w2).to(x.device)
    ho, wo = (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
    hp, wp = (ho - 1) // 2 + 1, (wo - 1) // 2 + 1
    out = torch.empty((b, hp, wp, 64), dtype=torch.float16, device=x.device)
    stem = torch.empty((b, ho, wo, 64), dtype=torch.float16, device=x.device) if stem_map else None
    lib.call("dirb200_stem_pool", _ptr(x), int(u8), b, h, w, None if ms is None else ms.ctypes.data_as(C.c_void_p), _ptr(w2d),
             _ptr(_chk(scale, torch.float32, "scale")), _ptr(_chk(shift, torch.float32, "shift")), _ptr(out), _ptr(stem),
             _stream())
    return (out, stem) if stem_map else out


def resize_bilinear_u8(x_u8, size):
    """uint8 HWC CUDA tensor (B,H,W,3) -> (B,Ho,Wo,3), byte-identical to PIL Image.resize((Wo,Ho), BILINEAR)."""
    _chk(x_u8, torch.uint8, "x_u8")
    b, h, w, c = x_u8.shape
    assert c == 3
    ho, wo = int(size[0]), int(size[1])
    out = torch.empty((b, ho, wo, 3), dtype=torch.uint8, device=x_u8.device)
    lib.call("dirb200_resize_bilinear_u8", _ptr(x_u8), b, h, w, ho, wo, _ptr(out), _stream())
    return out


def resize_coeffs(in_size, out_size):
    """Host-only: PIL's fixed-point bilinear coefficient table of one axis -> (bounds [out,2], kk [out,ksize])."""
    ks = C.c_int()
    lib.call("dirb200_resize_coeffs", int(in_size), int(out_size), C.c_void_p(0), C.c_void_p(0), C.byref(ks))
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ks.value), dtype=np.int32)
    lib.call("dirb200_resize_coeffs", int(in_size), int(out_size), bounds.ctypes.data_as(C.c_void_p),
             kk.ctypes.data_as(C.c_void_p), C.byref(ks))
    return bounds, kk


def _bytes_ptr(buf):
    """(pointer, size, keep-alive) of a host byte buffer: a uint8 CPU tensor, bytes or a numpy array."""
    if isinstance(buf, torch.Tensor):
        t = buf.contiguous()
        return t.data_ptr(), t.numel(), t
    a = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else buf,
                             dtype=np.uint8)
    return a.ctypes.data, a.size, a


def jpeg_probe(buf):
    """Host-only header parse of a JPEG held in memory -> (status, info).  status 0: the GPU decoder takes it;
    DIRB200_ENOTSUP (-2): a JPEG it does not take; DIRB200_EINVAL (-1): not a (complete) JPEG.  info = dict(height,
    width, components, h_samp, v_samp, restart_interval, color, scan_bytes) as far as the header was read."""
    ptr, n, keep = _bytes_ptr(buf)
    info = (C.c_int * 8)()
    status = lib.raw("dirb200_jpeg_probe")(C.c_void_p(ptr), n, info)
    del keep
    keys = ("height", "width", "components", "h_samp", "v_samp", "restart_interval", "color", "scan_bytes")
    return status, dict(zip(keys, list(info)))


class JpegDecoder:
    """Batched baseline-JPEG decoder on one GPU, byte-identical to np.array(Image.open(f).convert("RGB"))."""

    def __init__(self, device=None, subseq_bits=None):
        self.device = torch.cuda.current_device() if device is None else int(device)
        h = C.c_void_p()
        lib.call("dirb200_jpeg_decoder_create", self.device, C.byref(h))
        self._h = h
        self.last_rounds = 0
        if subseq_bits is not None:
            self.set_option("subseq_bits", subseq_bits)

    def set_option(self, key, value):
        lib.call("dirb200_jpeg_decoder_set_option", self._h, key.encode(), float(value))

    def decode(self, bufs):
        """List of JPEG files in host memory (uint8 CPU tensors, bytes or arrays) -> (list of (h, w, 3) uint8 CUDA
        tensors, bool list ok).  One upload for the whole list.  ok[i] False: file i was refused by the header parser
        or its entropy-coded data did not decode cleanly; its tensor is then undefined (decode it with PIL)."""
        n = len(bufs)
        if n == 0:
            return [], []
        held = [_bytes_ptr(b) for b in bufs]
        shapes, offs, total = [], [], 0
        for ptr, size, _ in held:
            info = (C.c_int * 8)()
            st = lib.raw("dirb200_jpeg_probe")(C.c_void_p(ptr), size, info)
            h, w = (info[0], info[1]) if st == 0 else (0, 0)
            shapes.append((h, w))
            offs.append(total)
            total += h * w * 3
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(dev):
            out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            ptrs = (C.c_void_p * n)(*[p for p, _, _ in held])
            sizes = (C.c_size_t * n)(*[s for _, s, _ in held])
            offsets = (C.c_int64 * n)(*offs)
            rounds = C.c_int()
            lib.call("dirb200_jpeg_decoder_decode", self._h, n, ptrs, sizes, _ptr(out), offsets, _ptr(status), C.byref(rounds),
                     _stream())
            self.last_rounds = rounds.value
            ok = (status.cpu().numpy() == 0).tolist()
        del held
        imgs = [out[o:o + h * w * 3].view(h, w, 3) for o, (h, w) in zip(offs, shapes)]
        return imgs, ok

    def debug_coefficients(self, image):
        """int16 (nblocks, 64) coefficients of image `image` of the last decode (natural order, MCU order, DC
        prediction applied)."""
        nb = C.c_int()
        lib.call("dirb200_jpeg_debug_coefficients", self._h, int(image), C.c_void_p(0), 0, C.byref(nb), _stream())
        out = torch.empty((nb.value, 64), dtype=torch.int16, device=torch.device("cuda", self.device))
        lib.call("dirb200_jpeg_debug_coefficients", self._h, int(image), _ptr(out), out.numel() * 2, C.byref(nb),
                 _stream())
        return out

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            lib.raw("dirb200_jpeg_decoder_destroy")(h)
            self._h = None


def maxpool_3x3s2(x):
    _chk(x, torch.float16, "x")
    b, h, w, c = x.shape
    out = torch.empty((b, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=torch.float16, device=x.device)
    lib.call("dirb200_maxpool_3x3s2", _ptr(x), b, h, w, c, _ptr(out), _stream())
    return out


POOLING = {"gem": 0, "max": 1, "avg": 2}


def head_pool_fc_l2(feat, pooling="gem", p=3.0, eps=1e-6, norm_features=False, fc_w=None, fc_b=None, want_f16=False):
    """feat NHWC fp16 (B,h,w,C) -> (B,D) fp32 L2-normalised (rmac_resnet.py:59-68)."""
    _chk(feat, torch.float16, "feat")
    b, h, w, c = feat.shape
    out_dim = fc_w.shape[0] if fc_w is not None else c
    if fc_w is not None:
        _chk(fc_w, torch.float32, "fc_w")
        _chk(fc_b, torch.float32, "fc_b")
    nws = lib.raw("dirb200_head_workspace_floats")(b, h * w, c, out_dim)
    ws = torch.empty(nws, dtype=torch.float32, device=feat.device)
    desc = torch.empty((b, out_dim), dtype=torch.float32, device=feat.device)
    d16 = torch.empty((b, out_dim), dtype=torch.float16, device=feat.device) if want_f16 else None
    mode = POOLING["gem" if pooling.startswith("gem") else pooling]
    lib.call("dirb200_head_pool_fc_l2", _ptr(feat), b, h * w, c, mode, float(p), float(eps), int(bool(norm_features)),
             _ptr(fc_w), _ptr(fc_b), out_dim, _ptr(ws), _ptr(desc), _ptr(d16), _stream())
    return (desc, d16) if want_f16 else desc


def pool_scales(xs, pooling="mean", gemp=3, l2=True):
    """common.pool (+ F.normalize when l2): list of (N,D) fp32 CUDA tensors -> (N,D)."""
    if pooling not in ("mean", "gem"):
        raise ValueError("Bad pooling mode: " + str(pooling))
    stacked = torch.stack([_chk(x, torch.float32, "xs[i]") for x in xs], dim=0).contiguous()
    s, n, d = stacked.shape
    out = torch.empty((n, d), dtype=torch.float32, device=stacked.device)
    lib.call("dirb200_pool_scales", _ptr(stacked), s, n, d, 0 if pooling == "mean" else 1, float(gemp), int(bool(l2)),
             _ptr(out), _stream())
    return out


def center_bias(feat, b):
    """In place on an NHWC fp16 map: feat *= 1 + bilinear(align_corners=True) resize of the 4x4 map holding b on its
    central 2x2 (rmac_resnet.py:52-56).  Returns feat."""
    _chk(feat, torch.float16, "feat")
    n, h, w, c = feat.shape
    lib.call("dirb200_center_bias", _ptr(feat), n, h, w, c, float(b), _stream())
    return feat


def l2_normalize(x, eps=1e-12, want_f16=False):
    """Rows x / max(||x||, eps) in fp32 (eps 0: x / ||x||, NaN for a zero row), optionally with an fp16 copy equal to
    out.half().  The sum of squares is fp32: rows need 2^-63 < ||x|| < 2^64.  Below, the squares underflow (such a row
    is below any eps > 0 and comes out x / eps); above, the sum overflows and the row comes out 0."""
    _chk(x, torch.float32, "x")
    n, d = x.shape
    out = torch.empty_like(x)
    o16 = torch.empty((n, d), dtype=torch.float16, device=x.device) if want_f16 else None
    lib.call("dirb200_l2_normalize", _ptr(x), n, d, float(eps), _ptr(out), _ptr(o16), _stream())
    return (out, o16) if want_f16 else out


def f32_to_f16(x):
    _chk(x, torch.float32, "x")
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    lib.call("dirb200_f32_to_f16", _ptr(x), x.numel(), _ptr(out), _stream())
    return out


def whiten(x, comp, mean=None, colscale=None, l2norm=True, want_f16=False):
    """((x - mean) . comp^T) * colscale, row L2 (common.py:221-239).  x (N,D), comp (Dout,D) fp32 CUDA."""
    _chk(x, torch.float32, "x")
    _chk(comp, torch.float32, "comp")
    n, d = x.shape
    dout = comp.shape[0]
    y = torch.empty((n, dout), dtype=torch.float32, device=x.device)
    y16 = torch.empty((n, dout), dtype=torch.float16, device=x.device) if want_f16 else None
    lib.call("dirb200_whiten", _ptr(x), n, d, _ptr(comp), _ptr(mean), _ptr(colscale), dout, int(bool(l2norm)), _ptr(y),
             _ptr(y16), _stream())
    return (y, y16) if want_f16 else y


def scores_exact(q, db):
    """Dense exact scores (Q,N) fp32 = q . db^T (fp64 accumulation).  Any D: the kernel reads rows as float4, so both
    operands are zero-padded to a multiple of 4 columns (zero columns change no score)."""
    _chk(q, torch.float32, "q")
    _chk(db, torch.float32, "db")
    if q.shape[1] != db.shape[1]:
        raise ValueError("descriptor dimensions differ: %d vs %d" % (q.shape[1], db.shape[1]))
    pad = (-q.shape[1]) % 4
    if pad:
        q = torch.nn.functional.pad(q, (0, pad)).contiguous()
        db = torch.nn.functional.pad(db, (0, pad)).contiguous()
    out = torch.empty((q.shape[0], db.shape[0]), dtype=torch.float32, device=q.device)
    lib.call("dirb200_scores_exact", _ptr(q), q.shape[0], _ptr(db), db.shape[0], q.shape[1], _ptr(out), _stream())
    return out


def _pad4(x):
    """(N,D) fp32 -> (N,D') with D' = D rounded up to a multiple of 4 (zero columns), and D."""
    d = x.shape[1]
    pad = (-d) % 4
    return (torch.nn.functional.pad(x, (0, pad)).contiguous() if pad else x), d


def col_sums_f64(x, out=None):
    """Column sums of x (N,D) fp32 CUDA in fp64, in a fixed order (bit-identical on every run).  out: optional (D,)
    fp64 CUDA buffer the sums are ADDED to (rows fed in chunks); returned."""
    _chk(x, torch.float32, "x")
    xp, d = _pad4(x)
    if out is None:
        out = torch.zeros(d, dtype=torch.float64, device=x.device)
    _chk(out, torch.float64, "out")
    if tuple(out.shape) != (d,):
        raise ValueError("out must have shape (%d,)" % d)
    buf = out if xp.shape[1] == d else torch.nn.functional.pad(out, (0, xp.shape[1] - d)).contiguous()
    lib.call("dirb200_col_sums_f64", _ptr(xp), xp.shape[0], xp.shape[1], _ptr(buf), _stream())
    if buf is not out:
        out.copy_(buf[:d])
    return out


def gram_f64(x, mean, out=None):
    """Centred Gram matrix G += (x - mean)^T (x - mean), fp64 (D,D), the centring done in fp64; x (N,D) fp32, mean (D,)
    fp64, CUDA.  out: optional (D,D) fp64 CUDA buffer the Gram is ADDED to (rows fed in chunks); returned.  Any D up
    to 8064: other D than multiples of 4 go through zero columns (zero mean), which add nothing."""
    _chk(x, torch.float32, "x")
    _chk(mean, torch.float64, "mean")
    xp, d = _pad4(x)
    if tuple(mean.shape) != (d,):
        raise ValueError("mean must have shape (%d,)" % d)
    if out is None:
        out = torch.zeros((d, d), dtype=torch.float64, device=x.device)
    _chk(out, torch.float64, "out")
    if tuple(out.shape) != (d, d):
        raise ValueError("out must have shape (%d, %d)" % (d, d))
    dp = xp.shape[1]
    if dp != d:
        mean = torch.nn.functional.pad(mean, (0, dp - d)).contiguous()
        buf = torch.nn.functional.pad(out, (0, dp - d, 0, dp - d)).contiguous()
    else:
        buf = out
    lib.call("dirb200_gram_f64", _ptr(xp), xp.shape[0], dp, _ptr(mean), _ptr(buf), _stream())
    if buf is not out:
        out.copy_(buf[:d, :d])
    return out


APLOSS_MODES = {"ap": 0, "tap": 1, "taps": 2}


def _aploss_args(x, label, nq, table):
    _chk(x, torch.float32, "x")
    _chk(label, torch.uint8, "label")
    _chk(table, torch.float32, "table")
    if x.dim() != 2 or tuple(label.shape) != tuple(x.shape):
        raise ValueError("x and label must be (N, M) tensors of the same shape")
    if table.numel() != 4 * nq:
        raise ValueError("table must hold 4 nq = %d values" % (4 * nq))
    return x.shape


def aploss_forward(x, label, nq, table, mode):
    """Per-row AP of the quantised scores (dirb200_aploss_forward).  x (N,M) fp32, label (N,M) uint8, table the 2nq
    weights then 2nq biases of the quantiser, mode 'ap' / 'tap' / 'taps'.  Returns (hist (N,2nq+1) int64 in units of
    2^-32, G (N,2nq) fp64 = [dAP/dc | dAP/dcp], ap (N,) fp32)."""
    n, m = _aploss_args(x, label, nq, table)
    hist = torch.empty((n, 2 * nq + 1), dtype=torch.int64, device=x.device)
    G = torch.empty((n, 2 * nq), dtype=torch.float64, device=x.device)
    ap = torch.empty(n, dtype=torch.float32, device=x.device)
    lib.call("dirb200_aploss_forward", _ptr(x), _ptr(label), n, m, int(nq), _ptr(table), APLOSS_MODES[mode],
             _ptr(hist), _ptr(G), _ptr(ap), _stream())
    return hist, G, ap


def aploss_backward(x, label, nq, table, G, grad_ap):
    """dx (N,M) fp32 = grad_ap[n] * sum_j (G_c + l G_cp)[n][j] dq_j/dx (dirb200_aploss_backward)."""
    n, m = _aploss_args(x, label, nq, table)
    _chk(G, torch.float64, "G")
    _chk(grad_ap, torch.float32, "grad_ap")
    if tuple(G.shape) != (n, 2 * nq) or tuple(grad_ap.shape) != (n,):
        raise ValueError("G must be (N, 2nq) and grad_ap (N,)")
    dx = torch.empty((n, m), dtype=torch.float32, device=x.device)
    lib.call("dirb200_aploss_backward", _ptr(x), _ptr(label), n, m, int(nq), _ptr(table), _ptr(G), _ptr(grad_ap),
             _ptr(dx), _stream())
    return dx


def topk_merge(scores, idx, k):
    """scores/idx: (G,Q,k) fp64 / int64 per-shard lists with global indices -> merged (Q,k)."""
    _chk(scores, torch.float64, "scores")
    _chk(idx, torch.int64, "idx")
    g, q, kk = scores.shape
    assert kk == k
    os_ = torch.empty((q, k), dtype=torch.float64, device=scores.device)
    oi = torch.empty((q, k), dtype=torch.int64, device=scores.device)
    lib.call("dirb200_topk_merge", _ptr(scores), _ptr(idx), g, q, k, 0, _ptr(os_), _ptr(oi), _stream())
    return os_, oi


def topk_merge_packed(packed, k):
    """packed: (G,2,Q,k) int64 all-gather buffer, [:,0] = fp64 score bits, [:,1] = global indices -> merged (Q,k)."""
    _chk(packed, torch.int64, "packed")
    g, two, q, kk = packed.shape
    assert two == 2 and kk == k
    os_ = torch.empty((q, k), dtype=torch.float64, device=packed.device)
    oi = torch.empty((q, k), dtype=torch.int64, device=packed.device)
    base = packed.data_ptr()
    lib.call("dirb200_topk_merge", C.c_void_p(base), C.c_void_p(base + q * k * 8), g, q, k, 2 * q * k, _ptr(os_),
             _ptr(oi), _stream())
    return os_, oi


def aqe_expand(q, db32, nn_idx, nn_scores, alpha, partial=False, row_offset=0, n_rows=0):
    _chk(q, torch.float32, "q")
    _chk(db32, torch.float32, "db32")
    _chk(nn_idx, torch.int64, "nn_idx")
    _chk(nn_scores, torch.float64, "nn_scores")
    out = torch.empty_like(q)
    lib.call("dirb200_aqe_expand", _ptr(q), q.shape[0], q.shape[1], _ptr(db32), _ptr(nn_idx), _ptr(nn_scores),
             nn_idx.shape[1], float(alpha), int(bool(partial)), int(row_offset), int(n_rows), _ptr(out), _stream())
    return out


def allow_rows(mask: torch.Tensor) -> torch.Tensor:
    """Allow set of a filtered search (DESIGN.md section 4.13, rule F1) from a bool mask (..., N): row r is bit r & 31 of
    int32 word r >> 5 -> (..., ceil(N / 32)) int32 words, on the mask's device."""
    if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or mask.dim() < 1:
        raise ValueError("mask must be a bool tensor (..., N)")
    n = mask.shape[-1]
    w = (n + 31) // 32
    bits = torch.zeros(mask.shape[:-1] + (32 * w,), dtype=torch.int64, device=mask.device)
    bits[..., :n] = mask.to(torch.int64)
    weights = torch.ones(32, dtype=torch.int64, device=mask.device) << torch.arange(32, device=mask.device)
    words = (bits.view(mask.shape[:-1] + (w, 32)) * weights).sum(dim=-1)
    return torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32).contiguous()


def allow_exclude(base: torch.Tensor, n_queries: int, rows_per_query) -> torch.Tensor:
    """Per-query allow sets (Q, W) = the shared set base (W,) int32 CUDA words with each query's rows cleared
    (dirb200_allow_exclude): leave-one-out when the queries are database rows, per-query junk lists.  rows_per_query:
    Q sequences of global row numbers in [0, 32 W)."""
    _chk(base, torch.int32, "base")
    if base.dim() != 1:
        raise ValueError("base must be one shared allow set (W,)")
    nq = int(n_queries)
    lists = [np.asarray(r, dtype=np.int64).reshape(-1) for r in rows_per_query]
    if len(lists) != nq:
        raise ValueError("rows_per_query must hold %d lists (got %d)" % (nq, len(lists)))
    w = base.shape[0]
    rows = np.concatenate(lists) if lists else np.zeros(0, np.int64)
    if rows.size and (rows.min() < 0 or rows.max() >= 32 * w):
        raise ValueError("excluded rows must lie in [0, %d)" % (32 * w))
    off = np.zeros(nq + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in lists])
    out = base.unsqueeze(0).expand(nq, w).contiguous()
    if nq == 0 or rows.size == 0:
        return out
    off_d = torch.from_numpy(off).to(base.device)
    rows_d = torch.from_numpy(rows).to(base.device)
    with torch.cuda.device(base.device):
        lib.call("dirb200_allow_exclude", _ptr(out), nq, w, _ptr(off_d), _ptr(rows_d), _stream())
    return out


class Exchange:
    """This rank's window of the peer-memory exchange of a sharded search (include/dirb200.h: dirb200_exchange_*)."""

    def __init__(self, device_index: int, world: int, rank: int, max_q: int, max_k: int):
        self.world, self.rank, self.max_q, self.max_k = int(world), int(rank), int(max_q), int(max_k)
        self._h = C.c_void_p()
        lib.call("dirb200_exchange_create", int(device_index), self.world, self.rank, self.max_q, self.max_k, C.byref(self._h))

    def ipc_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        lib.call("dirb200_exchange_ipc_handle", self._h, buf)
        return buf.raw

    def open(self, handles) -> None:
        """handles: the 64-byte IPC handles of all ranks in rank order (this rank's own entry is ignored)."""
        blob = b"".join(bytes(h) for h in handles)
        assert len(blob) == 64 * self.world
        lib.call("dirb200_exchange_open", self._h, C.c_char_p(blob))

    @staticmethod
    def open_local(group) -> None:
        """Same-process group: `group` = the exchange objects of all ranks, in rank order."""
        arr = (C.c_void_p * len(group))(*[x._h for x in group])
        for x in group:
            lib.call("dirb200_exchange_open_local", x._h, arr)

    def close_peers(self):
        """Unmap the other ranks' windows (every rank, then a barrier, then close())."""
        if self._h:
            lib.call("dirb200_exchange_close_peers", self._h)

    def close(self):
        if self._h:
            lib.raw("dirb200_exchange_destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Index:
    """One row shard of a descriptor database on one GPU (dirb200_index)."""

    def __init__(self, db32: torch.Tensor, index_offset: int = 0, db16: torch.Tensor = None, check_norms: bool = True):
        """check_norms: the exactness of the top-k rests on |fp16-path score - exact score| <= eps16 = 1.2e-3, which is
        derived for UNIT-NORM rows and queries (what pooling / whitening / query expansion produce).  Rows with larger
        norms are refused here instead of silently returning an inexact list.  To search un-normalised data, either
        scale queries and rows to unit norm (the order does not change), or pass check_norms=False and set option
        'eps16' to 1.2e-3 * max|q| * max|row| + 2^-24 * sqrt(D) * (max|q| + max|row|) (norms of queries and rows, D the
        dimension): below 2^-14 fp16 is subnormal and rounds to an absolute 2^-25 per entry, which the first term
        alone does not cover for small norms.  Every entry must stay below fp16's largest value, 65504."""
        _chk(db32, torch.float32, "db32")
        if check_norms:
            check_norm_at_most_1(db32, "database")
        self.db32 = db32
        self.n, self.dim = db32.shape
        if db16 is None:                      # an empty shard (more ranks than rows) has nothing to convert
            db16 = f32_to_f16(db32) if self.n else torch.empty((0, self.dim), dtype=torch.float16, device=db32.device)
        self.db16 = db16
        self.offset = int(index_offset)
        # rows numbered by the allow sets of a filtered search: a shard searched together with others (dist.ShardedIndex,
        # or the phases driven by hand) sets it to the rows of the whole database
        self.n_global = self.offset + self.n
        self._h = C.c_void_p()
        lib.call("dirb200_index_create", db32.device.index or 0, self.dim, C.byref(self._h))
        lib.call("dirb200_index_set_db", self._h, _ptr(self.db32), _ptr(self.db16), self.n, self.offset)

    def set_option(self, key, value):
        lib.call("dirb200_index_set_option", self._h, key.encode(), float(value))

    def _allow_ld(self, allow, nq):
        """Checks an allow set (rule F1) against this index and nq queries -> words per query row (0 = shared)."""
        if allow is None:
            return None
        w = (self.n_global + 31) // 32
        if not isinstance(allow, torch.Tensor) or allow.dtype != torch.int32:
            raise ValueError("allow must be an int32 tensor of bitmap words (ops.allow_rows)")
        if not allow.is_cuda or allow.device != self.db32.device:
            raise ValueError("allow must live on the index's device %s" % self.db32.device)
        if not allow.is_contiguous():
            raise ValueError("allow must be contiguous")
        if allow.dim() == 1 and allow.shape[0] == w:
            return 0
        if allow.dim() == 2 and allow.shape[1] == w:
            if allow.shape[0] != nq:
                raise ValueError("a per-query allow set needs one row per query (%d), got %d" % (nq, allow.shape[0]))
            return w
        raise ValueError("allow must be (%d,) or (Q, %d) words for %d rows, got %s" % (w, w, self.n_global, tuple(allow.shape)))

    def _set_allow(self, allow, ld):
        lib.call("dirb200_index_set_allow", self._h, _ptr(allow), 0 if ld is None else ld, self.offset)

    def search(self, q32: torch.Tensor, k: int, out=None, allow=None):
        """-> (scores fp64 (Q,k), idx int64 (Q,k)), exact order: score desc, index asc.
        out: optional (2,Q,k) int64 buffer that receives [score bits, indices] (the all-gather payload).
        allow: filtered search (DESIGN.md section 4.13): int32 CUDA words of one allow set (W,) shared by every query or
        one per query (Q, W), W = ceil(rows / 32) in global row numbering (ops.allow_rows, ops.allow_exclude); each
        query gets the exact top-k of its allowed rows, tail (-inf, -1).  Per-query sets take Q * W * 4 bytes (125 MB
        for 1000 queries over 2^20 rows): pass very large Q in blocks."""
        _chk(q32, torch.float32, "q32")
        nq = q32.shape[0]
        ld = self._allow_ld(allow, nq)
        if ld is None:
            return self._search(q32, k, out)
        self._set_allow(allow, ld)
        try:
            return self._search(q32, k, out)
        finally:
            self._set_allow(None, None)

    def _search(self, q32, k, out):
        nq = q32.shape[0]
        if out is not None:
            _chk(out, torch.int64, "out")
            assert tuple(out.shape) == (2, nq, k)
            scores, idx = out[0].view(torch.float64), out[1]
        else:
            scores = torch.empty((nq, k), dtype=torch.float64, device=q32.device)
            idx = torch.empty((nq, k), dtype=torch.int64, device=q32.device)
        try:
            lib.call("dirb200_index_search", self._h, _ptr(q32), nq, int(k), _ptr(scores), _ptr(idx), _stream())
        except lib.DirbError as e:
            if e.status != -4:                      # DIRB200_EOVERFLOW: candidate lists did not fit after the retry passes
                raise
            # rare (clustered databases whose first rows are not a sample of the rest): run again with more gated
            # retry passes and a larger candidate buffer, then restore the defaults
            self.set_option("retries", 4)
            self.set_option("cand_cap", 1 << 17)
            try:
                lib.call("dirb200_index_search", self._h, _ptr(q32), nq, int(k), _ptr(scores), _ptr(idx), _stream())
                lib.call("dirb200_index_check", self._h)
            finally:
                self.set_option("retries", 1)
                self.set_option("cand_cap", 0)
        return scores, idx

    def search_max_queries(self, k: int) -> int:
        """Most queries one search_begin of depth k takes within option 'ws_budget' (search() splits larger Q itself)."""
        out = C.c_int()
        lib.call("dirb200_index_search_max_queries", self._h, int(k), C.byref(out))
        return int(out.value)

    def search_begin(self, q32: torch.Tensor, k: int, k_shard: int, allow=None):
        """Phase 1 of a sharded search -> sel (Q,) fp32: local k_shard-th best fp16-path score (MIN-reduce it).
        allow: the filter of search(), applied by this search through its search_finish."""
        _chk(q32, torch.float32, "q32")
        ld = self._allow_ld(allow, q32.shape[0])
        sel = torch.empty(q32.shape[0], dtype=torch.float32, device=q32.device)
        if ld is not None:
            self._set_allow(allow, ld)
        try:
            lib.call("dirb200_index_search_begin", self._h, _ptr(q32), q32.shape[0], int(k), int(k_shard), _ptr(sel), _stream())
        finally:
            if ld is not None:
                self._set_allow(None, None)
        return sel

    def search_finish(self, q32: torch.Tensor, k: int, sel: torch.Tensor, out=None):
        """Phase 2: exact re-scoring of the rows within the band of the (reduced) threshold -> ordered local list."""
        nq = q32.shape[0]
        if out is not None:
            scores, idx = out[0].view(torch.float64), out[1]
        else:
            scores = torch.empty((nq, k), dtype=torch.float64, device=q32.device)
            idx = torch.empty((nq, k), dtype=torch.int64, device=q32.device)
        lib.call("dirb200_index_search_finish", self._h, _ptr(q32), _ptr(_chk(sel, torch.float32, "sel")), _ptr(scores),
                 _ptr(idx), _stream())
        return scores, idx

    def search_sharded(self, exchange: "Exchange", q32: torch.Tensor, k: int, k_shard: int, phase: int = 0, allow=None):
        """Collective exact top-k over all shards through the peer-memory exchange (no library collective): every rank
        calls it with the same (Q, k, k_shard).  phase 0 = the whole search; 1 .. 4 = one phase (seed bounds, filter +
        selection, re-scoring, merge: several shards driven shard by shard from one process).
        -> (scores fp64, idx int64) (Q,k) after phase 0 / 4, else None.
        allow: the filter of search() in global row numbering, the same on every rank; read by phase 0 / 1 (the later
        phases use what their search began with).
        Never synchronises: call check() (or the next search) to collect the status."""
        _chk(q32, torch.float32, "q32")
        ld = self._allow_ld(allow, q32.shape[0]) if phase in (0, 1) else None
        if ld is None:
            return self._search_sharded(exchange, q32, k, k_shard, phase)
        self._set_allow(allow, ld)
        try:
            return self._search_sharded(exchange, q32, k, k_shard, phase)
        finally:
            self._set_allow(None, None)

    def _search_sharded(self, exchange, q32, k, k_shard, phase):
        nq = q32.shape[0]
        scores = idx = None
        if phase in (0, 4):
            scores = torch.empty((nq, k), dtype=torch.float64, device=q32.device)
            idx = torch.empty((nq, k), dtype=torch.int64, device=q32.device)
        if phase == 0:
            lib.call("dirb200_index_search_sharded", self._h, exchange._h, _ptr(q32), nq, int(k), int(k_shard), _ptr(scores),
                     _ptr(idx), _stream())
        else:
            lib.call("dirb200_index_search_sharded_phase", self._h, exchange._h, int(phase), _ptr(q32), nq, int(k), int(k_shard),
                     _ptr(scores), _ptr(idx), _stream())
        return (scores, idx) if scores is not None else None

    def target_scores(self, q32, t_q, t_rows):
        """Exact scores <q32[t_q[t]], db[t_rows[t]]> (fp64) of the target rows this shard owns, 0 for the others.
        t_q int32 (T,), t_rows int64 (T,) global indices - CUDA tensors."""
        _chk(q32, torch.float32, "q32")
        _chk(t_q, torch.int32, "t_q")
        _chk(t_rows, torch.int64, "t_rows")
        out = torch.zeros(t_rows.shape[0], dtype=torch.float64, device=q32.device)
        lib.call("dirb200_index_target_scores", self._h, _ptr(q32), q32.shape[0], _ptr(t_q), _ptr(t_rows), t_rows.shape[0],
                 _ptr(out), _stream())
        return out

    def rank_count(self, q32, t_off, t_rows, t_flags, t_score):
        """above[t] = number of rows of this shard ranking before target t (exact score desc, ties -> lower index) for
        the flagged targets of each query.  t_off: host int32 ndarray (Q+1,), the CSR offsets of the targets; t_rows
        int64 / t_flags uint8 / t_score fp64 CUDA tensors (T,)."""
        _chk(q32, torch.float32, "q32")
        _chk(t_rows, torch.int64, "t_rows")
        _chk(t_flags, torch.uint8, "t_flags")
        _chk(t_score, torch.float64, "t_score")
        off_h = np.ascontiguousarray(t_off, dtype=np.int32)
        assert off_h.shape[0] == q32.shape[0] + 1
        off_d = torch.from_numpy(off_h).to(q32.device)
        above = torch.zeros(t_rows.shape[0], dtype=torch.int64, device=q32.device)
        lib.call("dirb200_index_rank_count", self._h, _ptr(q32), q32.shape[0], off_h.ctypes.data_as(C.c_void_p), _ptr(off_d),
                 _ptr(t_rows), _ptr(t_flags), _ptr(t_score), t_rows.shape[0], _ptr(above), _stream())
        return above

    def rank_counts(self, q32, t_off, t_rows, t_flags):
        """Single-shard convenience: (exact scores fp64 (T,), rows ranking before each flagged target int64 (T,))."""
        off = np.ascontiguousarray(t_off, dtype=np.int32)
        t_q = torch.from_numpy(np.repeat(np.arange(q32.shape[0], dtype=np.int32), np.diff(off))).to(q32.device)
        rows = torch.as_tensor(np.ascontiguousarray(t_rows, dtype=np.int64)).to(q32.device)
        flags = torch.as_tensor(np.ascontiguousarray(t_flags, dtype=np.uint8)).to(q32.device)
        sc = self.target_scores(q32, t_q, rows)
        return sc, self.rank_count(q32, off, rows, flags, sc)

    def count_ge(self, q32, thr_off, thr, skip_row=None):
        """count[t] = number of rows of this shard (global index != skip_row[q]) whose fp32-rounded exact score with
        query q reaches thr[t], for the thresholds thr[thr_off[q]:thr_off[q+1]] of each query (descending) - what
        label AP needs (datasets.ImageListLabels.eval_query_AP_from_ge_counts).  thr_off int32 (Q+1,), thr fp32 (T,),
        skip_row int64 (Q,) or None: CUDA tensors.  Afterwards stats()["candidates"] = pairs re-scored exactly
        (within eps of a boundary) and stats()["retries"] = queries counted exactly over all rows (band overflow)."""
        _chk(q32, torch.float32, "q32")
        _chk(thr_off, torch.int32, "thr_off")
        _chk(thr, torch.float32, "thr")
        if skip_row is not None:
            _chk(skip_row, torch.int64, "skip_row")
            assert skip_row.shape[0] == q32.shape[0]
        assert thr_off.shape[0] == q32.shape[0] + 1
        count = torch.zeros(thr.shape[0], dtype=torch.int64, device=q32.device)
        lib.call("dirb200_index_count_ge", self._h, _ptr(q32), q32.shape[0], _ptr(thr_off), _ptr(thr), thr.shape[0],
                 _ptr(skip_row), _ptr(count), _stream())
        return count

    def _join_result(self, rows, total):
        off = torch.empty(rows + 1, dtype=torch.int64, device=self.db32.device)
        idx = torch.empty(total, dtype=torch.int64, device=self.db32.device)
        sc = torch.empty(total, dtype=torch.float64, device=self.db32.device)
        lib.call("dirb200_index_join_fetch", self._h, _ptr(off), _ptr(idx), _ptr(sc), _stream())
        return off, idx, sc

    def range_search(self, q32: torch.Tensor, tau: float):
        """Every row with exact score >= tau for each query (DESIGN.md section 4.8, rule J2) -> CSR (offsets int64 (Q+1,),
        rows int64, scores fp64), each list ordered by (score desc, row asc); the same rows and score bits as the prefix
        of search(q32, N) down to its last score >= tau.  Exact for any tau, however many rows match."""
        _chk(q32, torch.float32, "q32")
        total = C.c_int64()
        lib.call("dirb200_index_range_search", self._h, _ptr(q32), q32.shape[0], float(tau), C.byref(total), _stream())
        return self._join_result(q32.shape[0], total.value)

    def self_join(self, tau: float, row_block: int = None):
        """Every pair (i, j), i < j, of the index's rows with exact score >= tau (rule J3) -> CSR by i (offsets int64
        (N+1,), partners j int64, scores fp64), partners ordered by (score desc, j asc): range_search(db, tau) without
        the entries j <= i.  Only the tiles on or above the diagonal of X X^T run on the tensor cores.  row_block (a
        multiple of 128): rows joined per call, whose results are concatenated (the result does not depend on it)."""
        n = self.n
        if row_block is not None and (int(row_block) <= 0 or int(row_block) % 128):
            raise ValueError("row_block must be a positive multiple of 128 (got %r)" % (row_block,))
        step = int(row_block) if row_block is not None else max(n, 1)
        offs, idxs, scs = [], [], []
        base = 0
        for r0 in range(0, max(n, 1), step):
            r1 = min(n, r0 + step)
            total = C.c_int64()
            lib.call("dirb200_index_self_join", self._h, r0, r1, float(tau), C.byref(total), _stream())
            off, idx, sc = self._join_result(r1 - r0, total.value)
            offs.append(off[:-1] + base if r1 < n else off + base)
            idxs.append(idx)
            scs.append(sc)
            base += total.value
        return torch.cat(offs), torch.cat(idxs), torch.cat(scs)

    def nearest(self, q32: torch.Tensor):
        """Exact nearest row of each query (DESIGN.md section 4.9, rules K2 / K3) -> (labels int64 (Q,), scores fp64
        (Q,)): the top-1 of search(q32, 1) bit for bit, from group maxima of the fp16 tensor-core pass and exact
        re-scoring of the groups within 2 eps16 of the best (all rows past option 'nearest_cap' groups)."""
        _chk(q32, torch.float32, "q32")
        if q32.dim() != 2 or q32.shape[1] != self.dim:
            raise ValueError("queries must be (Q, %d)" % self.dim)
        nq = q32.shape[0]
        labels = torch.empty(nq, dtype=torch.int64, device=q32.device)
        scores = torch.empty(nq, dtype=torch.float64, device=q32.device)
        lib.call("dirb200_index_nearest", self._h, _ptr(q32), nq, _ptr(labels), _ptr(scores), _stream())
        return labels, scores

    def nearest_stats(self):
        """Counters of the last nearest(): band_rows (queries with more than one candidate group), full_rescores
        (queries re-scored over all rows), rescored (rows re-scored in all)."""
        st = (C.c_int64 * 3)()
        lib.call("dirb200_index_nearest_stats", self._h, st)
        return dict(zip(["band_rows", "full_rescores", "rescored"], [int(v) for v in st]))

    def set_lists(self, db16_lists, perm, cell_off):
        """Attach inverted lists (DESIGN.md section 4.10, rule I2): db16_lists fp16 (N, D) = the rows in list order,
        perm int64 (N,) = list position -> row, cell_off int64 (K + 1,) = list boundaries (CUDA tensors, kept alive
        by the index).  Exact search, rank counts and the options keep working on the original-order rows."""
        _chk(db16_lists, torch.float16, "db16_lists")
        _chk(perm, torch.int64, "perm")
        _chk(cell_off, torch.int64, "cell_off")
        if tuple(db16_lists.shape) != (self.n, self.dim) or perm.shape[0] != self.n or cell_off.dim() != 1:
            raise ValueError("lists must hold the index's %d rows of dimension %d" % (self.n, self.dim))
        self._lists = (db16_lists, perm, cell_off)
        lib.call("dirb200_index_set_lists", self._h, _ptr(db16_lists), _ptr(perm), _ptr(cell_off), cell_off.shape[0] - 1,
                 _stream())

    def search_lists(self, q32: torch.Tensor, k: int, probes: torch.Tensor):
        """Exact top-k of the union of the lists each query probes (rules I3-I6) -> (scores fp64 (Q,k), idx int64 (Q,k)),
        order score desc, row asc, tail (-inf, -1) when the union holds fewer than k rows.  probes int64 (Q, nprobe)."""
        _chk(q32, torch.float32, "q32")
        _chk(probes, torch.int64, "probes")
        nq = q32.shape[0]
        if probes.dim() != 2 or probes.shape[0] != nq:
            raise ValueError("probes must be (Q, nprobe)")
        scores = torch.empty((nq, k), dtype=torch.float64, device=q32.device)
        idx = torch.empty((nq, k), dtype=torch.int64, device=q32.device)
        lib.call("dirb200_index_search_lists", self._h, _ptr(q32), nq, int(k), _ptr(probes), probes.shape[1], _ptr(scores),
                 _ptr(idx), _stream())
        return scores, idx

    def lists_stats(self):
        """Counters (and, with option 'profile', CUDA-event milliseconds per stage) of the last search_lists."""
        st = (C.c_int64 * 6)()
        ms = (C.c_double * 4)()
        lib.call("dirb200_index_lists_stats", self._h, st, ms)
        out = dict(zip(["pairs", "query_rows", "tiles", "probed_rows", "candidates", "reruns"], [int(v) for v in st]))
        out.update(zip(["build_ms", "gmax_ms", "filter_ms", "finish_ms"], [float(v) for v in ms]))
        return out

    def join_stats(self):
        """Counters (and, with option 'profile', CUDA-event milliseconds per stage) of the last range_search / self_join."""
        st = (C.c_int64 * 5)()
        ms = (C.c_double * 3)()
        lib.call("dirb200_index_join_stats", self._h, st, ms)
        out = dict(zip(["candidates", "pairs", "reruns", "filter_launches", "tiles"], [int(v) for v in st]))
        out.update(zip(["filter_ms", "rescore_ms", "sort_ms"], [float(v) for v in ms]))
        return out

    def check(self):
        """Collect the status of the last search (option deferred_check): raises DirbError on an unresolved overflow."""
        lib.call("dirb200_index_check", self._h)

    def stats(self):
        arr = (C.c_int64 * 5)()
        lib.call("dirb200_index_last_stats", self._h, arr)
        return dict(zip(["dense_rows", "candidates", "survivors", "retries", "launches"], [int(v) for v in arr]))

    def profile(self):
        arr = (C.c_double * 9)()
        lib.call("dirb200_index_last_profile", self._h, arr)
        names = ["prep", "seed_gemm", "seed_kth", "filter_gemm", "cand_select", "retry_gates", "finish"]
        out = {n: float(arr[i]) for i, n in enumerate(names)}
        if arr[7] or arr[8]:                        # k > 1024: the finish in three steps
            out.update(finish=arr[6] + arr[7] + arr[8], finish_compact=arr[6], finish_rescore=arr[7], finish_sort=arr[8])
        return out

    def close(self):
        if self._h:
            lib.raw("dirb200_index_destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def join_components(off, cols, n):
    """Connected components of the undirected graph of n rows given as a CSR (off int64 (n+1,), cols int64; CUDA
    tensors) -> labels int64 (n,): the smallest row of each row's component (DESIGN.md section 4.8, rule J4)."""
    n = int(n)
    if n < 1:
        return torch.empty(0, dtype=torch.int64, device=off.device)
    _chk(off, torch.int64, "off")
    _chk(cols, torch.int64, "cols")
    if off.shape[0] != n + 1:
        raise ValueError("off must have n + 1 entries")
    labels = torch.empty(n, dtype=torch.int64, device=off.device)
    ws = torch.empty(int(lib.raw("dirb200_join_components_workspace_bytes")(n)), dtype=torch.uint8, device=off.device)
    lib.call("dirb200_join_components", _ptr(off), _ptr(cols), n, cols.shape[0], _ptr(ws), _ptr(labels), _stream())
    return labels


def join_groups(labels):
    """Components of >= 2 rows by ascending label, members ascending -> (group offsets int64 (G+1,), members int64)."""
    _chk(labels, torch.int64, "labels")
    n = labels.shape[0]
    if n < 1:
        return torch.zeros(1, dtype=torch.int64, device=labels.device), labels.new_empty(0)
    off = torch.empty(n // 2 + 1, dtype=torch.int64, device=labels.device)
    members = torch.empty(n, dtype=torch.int64, device=labels.device)
    ws = torch.empty(int(lib.raw("dirb200_join_groups_workspace_bytes")(n)), dtype=torch.uint8, device=labels.device)
    counts = (C.c_int64 * 2)()
    lib.call("dirb200_join_groups", _ptr(labels), n, _ptr(ws), _ptr(off), _ptr(members), counts, _stream())
    return off[:counts[0] + 1].clone(), members[:counts[1]].clone()
