"""Numpy restatement of the baseline JPEG decode that csrc/jpeg.cu runs on the GPU: the spec of its kernels.

Decoding follows ITU-T T.81 (sequential Huffman, one interleaved scan) and the arithmetic libjpeg applies when PIL
calls it with its defaults: ISLOW integer IDCT with the wrap-then-clamp range limit, "fancy" triangle upsampling
(plain replication for components no more than two samples wide) and 16-bit fixed-point YCbCr->RGB tables.  The
tests check that it equals np.array(Image.open(f).convert("RGB")) byte for byte.
"""
import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
    21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
    61, 54, 47, 55, 62, 63], np.int64)       # zig-zag index -> natural (row-major) index


class Unsupported(Exception):
    pass


def parse(data):
    """Markers of a baseline JPEG -> dict(h, w, comps=[(id, hs, vs, tq, td, ta)], qt, dc, ac, ri, rgb, scan)."""
    data = bytes(data)
    if data[:2] != b"\xff\xd8":
        raise ValueError("no SOI")
    p, qt, dc, ac, ri = 2, {}, {}, {}, 0
    jfif, adobe, sof = False, None, None
    while True:
        while p < len(data) and data[p] == 0xFF and p + 1 < len(data) and data[p + 1] == 0xFF:
            p += 1
        if p + 4 > len(data) or data[p] != 0xFF:
            raise ValueError("bad marker")
        m = data[p + 1]
        ln = (data[p + 2] << 8) | data[p + 3]
        seg = data[p + 4:p + 2 + ln]
        if ln < 2 or p + 2 + ln > len(data):
            raise ValueError("truncated segment")
        if m == 0xE0 and len(seg) >= 14 and seg[:5] == b"JFIF\0":   # libjpeg: a JFIF APP0 of at least 14 bytes
            jfif = True
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                n = 128 if pq else 64
                v = np.frombuffer(seg[q + 1:q + 1 + n], ">u2" if pq else "u1").astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = v
                qt[tq] = t
                q += 1 + n
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                tc, th = seg[q] >> 4, seg[q] & 15
                counts = list(seg[q + 1:q + 17])
                vals = list(seg[q + 17:q + 17 + sum(counts)])
                (ac if tc else dc)[th] = (counts, vals)
                q += 17 + sum(counts)
        elif m == 0xDD:
            ri = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1):
            prec, h, w, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if prec != 8:
                raise Unsupported("precision")
            sof = (h, w, [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)])
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported("SOF%d" % (m - 0xC0))
        elif m == 0xDA:
            ns = seg[0]
            sel = {seg[1 + 2 * i]: (seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)}
            h, w, cs = sof
            comps = [(cid, hs, vs, tq) + sel[cid] for cid, hs, vs, tq in cs]
            ids = [c[0] for c in cs]
            rgb = len(cs) == 3 and (adobe == 0 if (not jfif and adobe is not None) else
                                    (not jfif and ids == [82, 71, 66]))
            return dict(h=h, w=w, comps=comps, qt=qt, dc=dc, ac=ac, ri=ri, rgb=rgb, scan=data[p + 2 + ln:])
        p += 2 + ln


def unstuff(scan):
    """Entropy-coded data -> list of restart-interval segments as bytes (FF 00 -> FF, split at RSTn)."""
    segs, cur, i = [], bytearray(), 0
    while i < len(scan):
        b = scan[i]
        if b == 0xFF:
            n = scan[i + 1]
            if n == 0x00:
                cur.append(0xFF)
                i += 2
                continue
            if 0xD0 <= n <= 0xD7:
                segs.append(bytes(cur))
                cur = bytearray()
                i += 2
                continue
            if n == 0xFF:
                i += 1
                continue
            break                                      # EOI (or any other marker) ends the scan
        cur.append(b)
        i += 1
    segs.append(bytes(cur))
    return segs


class _Huff:
    def __init__(self, counts, vals):
        self.map, code, k = {}, 0, 0
        for ln in range(1, 17):
            for _ in range(counts[ln - 1]):
                self.map[(ln, code)] = vals[k]
                k += 1
                code += 1
            code <<= 1


class _Bits:
    def __init__(self, seg):
        self.bits = np.unpackbits(np.frombuffer(seg, np.uint8)) if seg else np.zeros(0, np.uint8)
        self.pos = 0

    def get(self, n):
        v = 0
        for _ in range(n):
            if self.pos >= len(self.bits):
                raise ValueError("out of bits")
            v = (v << 1) | int(self.bits[self.pos])
            self.pos += 1
        return v

    def sym(self, h):
        code = 0
        for ln in range(1, 17):
            code = (code << 1) | self.get(1)
            if (ln, code) in h.map:
                return h.map[(ln, code)]
        raise ValueError("bad code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def geometry(hdr):
    """(mcux, mcuy, [(hs, vs) per component], blocks per MCU)."""
    comps = hdr["comps"]
    if len(comps) == 1:
        samp = [(1, 1)]
    else:
        samp = [(c[1], c[2]) for c in comps]
    hmax, vmax = max(s[0] for s in samp), max(s[1] for s in samp)
    mcux = -(-hdr["w"] // (8 * hmax))
    mcuy = -(-hdr["h"] // (8 * vmax))
    return mcux, mcuy, samp, sum(h * v for h, v in samp)


def decode_coefficients(hdr):
    """Sequential Huffman decode -> per component int16 array (by, bx, 64) of dequantisation-ready coefficients in
    natural order (DC prediction applied)."""
    mcux, mcuy, samp, _ = geometry(hdr)
    comps = hdr["comps"]
    out = [np.zeros((mcuy * vs, mcux * hs, 64), np.int64) for hs, vs in samp]
    dcs = [_Huff(*hdr["dc"][c[4]]) for c in comps]
    acs = [_Huff(*hdr["ac"][c[5]]) for c in comps]
    segs = unstuff(hdr["scan"])
    nmcu = mcux * mcuy
    ri = hdr["ri"] or nmcu
    mcu = 0
    for seg in segs:
        if mcu >= nmcu:
            break
        br, pred = _Bits(seg), [0] * len(comps)
        for _ in range(min(ri, nmcu - mcu)):
            my, mx = divmod(mcu, mcux)
            for ci, (hs, vs) in enumerate(samp):
                for by in range(vs):
                    for bx in range(hs):
                        blk = out[ci][my * vs + by, mx * hs + bx]
                        s = br.sym(dcs[ci])
                        pred[ci] += _extend(br.get(s), s)
                        blk[0] = pred[ci]
                        k = 1
                        while k < 64:
                            rs = br.sym(acs[ci])
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                blk[ZIGZAG[min(k, 63)]] = _extend(br.get(s), s)
                                k += 1
                            elif r == 15:
                                k += 16
                            else:
                                break
            mcu += 1
    return [o.astype(np.int16) for o in out]


_F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(x, z, shift):
    """One ISLOW pass over axis 0 of int64 arrays: x[k] are the 8 inputs; returns 8 outputs descaled by `shift`."""
    F = _F
    z2, z3 = x[2], x[6]
    z1 = (z2 + z3) * F["f0541"]
    tmp2 = z1 - z3 * F["f1847"]
    tmp3 = z1 + z2 * F["f0765"]
    tmp0 = (x[0] + x[4]) << 13
    tmp1 = (x[0] - x[4]) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[7], x[5], x[3], x[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["f1175"]
    t0, t1, t2, t3 = t0 * F["f0298"], t1 * F["f2053"], t2 * F["f3072"], t3 * F["f1501"]
    z1, z2 = z1 * -F["f0899"], z2 * -F["f2562"]
    z3, z4 = z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + t3 + r) >> shift, (tmp11 + t2 + r) >> shift, (tmp12 + t1 + r) >> shift,
            (tmp13 + t0 + r) >> shift, (tmp13 - t0 + r) >> shift, (tmp12 - t1 + r) >> shift,
            (tmp11 - t2 + r) >> shift, (tmp10 - t3 + r) >> shift]


def idct_islow(coef, q):
    """coef (..., 64) natural order, q (64,) -> (..., 8, 8) uint8 samples (libjpeg jpeg_idct_islow)."""
    d = coef.astype(np.int64) * q.astype(np.int64)
    d = d.reshape(d.shape[:-1] + (8, 8))
    cols = [d[..., k, :] for k in range(8)]                        # pass 1: columns (inputs = rows k of each col)
    ws = np.stack(_idct_1d(cols, None, 13 - 2), axis=-2)           # (..., 8 rows, 8 cols)
    rows = [ws[..., :, k] for k in range(8)]                       # pass 2: rows
    out = np.stack(_idct_1d(rows, None, 13 + 2 + 3), axis=-1)
    w = ((out + 512) & 1023) - 512                                 # post-IDCT range limit: wrap to 10 bits,
    return np.clip(w + 128, 0, 255).astype(np.uint8)               # then clamp


def planes(hdr, coefs):
    """Component sample planes (full MCU rows/columns), uint8."""
    out = []
    for c, co in zip(hdr["comps"], coefs):
        blocks = idct_islow(co, hdr["qt"][c[3]])                   # (by, bx, 8, 8)
        by, bx = blocks.shape[:2]
        out.append(blocks.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8))
    return out


def upsample(plane, ch, cw, fh, fw, oh, ow):
    """Component plane of ch x cw real samples (padding beyond) upsampled by (fh, fw) in {1,2} x {1,2}, as libjpeg's
    fancy upsampler; the result is cut to (oh, ow)."""
    x = plane[:ch, :cw].astype(np.int64)
    if fh == 1 and fw == 1:
        return x[:oh, :ow].astype(np.uint8)
    if cw <= 2:                                                    # libjpeg: fancy only where wider than 2
        return np.repeat(np.repeat(x, fh, 0), fw, 1)[:oh, :ow].astype(np.uint8)
    if fh == 1:                                                    # h2v1
        left = np.concatenate([x[:, :1], x[:, :-1]], 1)
        right = np.concatenate([x[:, 1:], x[:, -1:]], 1)
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * x + left + 1) >> 2
        out[:, 1::2] = (3 * x + right + 2) >> 2
        return out[:oh, :ow].astype(np.uint8)
    up = np.concatenate([x[:1], x[:-1]], 0)                        # h2v2: vertical 3:1 column sums
    dn = np.concatenate([x[1:], x[-1:]], 0)
    sums = np.empty((2 * ch, cw), np.int64)
    sums[0::2] = 3 * x + up
    sums[1::2] = 3 * x + dn
    left = np.concatenate([sums[:, :1], sums[:, :-1]], 1)
    right = np.concatenate([sums[:, 1:], sums[:, -1:]], 1)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * sums + left + 8) >> 4
    out[:, 1::2] = (3 * sums + right + 7) >> 4
    return out[:oh, :ow].astype(np.uint8)


def ycc_to_rgb(y, cb, cr):
    one_half, fix = 1 << 15, lambda v: int(v * 65536 + 0.5)
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (fix(1.40200) * x + one_half) >> 16
    cb_b = (fix(1.77200) * x + one_half) >> 16
    cr_g = -fix(0.71414) * x
    cb_g = -fix(0.34414) * x + one_half
    y = y.astype(np.int64)
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """Baseline JPEG bytes -> (h, w, 3) uint8 RGB, as np.array(Image.open(f).convert("RGB"))."""
    hdr = parse(data)
    h, w = hdr["h"], hdr["w"]
    pl = planes(hdr, decode_coefficients(hdr))
    if len(pl) == 1:
        g = pl[0][:h, :w]
        return np.repeat(g[:, :, None], 3, 2)
    _, _, samp, _ = geometry(hdr)
    hmax, vmax = max(s[0] for s in samp), max(s[1] for s in samp)
    full = []
    for p, (hs, vs) in zip(pl, samp):
        ch, cw = -(-h * vs // vmax), -(-w * hs // hmax)
        full.append(upsample(p, ch, cw, vmax // vs, hmax // hs, h, w))
    if hdr["rgb"]:
        return np.stack(full, -1)
    return ycc_to_rgb(*full)
