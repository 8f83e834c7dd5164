"""CPU checks of the JPEG decoder's spec and host side: the numpy model (tests/jpeg_model.py) equals PIL byte for
byte, dirb200_jpeg_probe reads headers and refuses what the GPU decoder does not take, and crop_u8 is Image.crop."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_model as M


def make_image(h, w, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "smooth":
        y, x = np.mgrid[:h, :w]
        a = np.stack([128 + 100 * np.sin(x / 5.0 + c) * np.cos(y / 7.0 - c) for c in range(3)], -1)
        return np.clip(a + rng.normal(0, 20, a.shape), 0, 255).astype(np.uint8)
    if kind == "sat":
        return (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def encode(a, gray=False, **kw):
    im = Image.fromarray(a)
    if gray:
        im = im.convert("L")
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def pil_rgb(data):
    return np.array(Image.open(io.BytesIO(data)).convert("RGB"))


SIZES = [(1, 1), (1, 2), (2, 1), (2, 3), (7, 9), (8, 8), (9, 17), (16, 16), (17, 33), (37, 53)]
VARIANTS = [dict(subsampling=0), dict(subsampling=1), dict(subsampling=2), dict(subsampling=2, optimize=True),
            dict(subsampling=2, restart_marker_blocks=1), dict(subsampling=1, restart_marker_rows=1),
            dict(subsampling=0, keep_rgb=True), dict(gray=True)]


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_model_equals_pil(variant):
    kw = VARIANTS[variant]
    n = 0
    for i, (h, w) in enumerate(SIZES):
        for q in (1, 50, 90, 100):
            for kind in ("smooth", "sat", "noise"):
                data = encode(make_image(h, w, kind, seed=i), quality=q, **kw)
                assert np.array_equal(M.decode(data), pil_rgb(data)), (h, w, q, kind, kw)
                n += 1
    assert n == len(SIZES) * 12


def test_probe_reports_header():
    from dirb200 import ops
    a = make_image(37, 53, "smooth")
    for kw, samp in ((dict(subsampling=0), (1, 1)), (dict(subsampling=1), (2, 1)), (dict(subsampling=2), (2, 2))):
        st, info = ops.jpeg_probe(encode(a, quality=90, **kw))
        assert st == 0
        assert (info["height"], info["width"], info["components"]) == (37, 53, 3)
        assert (info["h_samp"], info["v_samp"]) == samp and info["color"] == 0
    st, info = ops.jpeg_probe(encode(a, quality=90, subsampling=2, restart_marker_blocks=3))
    assert st == 0 and info["restart_interval"] > 0
    assert M.parse(encode(a, quality=90, subsampling=2, restart_marker_blocks=3))["ri"] == info["restart_interval"]
    st, info = ops.jpeg_probe(encode(a, gray=True, quality=90))
    assert st == 0 and info["components"] == 1 and info["color"] == 2
    st, info = ops.jpeg_probe(encode(a, quality=90, keep_rgb=True, subsampling=0))
    assert st == 0 and info["color"] == 1
    assert ops.jpeg_probe(np.frombuffer(encode(a), np.uint8))[0] == 0       # numpy input
    assert ops.jpeg_probe(torch.frombuffer(bytearray(encode(a)), dtype=torch.uint8))[0] == 0


def test_probe_refuses_unsupported_and_malformed():
    from dirb200 import lib, ops
    a = make_image(40, 56, "smooth")
    assert ops.jpeg_probe(encode(a, quality=90, progressive=True))[0] == lib_code("ENOTSUP")
    cmyk = io.BytesIO()
    Image.fromarray(a).convert("CMYK").save(cmyk, "JPEG")
    assert ops.jpeg_probe(cmyk.getvalue())[0] == lib_code("ENOTSUP")
    png = io.BytesIO()
    Image.fromarray(a).save(png, "PNG")
    assert ops.jpeg_probe(png.getvalue())[0] == lib_code("EINVAL")
    assert "no SOI" in lib.last_error()
    good = encode(a, quality=90)
    for cut in (3, 20, len(good) // 2, len(good) - 1):
        assert ops.jpeg_probe(good[:cut])[0] == lib_code("EINVAL"), cut
    assert ops.jpeg_probe(b"\xff\xd8" + bytes(range(256)) * 4)[0] == lib_code("EINVAL")
    assert ops.jpeg_probe(b"")[0] == lib_code("EINVAL")


def with_short_jfif(data, payload):
    """`data` with an APP0 'JFIF\\0' segment of `payload` bytes (< 14: libjpeg does not count it as JFIF) after SOI."""
    body = (b"JFIF\0" + bytes(range(1, 10)))[:payload]
    return data[:2] + b"\xff\xe0" + (payload + 2).to_bytes(2, "big") + body + data[2:]


def with_trailer(data):
    """`data` followed by bytes after its EOI, as MPF (second image) or vendor trailers put there."""
    return data + b"\xff\xd8\xff\xe1\x00\x04MP" + bytes(range(256)) + b"\xff\xd9trailer"


def test_short_jfif_app0_and_data_after_eoi():
    from dirb200 import ops
    rgb = encode(make_image(24, 40, "smooth", seed=2), quality=90, keep_rgb=True, subsampling=0)
    for payload in (10, 12):
        f = with_short_jfif(rgb, payload)
        st, info = ops.jpeg_probe(f)
        assert st == 0 and info["color"] == 1                # Adobe transform 0 rules: RGB
        assert np.array_equal(M.decode(f), pil_rgb(f))
    ycc = encode(make_image(24, 40, "smooth", seed=2), quality=90)
    for base in (ycc, encode(make_image(33, 47, "noise", seed=5), quality=80, subsampling=2, restart_marker_blocks=2)):
        f = with_trailer(base)
        st, info = ops.jpeg_probe(f)
        assert st == 0 and info["scan_bytes"] == ops.jpeg_probe(base)[1]["scan_bytes"]
        assert np.array_equal(M.decode(f), pil_rgb(f))


def lib_code(name):
    return {"EINVAL": -1, "ENOTSUP": -2}[name]


def test_crop_matches_pil():
    from dirb200.pipeline import crop_u8
    a = make_image(23, 31, "noise")
    im = Image.fromarray(a)
    boxes = [(0, 0, 31, 23), (2.5, 3.5, 20.5, 17.5), (1.5, 0.49, 12.51, 9.5), (-3.2, -1.7, 10.4, 8.6),
             (20.6, 15.5, 40.2, 30.5), (5, 5, 6, 6), (0.5, 1.5, 30.5, 22.5)]
    for box in boxes:
        ref = np.array(im.crop(box))
        got = crop_u8(torch.from_numpy(a), box).numpy()
        assert got.shape == ref.shape and np.array_equal(got, ref), box
