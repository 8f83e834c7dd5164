"""GPU JPEG decoding: byte-identical to np.array(Image.open(f).convert("RGB")), coefficients equal to the sequential
decode of tests/jpeg_model.py, corrupt data flagged, and extraction from JPEG files bit-identical to PIL decoding."""
import io
import os
import pickle

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_model as M
import synthdata as synth
from test_jpeg_host import SIZES, VARIANTS, encode, make_image, pil_rgb

pytestmark = pytest.mark.gpu

LARGE = [(768, 1024), (1023, 769), (2048, 1536)]


def _decoder(**kw):
    from dirb200 import ops
    ops.require_gpu(0)
    return ops.JpegDecoder(0, **kw)


def _matrix():
    files = []
    for v, kw in enumerate(VARIANTS):
        for i, (h, w) in enumerate(SIZES):
            for q, kind in ((1, "sat"), (50, "noise"), (90, "smooth"), (100, "noise")):
                files.append(encode(make_image(h, w, kind, seed=i + 31 * v), quality=q, **kw))
    for i, (h, w) in enumerate(LARGE):
        a = make_image(h, w, "smooth", seed=100 + i)
        files.append(encode(a, quality=90, subsampling=2))
        files.append(encode(a, quality=75, subsampling=1, restart_marker_rows=2))
    return files


def _check(dec, files):
    out, ok = dec.decode(files)
    assert all(ok)
    for k, (data, x) in enumerate(zip(files, out)):
        assert np.array_equal(x.cpu().numpy(), pil_rgb(data)), k


@pytest.mark.parametrize("subseq_bits", [None, 64])
def test_decode_equals_pil(subseq_bits):
    """Every variant one file per call, then mixed batches of up to 64 files; subseq_bits=64 makes every subsequence
    boundary need a synchronisation chain."""
    dec = _decoder(subseq_bits=subseq_bits)
    files = _matrix()
    for f in files[::7]:
        _check(dec, [f])
    rng = np.random.default_rng(0)
    order = rng.permutation(len(files))
    for s in range(0, len(files), 64):
        _check(dec, [files[i] for i in order[s:s + 64]])
    if subseq_bits == 64:
        assert dec.last_rounds >= 1


def test_coefficients_equal_model():
    dec = _decoder(subseq_bits=96)
    files = [encode(make_image(37, 53, "smooth", seed=3), quality=90, subsampling=2, restart_marker_blocks=2),
             encode(make_image(33, 17, "noise", seed=4), quality=100, subsampling=1),
             encode(make_image(40, 24, "smooth", seed=5), gray=True, quality=50),
             encode(make_image(300, 400, "smooth", seed=6), quality=95, subsampling=0, optimize=True)]
    _, ok = dec.decode(files)
    assert all(ok)
    for k, data in enumerate(files):
        hdr = M.parse(data)
        per_comp = M.decode_coefficients(hdr)
        mcux, mcuy, samp, bpm = M.geometry(hdr)
        ref = np.zeros((mcux * mcuy * bpm, 64), np.int16)
        b = 0
        for my in range(mcuy):
            for mx in range(mcux):
                for ci, (hs, vs) in enumerate(samp):
                    for by in range(vs):
                        for bx in range(hs):
                            ref[b] = per_comp[ci][my * vs + by, mx * hs + bx]
                            b += 1
        got = dec.debug_coefficients(k).cpu().numpy()
        assert np.array_equal(got, ref), k


def test_corrupt_code_is_flagged_and_truncation_refused():
    from dirb200 import ops
    dec = _decoder()
    good = encode(make_image(64, 96, "noise", seed=9), quality=95, subsampling=2)
    hdr = M.parse(good)
    start = len(good) - len(hdr["scan"])
    bad = bytearray(good)
    # 48 one-bits (stuffed as FF 00) in the middle of the entropy-coded data: no Huffman code fits there
    mid = start + (len(good) - start) // 2
    if bad[mid - 1] == 0xFF:
        mid += 1
    bad[mid:mid + 2] = b"\xff\x00" * 6
    out, ok = dec.decode([good, bytes(bad), good[:len(good) // 2]])
    assert ok == [True, False, False]
    assert np.array_equal(out[0].cpu().numpy(), pil_rgb(good))
    assert ops.jpeg_probe(good[:len(good) // 2])[0] == -1


def test_refused_files_anywhere_in_a_batch():
    """Files the header parser refuses, first, in the middle and last, leave the others decoded; a short JFIF APP0 and
    data after the EOI decode as PIL decodes them."""
    from test_jpeg_host import with_short_jfif, with_trailer
    dec = _decoder()
    a = encode(make_image(37, 53, "smooth", seed=11), quality=90, subsampling=2)
    b = encode(make_image(64, 80, "noise", seed=12), quality=75, subsampling=1, restart_marker_blocks=3)
    c = with_trailer(encode(make_image(48, 30, "smooth", seed=13), quality=95, gray=True))
    d = with_short_jfif(encode(make_image(20, 28, "smooth", seed=14), quality=90, keep_rgb=True, subsampling=0), 10)
    prog = encode(make_image(40, 40, "smooth", seed=15), quality=90, progressive=True)
    trunc = a[:len(a) // 2]
    for batch, want in (([prog, a, trunc, b, c, prog, d, trunc], [0, 1, 0, 1, 1, 0, 1, 0]),
                        ([a, trunc, b], [1, 0, 1]), ([a, b, prog], [1, 1, 0]), ([trunc, d], [0, 1])):
        out, ok = dec.decode(batch)
        assert ok == [bool(w) for w in want]
        for x, f, good in zip(out, batch, ok):
            if good:
                assert np.array_equal(x.cpu().numpy(), pil_rgb(f))


def _count_gpu_decodes(monkeypatch):
    """Wraps JpegDecoder.decode: the returned list collects, per call, how many files the GPU decoded."""
    from dirb200 import ops
    counts, decode = [], ops.JpegDecoder.decode

    def counting(self, bufs):
        imgs, ok = decode(self, bufs)
        counts.append(sum(ok))
        return imgs, ok
    monkeypatch.setattr(ops.JpegDecoder, "decode", counting)
    return counts


def _write_dataset(root, n=40, seed=7):
    """Mixed files: baseline JPEGs of every supported kind, progressive JPEGs and PNGs, Oxford-like odd sizes."""
    os.makedirs(os.path.join(root, "jpg"), exist_ok=True)
    rs = np.random.RandomState(seed)
    names = []
    for i in range(n):
        h, w = int(rs.randint(96, 260)), int(rs.randint(96, 260))
        a = synth.make_images_u8(1, h, w, seed=seed + i)[0]
        kind = i % 6
        name = "im%03d.%s" % (i, "png" if kind == 5 else "jpg")
        path = os.path.join(root, "jpg", name)
        kw = [dict(quality=90, subsampling=2), dict(quality=85, subsampling=1, restart_marker_blocks=5),
              dict(quality=80, subsampling=0, optimize=True), dict(quality=80, gray=True),
              dict(quality=90, progressive=True)]
        if kind == 5:
            Image.fromarray(a).save(path)
        else:
            with open(path, "wb") as f:
                f.write(encode(a, **kw[kind]))
        names.append(name)
    return names


def _net():
    from dirb200 import nets
    net = nets.create_model("resnet50_rmac")
    net.load_state_dict(synth.make_state_dict("resnet50_rmac", seed=1))
    return net.eval()


def test_extraction_with_gpu_decode_equals_pil(tmp_path, monkeypatch):
    from dirb200 import datasets, pipeline
    _decoder()
    root = str(tmp_path)
    names = _write_dataset(root)
    ds = datasets.ImageList(imgs=names, root=os.path.join(root, "jpg"))
    assert pipeline._image_source(ds) is not None
    net = _net()
    counts = _count_gpu_decodes(monkeypatch)
    baseline = [i % 6 < 4 for i in range(len(names))]      # _write_dataset: kinds 0-3 are baseline JPEGs
    flips = [bool(v) for v in np.random.RandomState(1).randint(0, 2, len(names))]
    for chain in ("", "Scale(0.7)", "Scale(1.4)"):
        ref = pipeline.extract_image_features(ds, chain, net, threads=2, batch_size=1, gpu_preprocess=False,
                                              flip=list(flips))
        assert not counts
        for bs in (1, 16):
            got = pipeline.extract_image_features(ds, chain, net, threads=2, batch_size=bs, flip=list(flips))
            assert torch.equal(got, ref), (chain, bs)
            assert sum(counts) == sum(baseline), (chain, bs)        # every baseline JPEG was decoded on the GPU
            counts.clear()
    # queries of an Oxford-format dataset: crops to fractional bounding boxes, some reaching outside the image
    rs = np.random.RandomState(2)
    gnd, qnames = [], names[:12]
    for n in qnames:
        w, h = Image.open(os.path.join(root, "jpg", n)).size
        x0, y0 = rs.uniform(-3, 20), rs.uniform(-3, 20)
        gnd.append({"bbx": (x0, y0, x0 + rs.uniform(60, w), y0 + rs.uniform(60, h)) if rs.rand() < 0.7 else
                    (round(x0) + 0.5, round(y0) + 0.5, w - 10.5, h - 9.5), "ok": [0], "junk": []})
    with open(os.path.join(root, "gnd.pkl"), "wb") as f:
        pickle.dump({"imlist": names, "qimlist": qnames, "gnd": gnd}, f)
    q = datasets.ImageListRelevants(os.path.join(root, "gnd.pkl"), root=root, img_dir="jpg").get_query_db()
    for chain in ("", "Scale(0.7)"):
        ref = pipeline.extract_image_features(q, chain, net, threads=2, batch_size=1, gpu_preprocess=False)
        for bs in (1, 16):
            assert torch.equal(pipeline.extract_image_features(q, chain, net, threads=2, batch_size=bs), ref), (chain, bs)
            assert sum(counts) == sum(baseline[:len(qnames)]), (chain, bs)
            counts.clear()
    # a dataset whose get_image is its own keeps PIL
    class Own(datasets.ImageList):
        def get_image(self, i, resize=None):
            return super().get_image(i, resize).transpose(Image.FLIP_TOP_BOTTOM)
    assert pipeline._image_source(Own(imgs=names, root=os.path.join(root, "jpg"))) is None
    ref = pipeline.extract_image_features(ds, "", net, threads=2, batch_size=1, gpu_preprocess=False)
    monkeypatch.setattr(pipeline, "GPU_JPEG", False)
    assert torch.equal(pipeline.extract_image_features(ds, "", net, threads=2, batch_size=16), ref)
    assert not counts


def test_dir_main_on_jpeg_copy_prints_pil_aps(tmp_path, monkeypatch, capsys):
    import e2e_data
    from dirb200 import pipeline
    from dirtorch import test_dir
    _decoder()
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root)
    d = os.path.join(root, "oxford5k", "jpg")
    jnames = []
    for i, n in enumerate(names):
        im = Image.open(os.path.join(d, n))
        jn = n.replace(".png", ".jpg")
        im.save(os.path.join(d, jn), quality=90, subsampling=(2, 1, 0)[i % 3], restart_marker_blocks=i % 2 * 7)
        os.remove(os.path.join(d, n))
        jnames.append(jn)
    with open(os.path.join(root, "oxford5k", "gnd_oxford5k.pkl"), "wb") as f:
        pickle.dump({"imlist": jnames, "qimlist": [jnames[i] for i in qn], "gnd": gnd}, f)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)},
               os.path.join(root, "ckpt.pt"))
    monkeypatch.setenv("DB_ROOT", root)
    args = ["--dataset", "Oxford5K", "--checkpoint", os.path.join(root, "ckpt.pt"), "--whiten", "", "--gpu", "0",
            "--threads", "2", "--detailed", "--trfs", "", "Scale(0.7)"]
    counts = _count_gpu_decodes(monkeypatch)
    res_gpu = test_dir.test_dir_main(args)
    out_gpu = capsys.readouterr().out
    assert sum(counts) == 2 * (len(jnames) + len(qn))             # two chains, database and (cropped) queries
    counts.clear()
    monkeypatch.setattr(pipeline, "GPU_JPEG", False)
    res_pil = test_dir.test_dir_main(args)
    assert not counts
    out_pil = capsys.readouterr().out
    assert res_gpu["APs"] == res_pil["APs"] and res_gpu["mAP"] == res_pil["mAP"]
    line = [l for l in out_pil.splitlines() if l.startswith(" * mAP")]
    assert line and line[0] in out_gpu
