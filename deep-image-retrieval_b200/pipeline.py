"""The extraction / evaluation drivers of the reference, on the CUDA path.

Function names, keyword arguments and console output follow ``dirtorch/test_dir.py`` (``expand_descriptors`` :24-44,
``extract_image_features`` :47-94, ``eval_model`` :97-180, ``load_model`` :183-191, CLI :194-259) and
``dirtorch/extract_features.py`` (``extract_features`` :26-68, CLI :82-124).  What runs underneath:
``net(imgs)`` is the libdirb200 network, multi-scale pooling / whitening / similarity / alpha-QE are libdirb200
kernels; only AP bookkeeping (datasets.py) stays on the host, as in the reference.
"""
from __future__ import annotations

import json
import os
import os.path as osp

import numpy as np
import torch
import tqdm

from . import common, datasets, inputs, nets, ops
from .common import matmul, pool, tonumpy
from .inputs import rows64
from .loader import get_loader
from .store import DescriptorStore


def mkdir(fname, isfile="auto"):
    if isfile == "auto":
        isfile = bool(os.path.splitext(fname)[1])
    directory = os.path.split(fname)[0] if isfile else fname
    if directory and not os.path.isdir(directory):
        os.makedirs(directory)


def _drop_self(scores, idx, own_rows, k):
    """Neighbour lists (best first, one more entry than needed) of database rows queried against their own
    database -> the first k entries that are not the row itself, order preserved.  A row need not be in its own
    list (exact duplicates with a lower index rank before it); then the list is just cut to k."""
    own = np.asarray(own_rows)[:, None]
    keep = np.argsort(idx == own, axis=1, kind="stable")[:, :k]                              # non-self entries first
    s, i = np.take_along_axis(scores, keep, 1).copy(), np.take_along_axis(idx, keep, 1).copy()
    left = i == own                                   # only when the database has no more than k rows: no neighbour
    i[left], s[left] = -1, 0.0                        # (index -1 = skipped by dirb200_aqe_expand)
    return s, i


def expand_descriptors(descs, db=None, alpha=0, k=0, q_block=4096, to_numpy=True):
    """alpha query expansion (db given) / database augmentation (db=None): test_dir.py:24-44.
    q' = normalize(mean([q] + [db_j * sim_ij^alpha for the k nearest j])).  Returns a host ndarray like the
    reference (to_numpy=False, extension: the device tensor).  q_block (extension): queries searched per pass."""
    assert k >= 0 and alpha >= 0, "k and alpha must be non-negative"
    if k == 0:
        return descs
    dim = np.shape(descs)[1]
    q = rows64(descs)
    d = rows64(db) if db is not None else q
    index = ops.Index(d)
    out = torch.empty_like(q)
    # Queries go through in blocks so that database augmentation (an N x N self-search) needs O(block) scratch.
    for c0 in range(0, q.shape[0], q_block):
        qc = q[c0:c0 + q_block].contiguous()
        if db is not None:
            s, i = index.search(qc, min(k, d.shape[0]))
        else:
            # the reference zeroes the diagonal of the self-similarity (test_dir.py:33-34): drop each row from its
            # own neighbour list
            s1, i1 = index.search(qc, min(k + 1, d.shape[0]))
            s1, i1 = _drop_self(s1.cpu().numpy(), i1.cpu().numpy(), np.arange(c0, c0 + qc.shape[0]), k)
            s, i = torch.from_numpy(s1).cuda(), torch.from_numpy(i1).cuda()
        out[c0:c0 + qc.shape[0]] = ops.aqe_expand(qc, d, i.contiguous(), s.contiguous(), float(alpha))
    out = out[:, :dim].contiguous()
    return out.cpu().numpy() if to_numpy else out


_GPU_CHAIN = None


def _gpu_chain_scale(transforms):
    """Transform chains the GPU preprocessing path reproduces bit for bit: '' (ToTensor + Normalize only) and
    'Scale(<float>)' (transforms.py:133-185 with PIL bilinear) -> the scale factor (1.0 for ''), else None."""
    import re
    global _GPU_CHAIN
    if _GPU_CHAIN is None:
        _GPU_CHAIN = re.compile(r"^\s*(?:Scale\(\s*([0-9]*\.[0-9]+|[0-9]+\.[0-9]*)\s*\))?\s*$")
    m = _GPU_CHAIN.match(transforms or "")
    if not m:
        return None
    s = float(m.group(1)) if m.group(1) else 1.0
    return s if 0 < s <= 4 else None


# Mixed-size extraction in batches: decoded images are collected in windows of RAGGED_WINDOW x batch_size, and each
# window is cut into network passes (ragged_groups) run by the ragged forward, which pads every image of a pass to
# the pass's largest height and width and masks the padding out.  A pass's padded area B * H * W stays within
# RAGGED_AREA_BOUND x the sum of its images' true areas.
RAGGED_WINDOW = 4
RAGGED_AREA_BOUND = (5, 4)          # 1.25 as an exact ratio: 4 * B * H * W <= 5 * sum(h * w)


def ragged_groups(sizes, batch_size):
    """Cut images of sizes [(h, w), ...] into network passes: sorted by shape, then greedily grouped into runs of at
    most batch_size images whose padded area (len * max h * max w) is at most 1.25 x the sum of their areas.
    -> list of lists of indices into `sizes`; every index appears exactly once."""
    num, den = RAGGED_AREA_BOUND
    order = sorted(range(len(sizes)), key=lambda i: (int(sizes[i][0]), int(sizes[i][1]), i))
    groups, cur, hmax, wmax, area = [], [], 0, 0, 0
    for i in order:
        h, w = int(sizes[i][0]), int(sizes[i][1])
        nh, nw, na = max(hmax, h), max(wmax, w), area + h * w
        if cur and (len(cur) >= batch_size or den * (len(cur) + 1) * nh * nw > num * na):
            groups.append(cur)
            cur, nh, nw, na = [], h, w, h * w
        cur.append(i)
        hmax, wmax, area = nh, nw, na
    if cur:
        groups.append(cur)
    return groups


def _ragged_window(net, imgs, batch_size):
    """Descriptors (len(imgs), D), in order, of one window of preprocessed images on the GPU: uint8 HWC (h,w,3) or
    normalised fp32 CHW (3,h,w), through ragged_groups passes of the ragged forward."""
    u8 = imgs[0].dtype == torch.uint8
    sizes = [(int(x.shape[0]), int(x.shape[1])) if u8 else (int(x.shape[1]), int(x.shape[2])) for x in imgs]
    out = [None] * len(imgs)
    for g in ragged_groups(sizes, batch_size):
        hh, ww = max(sizes[i][0] for i in g), max(sizes[i][1] for i in g)
        # slot content outside an image is ignored by the forward: no need to clear it
        slots = imgs[g[0]].new_empty((len(g), hh, ww, 3) if u8 else (len(g), 3, hh, ww))
        for k, i in enumerate(g):
            h, w = sizes[i]
            if u8:
                slots[k, :h, :w] = imgs[i]
            else:
                slots[k, :, :h, :w] = imgs[i]
        d = net.forward_ragged_slots(slots, [sizes[i] for i in g])
        for k, i in enumerate(g):
            out[i] = d[k:k + 1]
    return torch.cat(out, dim=0)


# Baseline JPEGs are decoded on the GPU (ops.JpegDecoder, byte-identical to PIL) in calls of one window of images:
# the ragged window, or JPEG_WINDOW images when images go through the network one at a time.  False: PIL decodes
# every file on the loader workers.
GPU_JPEG = True
JPEG_WINDOW = 16


def _image_source(dataset):
    """dataset.get_image_source where get_image is exactly the decode (+ ROI crop) that it describes, else None (a
    dataset that overrides get_image keeps its own decode)."""
    if isinstance(dataset, _RowRange):
        return dataset.get_image_source if _image_source(dataset.dataset) else None
    if type(dataset).get_image in (datasets.Dataset.get_image, datasets.ImageListROIs.get_image):
        return dataset.get_image_source
    return None


def crop_u8(x, box):
    """Image.crop(box) of a uint8 HWC tensor: PIL rounds the box with round() (half to even) and fills 0 outside."""
    x0, y0, x1, y1 = (int(round(v)) for v in box)
    h, w = int(x.shape[0]), int(x.shape[1])
    if (x0, y0, x1, y1) == (0, 0, w, h):
        return x
    out = x.new_zeros((max(y1 - y0, 0), max(x1 - x0, 0), 3))
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, h), max(x0, 0), min(x1, w)
    if sy1 > sy0 and sx1 > sx0:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = x[sy0:sy1, sx0:sx1]
    return out


class _RawImages(torch.utils.data.Dataset):
    """Images for the GPU preprocessing path, as (data, is_jpeg, crop box).  With a source (_image_source), a file the
    GPU decoder takes comes back as its bytes (uint8 tensor) and its crop box; anything else is decoded here with
    PIL, as uint8 HWC pixels (crop applied)."""

    def __init__(self, dataset, source=None):
        self.dataset, self.source = dataset, source

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, i):
        if self.source is not None:
            fname, box = self.source(i)
            with open(fname, "rb") as f:
                data = f.read()
            if ops.jpeg_probe(data)[0] == 0:
                return torch.frombuffer(bytearray(data), dtype=torch.uint8), True, box
        return torch.from_numpy(np.array(self.dataset.get_image(i).convert("RGB"), dtype=np.uint8)), False, None


def _decode_window(items, first, dataset, decoder):
    """Loader items of images first, first + 1, ... -> their uint8 HWC pixels on the GPU.  The JPEGs go through one
    decoder call; a file whose data does not decode cleanly there is decoded again with PIL."""
    imgs = [None] * len(items)
    jpeg = [k for k, it in enumerate(items) if it[1]]
    if jpeg:
        dec, ok = decoder.decode([items[k][0] for k in jpeg])
        for k, x, good in zip(jpeg, dec, ok):
            if good:
                imgs[k] = crop_u8(x, items[k][2]) if items[k][2] is not None else x
    for k, it in enumerate(items):
        if imgs[k] is None:
            px = it[0] if not it[1] else torch.from_numpy(np.array(dataset.get_image(first + k).convert("RGB"), np.uint8))
            imgs[k] = px.cuda(non_blocking=True)
    return imgs


def extract_image_features(dataset, transforms, net, ret_imgs=False, same_size=False, flip=None,
                           desc="Extract feats...", iscuda=True, threads=8, batch_size=8, gpu_preprocess=True):
    """Descriptors of every image of `dataset`, (N, D) on the GPU (test_dir.py:47-94).
    gpu_preprocess (extension): when the chain is '' or 'Scale(<float>)' and images go through one by one, resize
    (byte-identical to PIL bilinear), ToTensor and Normalize run on the GPU from the decoded uint8 pixels
    (dirb200_resize_bilinear_u8 + dirb200_net_forward_u8) - bit-identical descriptors, no PIL resize / float
    conversion on the host and 4x fewer bytes over PCIe.
    Images of different sizes (no Pad / Crop in the chain) go through the network batch_size at a time as ragged
    batches (ragged_groups, ResNetRMAC.forward_ragged_slots): the same descriptors, bit for bit, as one image per call,
    which is what batch_size = 1 and FPN networks (whose head depends on each image's size) still do."""
    ragged = (not same_size and not ret_imgs and batch_size > 1 and hasattr(net, "forward_ragged_slots")
              and not getattr(net, "fpn", False))
    group = batch_size if ragged else 1
    window = RAGGED_WINDOW * group
    if not same_size:
        batch_size = 1
    scale = _gpu_chain_scale(transforms) if (gpu_preprocess and not same_size and not ret_imgs and hasattr(net, "forward_u8")) else None
    if hasattr(net, "eval"):
        net.eval()
    if scale is not None:
        source = _image_source(dataset) if GPU_JPEG else None
        decoder = ops.JpegDecoder() if source is not None else None
        loader = torch.utils.data.DataLoader(_RawImages(dataset, source), batch_size=None, shuffle=False,
                                             num_workers=max(0, threads if threads > 1 else 0), pin_memory=True)
        img_feats, items, done = [], [], 0
        step = window if ragged else (JPEG_WINDOW if decoder is not None else 1)

        def run(items, first):
            pending = []
            for x in _decode_window(items, first, dataset, decoder):
                if flip and flip.pop(0):
                    x = x.flip(1)                        # horizontal flip (imgs[i].flip(2) on CHW, test_dir.py:70-72)
                h, w = int(x.shape[0]), int(x.shape[1])
                oh, ow = int(0.5 + scale * h), int(0.5 + scale * w)      # Scale.get_params, transforms.py:168
                x = x.unsqueeze(0).contiguous()
                if (oh, ow) != (h, w) and min(oh, ow) != min(h, w):      # Scale.__call__: can_upscale / can_downscale
                    x = ops.resize_bilinear_u8(x, (oh, ow))
                if ragged:
                    pending.append(x[0])
                    continue
                d = net.forward_u8(x)
                img_feats.append(d.unsqueeze(0) if d.dim() == 1 else d)
            if pending:
                img_feats.append(_ragged_window(net, pending, group))

        for item in tqdm.tqdm(loader, desc, total=len(dataset)):
            items.append(item)
            if len(items) == step:
                run(items, done)
                done += len(items)
                items = []
        if items:
            run(items, done)
        return torch.cat(img_feats, dim=0)
    loader = get_loader(dataset, trf_chain=transforms, preprocess=net.preprocess, iscuda=iscuda, output=["img"],
                        batch_size=batch_size, threads=threads, shuffle=False)
    tocpu = (lambda x: x.cpu()) if ret_imgs == "cpu" else (lambda x: x)
    img_feats, trf_images, pending = [], [], []
    for inputs in tqdm.tqdm(loader, desc, total=1 + (len(dataset) - 1) // batch_size):
        imgs = inputs[0]
        for i in range(len(imgs)):
            if flip and flip.pop(0):
                imgs[i] = imgs[i].flip(2)
        imgs = common.variables(inputs[:1], net.iscuda)[0]
        if ragged:
            pending.extend(imgs[i].float().cuda() for i in range(len(imgs)))
            if len(pending) >= window:
                img_feats.append(_ragged_window(net, pending, group))
                pending = []
            continue
        d = net(imgs)
        if ret_imgs:
            trf_images.append(tocpu(imgs))
        if d.dim() == 1:
            d = d.unsqueeze(0)
        img_feats.append(d)
    if pending:
        img_feats.append(_ragged_window(net, pending, group))
    img_feats = torch.cat(img_feats, dim=0)
    if ret_imgs:
        if same_size:
            trf_images = torch.cat(trf_images, dim=0)
        return trf_images, img_feats
    return img_feats


def _pool_and_normalize(descs, pooling, gemp):
    """pool() over transform chains followed by F.normalize(p=2, dim=1): test_dir.py:121-122."""
    if len(descs) == 1:
        return ops.l2_normalize(inputs.rows(descs[0]))
    if pooling not in ("mean", "gem"):
        raise ValueError("Bad pooling mode: " + str(pooling))
    return ops.pool_scales([inputs.rows(d) for d in descs], pooling, gemp, l2=True)


def _rank_target_csr(db, nq):
    """The targets of the APs of queries 0 .. nq-1 (db.rank_targets) as one host CSR -> (offsets int64 (nq+1,), rows
    int64 (T,), flags uint8 (T,))."""
    offs, rows, flags = [0], [], []
    for q in range(nq):
        r, fl = db.rank_targets(q)
        rows.append(r)
        flags.append(fl)
        offs.append(offs[-1] + len(r))
    rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    flags = np.concatenate(flags) if flags else np.zeros(0, np.uint8)
    return np.array(offs, np.int64), rows, flags


def _grade(grade, offs, rows, *per_target):
    """Per-query APs from per-target results (CUDA tensors over the CSR offs / rows of _rank_target_csr):
    grade(q, the rows of q, *the results at those rows) for every query q."""
    per_target = [t.cpu().numpy() for t in per_target]
    return [grade(q, rows[offs[q]:offs[q + 1]], *(t[offs[q]:offs[q + 1]] for t in per_target))
            for q in range(len(offs) - 1)]


def _aps_from_topk(db, qdescs, bdescs, k):
    """Per-query AP from the exact top-k ranking (dirb200_index_search); dense score row only where needed."""
    qd, bd = rows64(qdescs), rows64(bdescs)
    k = min(k, bd.shape[0])
    _, idx = ops.Index(bd).search(qd, k)
    idx = idx.cpu().numpy()
    aps = []
    for q in range(qd.shape[0]):
        ap = db.eval_query_AP_from_ranking(q, idx[q])
        incomplete = ap is None or (isinstance(ap, dict) and any(v is None for v in ap.values()))
        if incomplete:
            row = ops.scores_exact(qd[q:q + 1].contiguous(), bd).cpu().numpy()[0]
            ap = db.eval_query_AP(q, row)
        aps.append(ap)
    return aps


def _aps_from_counts(db, qdescs, bdescs):
    """Per-query AP without the Q x N score matrix and without any host-side ranking: the GPU returns the exact scores
    of the labelled rows and, for every positive, the number of database rows ranking before it
    (dirb200_index_rank_count); datasets.eval_query_AP_from_counts turns that into the AP of generic.py:196-224."""
    qd, bd = rows64(qdescs), rows64(bdescs)
    offs, rows, flags = _rank_target_csr(db, qd.shape[0])
    sc, above = ops.Index(bd).rank_counts(qd, offs, rows, flags)
    return _grade(db.eval_query_AP_from_counts, offs, rows, sc, above)


def _aps_from_label_counts(db, qdescs, bdescs, max_thresholds=1 << 26, q_block=4096):
    """Per-query label AP and top-k without the Q x N score matrix (label datasets, dataset.py:83-101).  AP: the fp32
    exact scores of each query's positives are the thresholds, dirb200_index_count_ge counts the rows reaching each
    one, datasets.eval_query_AP_from_ge_counts turns that into sklearn's AP.  Top-k: the exact top-100 of
    dirb200_index_search.  Queries go through in blocks of at most ~max_thresholds thresholds (a class of c images
    gives c^2 of them).  -> (aps, tops)."""
    from .dist import ShardedIndex
    qd, bd = rows64(qdescs), rows64(bdescs)
    nq, n, dev = qd.shape[0], bd.shape[0], qd.device
    index = ShardedIndex(bd, 0)
    t_off, t_rows, skip = db.label_targets()
    aps, q0 = [], 0
    while q0 < nq:
        q1 = int(np.searchsorted(t_off, t_off[q0] + max_thresholds, side="right")) - 1
        q1 = min(max(q1, q0 + 1), nq)
        lo, hi = int(t_off[q0]), int(t_off[q1])
        off = t_off[q0:q1 + 1] - lo
        thr, cnt = index.count_ge(qd[q0:q1], torch.from_numpy(off.astype(np.int32)).to(dev),
                                  torch.from_numpy(t_rows[lo:hi]).to(dev), torch.from_numpy(skip[q0:q1]).to(dev))
        thr, cnt = thr.cpu().numpy(), cnt.cpu().numpy()
        aps += [db.eval_query_AP_from_ge_counts(q0 + i, thr[off[i]:off[i + 1]], cnt[off[i]:off[i + 1]]) for i in range(q1 - q0)]
        q0 = q1
    tops, k = [], min(100, n)
    for c0 in range(0, nq, q_block):
        _, idx = index.search(qd[c0:c0 + q_block].contiguous(), k)
        idx = idx.cpu().numpy()
        tops += [db.eval_query_top_from_ranking(c0 + i, idx[i]) for i in range(idx.shape[0])]
    return aps, tops


def _aps_from_diffusion(db, qdescs, bdescs, params):
    """Per-query AP after diffusion re-ranking (extension): the graph of the database rows, the CG solve of every
    query, and for every positive the number of rows ranking before it by f (dirb200_diffusion_rank_count), graded by
    datasets.eval_query_AP_from_counts with f in place of the scores."""
    from .diffusion import Diffusion
    build = {k: params[k] for k in ("k", "gamma") if k in params}
    solve = {k: params[k] for k in ("kq", "alpha", "iters", "tol") if k in params}
    offs, rows, flags = _rank_target_csr(db, qdescs.shape[0])
    if params.get("truncate") is not None:
        # truncated diffusion: a junk row and a positive are ordered by (inside R_q, value, index), rule T6
        d = Diffusion(bdescs, truncation=True, **build)
        inside, sc, above = d.rank_counts_truncated(qdescs, offs, rows, flags, params["truncate"], **solve)
        return _grade(db.eval_query_AP_from_truncated_counts, offs, rows, inside, sc, above)
    sc, above = Diffusion(bdescs, **build).rank_counts(qdescs, offs, rows, flags, **solve)
    return _grade(db.eval_query_AP_from_counts, offs, rows, sc, above)


def _aps_from_ivf(db, qdescs, bdescs, params):
    """Per-query AP with inverted-file ranking (extension; DESIGN.md section 4.10, rule I7): the lists are k-means lists
    of the database rows (IVFIndex.train), each query ranks the union R_q of its nprobe best lists first, in exact
    order, then every other row in exact order; a junk row ranks before a positive by (inside R_q, score, index)."""
    from .ivf import IVFIndex
    qd, bd = rows64(qdescs), rows64(bdescs)
    offs, rows, flags = _rank_target_csr(db, qd.shape[0])
    if params.get("pq"):
        from .ivfpq import IVFPQIndex
        index = IVFPQIndex.train(bd, params["n_lists"], params["pq"], seed=params.get("seed", 0))
        exact = ops.Index(bd)
        try:
            inside, sc, rank = index.rank_counts(qd, offs, rows, flags, params["nprobe"], refine=params.get("refine"),
                                                 exact=exact)
        finally:
            exact.close()
            index.close()
    else:
        index = IVFIndex.train(bd, params["n_lists"], seed=params.get("seed", 0))
        try:
            inside, sc, rank = index.rank_counts(qd, offs, rows, flags, params["nprobe"])
        finally:
            index.close()
    return _grade(db.eval_query_AP_from_truncated_counts, offs, rows, inside, sc, rank)


def _aps_from_graph(db, qdescs, bdescs, params):
    """Per-query AP with graph-search ranking (extension; DESIGN.md section 4.12, rule G8): the pruned kNN graph of the
    database rows (GraphIndex), each query ranks the rows its traversal visited, V_q, first, in exact order, then every
    other row in exact order; a junk row ranks before a positive by (inside V_q, score, index)."""
    from .graph import GraphIndex
    qd, bd = rows64(qdescs), rows64(bdescs)
    offs, rows, flags = _rank_target_csr(db, qd.shape[0])
    build = {k: params[k] for k in ("degree", "build_k", "n_entry", "seed") if k in params}
    walk = {k: params[k] for k in ("itopk", "width", "max_iter", "n_seeds") if k in params}
    index = GraphIndex(bd, **build)
    walk["n_seeds"] = min(walk.get("n_seeds", 16), index.entry_.shape[0])     # see eval_model
    exact = ops.Index(bd)
    try:
        inside, sc, rank = index.rank_counts(qd, offs, rows, flags, exact=exact, **walk)
    finally:
        exact.close()
        index.close()
    return _grade(db.eval_query_AP_from_truncated_counts, offs, rows, inside, sc, rank)


def graph_params(values):
    """--graph DEGREE ITOPK -> the eval_model `graph` dict (integers, 1 <= DEGREE <= 128, ITOPK >= 1)."""
    from .graph import MAX_DEGREE
    if len(values) != 2:
        raise ValueError("--graph takes DEGREE ITOPK (got %d values)" % len(values))
    out = {}
    for key, v in zip(("degree", "itopk"), values):
        if float(v) != int(v) or int(v) < 1:
            raise ValueError("--graph: %s must be an integer >= 1 (got %r)" % (key.upper(), v))
        out[key] = int(v)
    if out["degree"] > MAX_DEGREE:
        raise ValueError("--graph: DEGREE must be at most %d (got %d)" % (MAX_DEGREE, out["degree"]))
    return out


def ivf_params(values):
    """--ivf NLIST NPROBE -> the eval_model `ivf` dict (integers, 1 <= NPROBE <= NLIST; NLIST <= N is checked by the
    k-means fit)."""
    if len(values) != 2:
        raise ValueError("--ivf takes NLIST NPROBE (got %d values)" % len(values))
    out = {}
    for key, v in zip(("n_lists", "nprobe"), values):
        if float(v) != int(v) or int(v) < 1:
            raise ValueError("--ivf: %s must be an integer >= 1 (got %r)" % ("NLIST" if key == "n_lists" else "NPROBE", v))
        out[key] = int(v)
    if out["nprobe"] > out["n_lists"]:
        raise ValueError("--ivf: NPROBE must not exceed NLIST (got %d > %d)" % (out["nprobe"], out["n_lists"]))
    return dict(out, seed=0)


def pq_params(ivf, pq, refine):
    """--pq M [--refine R] on top of --ivf -> the `pq` / `refine` entries of eval_model's `ivf` dict (M one of 8, 16,
    32, 64, 128; R an integer >= 1, default 400)."""
    if pq is None:
        if refine is not None:
            raise ValueError("--refine needs --pq")
        return ivf
    if ivf is None:
        raise ValueError("--pq needs --ivf")
    from .ivfpq import MS, RANK_REFINE
    if pq not in MS:
        raise ValueError("--pq: M must be one of %s (got %r)" % (MS, pq))
    if refine is not None and refine < 1:
        raise ValueError("--refine: R must be an integer >= 1 (got %r)" % (refine,))
    return dict(ivf, pq=pq, refine=RANK_REFINE if refine is None else refine)


def diffusion_params(values):
    """--diffusion K KQ [GAMMA [ALPHA]] -> the eval_model `diffusion` dict (the paper's defaults for what is not given)."""
    from .diffusion import DEFAULTS, check_params
    if not 2 <= len(values) <= 4:
        raise ValueError("--diffusion takes K KQ [GAMMA [ALPHA]] (got %d values)" % len(values))
    out = dict(DEFAULTS)
    for key, v in zip(("k", "kq", "gamma", "alpha"), values):
        if key in ("k", "kq") and float(v) != int(v):
            raise ValueError("--diffusion: %s must be an integer (got %r)" % (key.upper(), v))
        out[key] = int(v) if key in ("k", "kq") else float(v)
    check_params(**out)
    return out


def diffusion_truncate(value):
    """--diffusion-truncate M -> the `truncate` entry of eval_model's `diffusion` dict (an integer >= 1; M >= KQ is
    checked once the number of rows N is known, as min(M, N) >= KQ)."""
    from .diffusion import check_truncate
    try:
        return check_truncate(value)
    except (ValueError, OverflowError):
        raise ValueError("--diffusion-truncate: M must be an integer >= 1 (got %r)" % (value,))


def eval_model(db, net, trfs, pooling="mean", gemp=3, detailed=False, whiten=None, aqe=None, adba=None, threads=8,
               batch_size=16, save_feats=None, load_feats=None, dbg=(), rank_topk=0, dense_scores=False, diffusion=None,
               ivf=None, graph=None):
    """Evaluate a network on a retrieval dataset (test_dir.py:97-180).  aqe / adba: dict(k=..., alpha=...).
    diffusion (extension): dict of dirb200.diffusion parameters (k, kq, gamma, alpha, iters, tol, and optionally
    truncate = m: each query solved on the subgraph of its own m nearest rows); the rows are then
    ranked by diffusion over the database's mutual-kNN graph, after whitening and alpha-DBA / alpha-QE.  Only datasets
    with relevance lists are graded that way (NotImplementedError otherwise).
    ivf (extension): dict(n_lists=..., nprobe=..., seed=0): inverted-file ranking (rule I7): k-means lists of the
    database rows after whitening and alpha-DBA, queries probed after alpha-QE (whose own search stays exact); relevance
    lists only (NotImplementedError otherwise), not together with diffusion (ValueError).  With pq=M (and refine=R,
    default 400) the lists hold product-quantisation codes and the ranking is rule P8's: the best R probed rows by ADC
    score first, in exact order, then every other row.
    graph (extension): dict(degree=..., itopk=..., and optionally build_k, n_entry, seed, width, max_iter, n_seeds):
    graph-search ranking (rule G8): the rows each query's traversal of the database's pruned kNN graph visited first,
    in exact order, then every other row; relevance lists only, not together with ivf or diffusion (ValueError).
    n_seeds (default 16) is lowered to the size of the entry sample, min(N, n_entry), when it exceeds it, so that the
    default grades databases of fewer than 16 rows; GraphIndex.search itself refuses such an n_seeds.
    Ranking: datasets with relevance lists (Oxford/Paris style) are graded from GPU rank counts and label datasets
    from GPU threshold counts + the exact top-100 - no Q x N score matrix, no host argsort; dense_scores=True
    (extension) forces the literal matmul + per-query sort of the reference; rank_topk > 0 (extension) grades
    relevance-list datasets from the exact top-k lists."""
    print("\n>> Evaluation...")
    query_db = db.get_query_db()
    bdescs, qdescs = [], []
    if not load_feats:
        trfs_list = [trfs] if isinstance(trfs, str) else trfs
        for trf in trfs_list:
            kw = dict(iscuda=net.iscuda, threads=threads, batch_size=batch_size, same_size="Pad" in trf or "Crop" in trf)
            bdescs.append(extract_image_features(db, trf, net, desc="DB", **kw))
            qdescs.append(bdescs[-1] if db is query_db else extract_image_features(query_db, trf, net, desc="query", **kw))
        bdescs = _pool_and_normalize(bdescs, pooling, gemp)
        qdescs = _pool_and_normalize(qdescs, pooling, gemp)
    elif DescriptorStore.is_store(os.path.join(load_feats, "bdescs")):
        # extension: row-sharded descriptor store (store.py) instead of one .npy per side
        bdescs = DescriptorStore(os.path.join(load_feats, "bdescs")).read_all().astype(np.float32, copy=False)
        qdescs = (DescriptorStore(os.path.join(load_feats, "qdescs")).read_all().astype(np.float32, copy=False)
                  if query_db is not db else bdescs)
    else:
        bdescs = np.load(os.path.join(load_feats, "feats.bdescs.npy"))
        qdescs = np.load(os.path.join(load_feats, "feats.qdescs.npy")) if query_db is not db else bdescs
    if save_feats:
        mkdir(save_feats, isfile=False)
        np.save(os.path.join(save_feats, "feats.bdescs.npy"), tonumpy(bdescs))
        if query_db is not db:
            np.save(os.path.join(save_feats, "feats.qdescs.npy"), tonumpy(qdescs))
    # From here on the descriptors stay in HBM (the reference hops GPU -> numpy -> GPU -> numpy between the steps,
    # test_dir.py:136-145): whitening, database augmentation, query expansion and the grading all take device tensors.
    same = qdescs is bdescs
    if whiten is not None:
        bdescs = common.whiten_features_gpu(bdescs, net.pca, **whiten)
        qdescs = bdescs if same else common.whiten_features_gpu(qdescs, net.pca, **whiten)
    if adba is not None:
        # (the reference augments the database rows only: queries drawn from the database keep their un-augmented rows)
        bdescs = expand_descriptors(bdescs, to_numpy=False, **adba)
    if aqe is not None:
        qdescs = expand_descriptors(qdescs, db=bdescs, to_numpy=False, **aqe)
    res = {}
    tops = None
    qn, bn = inputs.rows(qdescs), inputs.rows(bdescs)
    unit = bool(float((qn.norm(dim=1) - 1).abs().max()) < 1e-3 and float((bn.norm(dim=1) - 1).abs().max()) < 1e-3)
    if ivf is not None and diffusion is not None:
        raise ValueError("ivf and diffusion are two rankings: choose one")
    if graph is not None and (ivf is not None or diffusion is not None):
        raise ValueError("graph and %s are two rankings: choose one" % ("ivf" if ivf is not None else "diffusion"))
    if graph is not None:
        if not hasattr(db, "eval_query_AP_from_truncated_counts"):
            raise NotImplementedError("graph-search ranking grades datasets with relevance lists (Oxford / Paris "
                                      "style) only; %s has none" % type(db).__name__)
        aps = _aps_from_graph(db, qn, bn, graph)
        scores = None
    elif ivf is not None:
        if not hasattr(db, "eval_query_AP_from_truncated_counts"):
            raise NotImplementedError("inverted-file ranking grades datasets with relevance lists (Oxford / Paris "
                                      "style) only; %s has none" % type(db).__name__)
        aps = _aps_from_ivf(db, qn, bn, ivf)
        scores = None
    elif diffusion is not None:
        if not hasattr(db, "eval_query_AP_from_counts"):
            raise NotImplementedError("diffusion re-ranking grades datasets with relevance lists (Oxford / Paris "
                                      "style) only; %s has none" % type(db).__name__)
        aps = _aps_from_diffusion(db, qn, bn, diffusion)
        scores = None
    elif rank_topk and hasattr(db, "eval_query_AP_from_ranking"):
        # Large databases: rank with the exact top-k engine instead of materialising the Q x N score matrix; a
        # query whose positives are not all inside the top-k falls back to its exact dense score row.
        aps = _aps_from_topk(db, qn, bn, int(rank_topk))
        scores = None
    elif not dense_scores and unit and hasattr(db, "eval_query_AP_from_counts"):
        # default for relevance-list datasets: exact rank counts of the labelled rows from one tensor-core pass
        # (the error bound of the fp16 pass assumes unit-norm rows, which pooling / whitening / QE all produce)
        aps = _aps_from_counts(db, qn, bn)
        scores = None
    elif not dense_scores and unit and hasattr(db, "eval_query_AP_from_ge_counts"):
        # label datasets: threshold counts on fp64 tensor cores (same unit-norm condition: the top-k search needs it)
        aps, tops = _aps_from_label_counts(db, qn, bn)
        scores = None
    else:
        scores = matmul(qn, bn)
        aps = None
    del bdescs, qdescs
    try:
        if aps is None:
            aps = [db.eval_query_AP(q, s) for q, s in enumerate(tqdm.tqdm(scores, desc="AP"))]
        if not isinstance(aps[0], dict):
            aps = [float(e) for e in aps]
            if detailed:
                res["APs"] = aps
            res["mAP"] = float(np.mean([e for e in aps if e >= 0]))      # AP = -1: query without relevants
        else:
            for mode in aps[0].keys():
                apst = [float(e[mode]) for e in aps]
                if detailed:
                    res["APs-" + mode] = apst
                res["mAP-" + mode] = float(np.mean([e for e in apst if e >= 0]))
    except NotImplementedError:
        print(" AP not implemented!")
    try:
        if tops is None:
            if scores is None:
                raise NotImplementedError()
            tops = [db.eval_query_top(q, s) for q, s in enumerate(tqdm.tqdm(scores, desc="top1"))]
        if detailed:
            res["tops"] = tops
        for k in tops[0]:
            res["top%d" % k] = float(np.mean([top[k] for top in tops]))
    except NotImplementedError:
        pass
    return res


def extract_features(db, net, trfs, pooling="mean", gemp=3, detailed=False, whiten=None, threads=8, batch_size=16,
                     output=None, dbg=()):
    """Extract (and optionally whiten) descriptors and save them as .npy (extract_features.py:26-68)."""
    print("\n>> Extracting features...")
    try:
        query_db = db.get_query_db()
    except NotImplementedError:
        query_db = None
    bdescs, qdescs = [], []
    trfs_list = [trfs] if isinstance(trfs, str) else trfs
    for trf in trfs_list:
        kw = dict(iscuda=net.iscuda, threads=threads, batch_size=batch_size, same_size="Pad" in trf or "Crop" in trf)
        bdescs.append(extract_image_features(db, trf, net, desc="DB", **kw))
        if query_db is not None:
            qdescs.append(bdescs[-1] if db is query_db else extract_image_features(query_db, trf, net, desc="query", **kw))
    bdescs = tonumpy(_pool_and_normalize(bdescs, pooling, gemp))
    if query_db is not None:
        qdescs = tonumpy(_pool_and_normalize(qdescs, pooling, gemp))
    if whiten is not None:
        bdescs = common.whiten_features(bdescs, net.pca, **whiten)
        if query_db is not None:
            qdescs = common.whiten_features(qdescs, net.pca, **whiten)
    mkdir(output, isfile=True)
    if query_db is db or query_db is None:
        np.save(output, bdescs)
    else:
        o = osp.splitext(output)
        np.save(o[0] + ".qdescs" + o[1], qdescs)
        np.save(o[0] + ".dbdescs" + o[1], bdescs)
    print("Features extracted.")


class _RowRange:
    """The images [start, end) of a dataset, seen as a dataset (what one rank of a sharded extraction owns)."""

    def __init__(self, dataset, start, end):
        self.dataset, self.start, self.nimg = dataset, int(start), int(end) - int(start)

    def __len__(self):
        return self.nimg

    def get_key(self, i):
        return self.dataset.get_key(self.start + i)

    def get_filename(self, i, root=None):
        return self.dataset.get_filename(self.start + i, root=root)

    def get_image(self, i, resize=None):
        return self.dataset.get_image(self.start + i, resize=resize)

    def get_image_source(self, i):
        return self.dataset.get_image_source(self.start + i)


def extract_to_store(db, net, trfs, store_path, pooling="mean", gemp=3, whiten=None, threads=8, batch_size=16,
                     dtype=np.float32, group=None):
    """Multi-GPU extraction (extension; the reference's analogue is nn.DataParallel, common.py:155).  Run under
    torchrun, one process per GPU: rank r extracts the contiguous image range ``shard_rows(len(db), world, r)`` with
    its own network handle, pools over the transform chains, normalises and optionally whitens exactly as
    ``extract_features`` does, and writes its rows as one shard of a descriptor store (store.py); rank 0 writes the
    manifest.  Images are independent, so there is no data-path collective.  Returns the opened store; each rank can
    then search its rows with ``ShardedIndex.from_store``."""
    import torch.distributed as tdist
    from .dist import shard_rows
    from .store import write_distributed
    on = tdist.is_available() and tdist.is_initialized()
    rank, world = (tdist.get_rank(group), tdist.get_world_size(group)) if on else (0, 1)
    start, end = shard_rows(len(db), world, rank)
    part = _RowRange(db, start, end)
    trfs_list = [trfs] if isinstance(trfs, str) else trfs
    dim = net.descriptor_dim if hasattr(net, "descriptor_dim") else net.feat_dim
    if len(part):
        descs = []
        for trf in trfs_list:
            descs.append(extract_image_features(part, trf, net, desc="DB[%d/%d]" % (rank, world), iscuda=net.iscuda,
                                                threads=threads, batch_size=batch_size,
                                                same_size="Pad" in trf or "Crop" in trf))
        rows = tonumpy(_pool_and_normalize(descs, pooling, gemp))
        if whiten is not None:
            rows = common.whiten_features(rows, net.pca, **whiten)
    else:                                                     # more ranks than images: an empty shard with the
        if whiten is not None:                                # dimension the other ranks' rows have after whitening
            ncomp = np.asarray(net.pca.components_).shape[0]
            dim = min(ncomp, whiten.get("whitenv") or ncomp)
        rows = np.zeros((0, dim), np.float32)
    meta = dict(arch=getattr(net, "arch", ""), trfs=list(trfs_list), pooling=pooling, gemp=gemp, whiten=whiten or {},
                n_images=len(db))
    return write_distributed(store_path, rows, group=group, dtype=dtype, meta=meta)


def load_model(path, iscuda):
    """Build the network from a checkpoint dict (test_dir.py:183-191)."""
    checkpoint = common.load_checkpoint(path, iscuda)
    net = nets.create_model(pretrained="", **checkpoint["model_options"])
    net = common.switch_model_to_cuda(net, iscuda, checkpoint)
    net.load_state_dict(checkpoint["state_dict"])
    net.preprocess = checkpoint.get("preprocess", net.preprocess)
    if "pca" in checkpoint:
        net.pca = checkpoint.get("pca")
    return net


def _common_args(parser, whiten_default, whitenp_default):
    parser.add_argument("--dataset", "-d", type=str, required=True, help="Command to load dataset")
    parser.add_argument("--checkpoint", type=str, required=True, help="path to weights")
    parser.add_argument("--trfs", type=str, required=False, default="", nargs="+", help="test transforms (can be several)")
    parser.add_argument("--pooling", type=str, default="gem", help="pooling scheme if several trf chains")
    parser.add_argument("--gemp", type=int, default=3, help="GeM pooling power")
    parser.add_argument("--out-json", type=str, default="", help="path to output json")
    parser.add_argument("--detailed", action="store_true", help="return detailed evaluation")
    parser.add_argument("--threads", type=int, default=8, help="number of thread workers")
    parser.add_argument("--dbg", default=(), nargs="*", help="debugging options")
    parser.add_argument("--whiten", type=str, default=whiten_default, help="applies whitening")
    parser.add_argument("--whitenp", type=float, default=whitenp_default, help="whitening power")
    parser.add_argument("--whitenv", type=int, default=None, help="number of components, default is None (all)")
    parser.add_argument("--whitenm", type=float, default=1.0, help="whitening multiplier")


def _select_pca(net, args):
    if args.whiten:
        net.pca = net.pca[args.whiten]
        return {"whitenp": args.whitenp, "whitenv": args.whitenv, "whitenm": args.whitenm}
    net.pca = None
    return None


def test_dir_main(argv=None):
    """python -m dirtorch.test_dir (test_dir.py:194-259).  --aqe / --adba also accept a float alpha."""
    import argparse
    parser = argparse.ArgumentParser(description="Evaluate a model")
    _common_args(parser, whiten_default="Landmarks_clean", whitenp_default=0.25)
    parser.add_argument("--save-feats", type=str, default="", help="path to output features")
    parser.add_argument("--load-feats", type=str, default="", help="path to load features from")
    parser.add_argument("--gpu", type=int, default=0, nargs="+", help="GPU ids")
    parser.add_argument("--aqe", type=float, nargs="+",
                        help="alpha-query expansion parameters: k alpha (any k: the k nearest rows come from the exact top-k search)")
    parser.add_argument("--adba", type=float, nargs="+",
                        help="alpha-database augmentation parameters: k alpha (any k; with k >= the number of rows every other row is a neighbour)")
    parser.add_argument("--rank-topk", type=int, default=0,
                        help="(extension) rank with the exact top-k search (any k; queries whose positives lie deeper fall "
                             "back to their dense score row) instead of the dense score matrix")
    parser.add_argument("--dense-scores", action="store_true",
                        help="(extension) force the reference's literal matmul + per-query sort instead of GPU rank counts")
    parser.add_argument("--diffusion", type=float, nargs="+", metavar="K KQ [GAMMA [ALPHA]]",
                        help="(extension) rank by diffusion over the mutual K-NN graph of the database, seeded by each "
                             "query's KQ nearest rows (defaults: gamma 3, alpha 0.99, 20 CG iterations)")
    parser.add_argument("--diffusion-truncate", type=float, default=None, metavar="M",
                        help="(extension, with --diffusion) truncated diffusion: solve each query on the subgraph of "
                             "its own M nearest rows and rank the other rows after them in exact-score order")
    parser.add_argument("--ivf", type=float, nargs="+", metavar="NLIST NPROBE",
                        help="(extension) rank by an inverted file: k-means lists of the database (NLIST centres, "
                             "k-means++ seed 0); each query's NPROBE best lists first, in exact order, then the other rows")
    parser.add_argument("--pq", type=int, default=None, metavar="M",
                        help="(extension, with --ivf) product-quantisation codes of M bytes per row in the lists: each "
                             "query's best R probed rows by ADC score first, in exact order, then the other rows")
    parser.add_argument("--refine", type=int, default=None, metavar="R",
                        help="(extension, with --pq) rows re-ranked exactly per query (default 400)")
    parser.add_argument("--graph", type=float, nargs="+", metavar="DEGREE ITOPK",
                        help="(extension) rank by graph search: a pruned kNN graph of the database with DEGREE edges "
                             "per row; the rows each query's traversal visits (running list of ITOPK) first, in exact "
                             "order, then the other rows")
    args = parser.parse_args(argv)
    try:
        if args.ivf is not None and args.diffusion is not None:
            raise ValueError("--ivf and --diffusion are two rankings: choose one")
        if args.graph is not None and (args.ivf is not None or args.diffusion is not None):
            raise ValueError("--graph and --%s are two rankings: choose one"
                             % ("ivf" if args.ivf is not None else "diffusion"))
        graph = graph_params(args.graph) if args.graph is not None else None
        ivf = pq_params(ivf_params(args.ivf) if args.ivf is not None else None, args.pq, args.refine)
        diffusion = diffusion_params(args.diffusion) if args.diffusion is not None else None
        if args.diffusion_truncate is not None:
            if diffusion is None:
                raise ValueError("--diffusion-truncate needs --diffusion")
            diffusion["truncate"] = diffusion_truncate(args.diffusion_truncate)
    except ValueError as e:
        parser.error(str(e))
    args.iscuda = common.torch_set_gpu(args.gpu)
    aqe = {"k": int(args.aqe[0]), "alpha": args.aqe[1]} if args.aqe is not None else None
    adba = {"k": int(args.adba[0]), "alpha": args.adba[1]} if args.adba is not None else None
    dataset = datasets.create(args.dataset)
    print("Test dataset:", dataset)
    net = load_model(args.checkpoint, args.iscuda)
    whiten = _select_pca(net, args)
    res = eval_model(dataset, net, args.trfs, pooling=args.pooling, gemp=args.gemp, detailed=args.detailed,
                     threads=args.threads, dbg=args.dbg, whiten=whiten, aqe=aqe, adba=adba,
                     save_feats=args.save_feats, load_feats=args.load_feats, rank_topk=args.rank_topk,
                     dense_scores=args.dense_scores, diffusion=diffusion, ivf=ivf, graph=graph)
    # (the reference's '%s = %g' line raises on the list-valued entries that --detailed adds; print scalars only)
    print(" * " + "\n * ".join(["%s = %g" % p for p in res.items() if isinstance(p[1], (int, float))]))
    if args.out_json:
        try:
            data = json.load(open(args.out_json))
        except IOError:
            data = {}
        data[args.dataset] = res
        mkdir(args.out_json)
        open(args.out_json, "w").write(json.dumps(data, indent=1))
        print("saved to " + args.out_json)
    return res


def merge_pca(checkpoint, name, pca):
    """A shallow copy of the checkpoint dict whose 'pca' dict (a new one; other entries kept) maps name -> pca.
    -> (new checkpoint, True if an entry of that name was replaced)."""
    pcas = dict(checkpoint.get("pca") or {})
    replaced = name in pcas
    pcas[name] = pca
    out = dict(checkpoint)
    out["pca"] = pcas
    return out, replaced


def learn_whiten_main(argv=None):
    """python -m dirtorch.learn_whiten (extension; the reference has no such command): fit PCA(whiten=True) on the GPU
    (whitening.fit_pca) and write a copy of the checkpoint with pca[--name] set, for test_dir / extract_features
    --whiten NAME.  The descriptors come from exactly one of: --dataset (extracted, pooled and normalised as
    extract_features does, without whitening; database images only), --load-feats (an .npy of such descriptors) or
    --store (a descriptor store of extract_to_store)."""
    import argparse
    from .whitening import fit_pca
    parser = argparse.ArgumentParser(description="Learn a PCA whitening on the GPU and store it in a checkpoint")
    parser.add_argument("--checkpoint", type=str, required=True, help="path to weights")
    parser.add_argument("--name", type=str, required=True, help="name of the whitening in checkpoint['pca']")
    parser.add_argument("--output", type=str, required=True, help="path of the checkpoint to write")
    parser.add_argument("--dataset", "-d", type=str, default="", help="command to load the dataset to fit on")
    parser.add_argument("--load-feats", type=str, default="", help=".npy of descriptors to fit on")
    parser.add_argument("--store", type=str, default="", help="descriptor store to fit on")
    parser.add_argument("--trfs", type=str, required=False, default="", nargs="+", help="test transforms (can be several)")
    parser.add_argument("--pooling", type=str, default="gem", help="pooling scheme if several trf chains")
    parser.add_argument("--gemp", type=int, default=3, help="GeM pooling power")
    parser.add_argument("--threads", type=int, default=8, help="number of thread workers")
    parser.add_argument("--n-components", type=int, default=None, help="number of components kept (default: all)")
    parser.add_argument("--gpu", type=int, default=0, help="GPU id")
    args = parser.parse_args(argv)
    if sum(bool(s) for s in (args.dataset, args.load_feats, args.store)) != 1:
        parser.error("exactly one of --dataset, --load-feats and --store is required")
    if os.path.abspath(args.output) == os.path.abspath(args.checkpoint):
        parser.error("--output must differ from --checkpoint")
    common.torch_set_gpu([args.gpu])
    if args.dataset:
        dataset = datasets.create(args.dataset)
        print("Dataset:", dataset)
        net = load_model(args.checkpoint, True)
        descs = []
        for trf in [args.trfs] if isinstance(args.trfs, str) else args.trfs:
            kw = dict(iscuda=net.iscuda, threads=args.threads, batch_size=16, same_size="Pad" in trf or "Crop" in trf)
            descs.append(extract_image_features(dataset, trf, net, desc="DB", **kw))
        X = _pool_and_normalize(descs, args.pooling, args.gemp)
        del net
    elif args.load_feats:
        X = np.load(args.load_feats, mmap_mode="r")
    else:
        X = DescriptorStore(args.store)
    pca = fit_pca(X, n_components=args.n_components)
    print(">> PCA fit on %d x %d descriptors: %d components, %.4g of the variance kept" % (
        pca.n_samples_, pca.n_features_in_, pca.n_components_, float(np.sum(pca.explained_variance_ratio_))))
    checkpoint = torch.load(args.checkpoint, map_location="cpu", weights_only=False)
    checkpoint, replaced = merge_pca(checkpoint, args.name, pca)
    if replaced:
        print("replacing the existing whitening '%s'" % args.name)
    common.save_checkpoint(checkpoint, False, args.output)
    return pca


def extract_features_main(argv=None):
    """python -m dirtorch.extract_features (extract_features.py:82-124)."""
    import argparse
    parser = argparse.ArgumentParser(description="Extract features")
    _common_args(parser, whiten_default=None, whitenp_default=0.5)
    parser.add_argument("--output", type=str, default="", help="path to output features")
    parser.add_argument("--gpu", type=int, nargs="+", help="GPU ids")
    args = parser.parse_args(argv)
    args.iscuda = common.torch_set_gpu(args.gpu if args.gpu is not None else [0])
    dataset = datasets.create(args.dataset)
    print("Dataset:", dataset)
    net = load_model(args.checkpoint, args.iscuda)
    whiten = _select_pca(net, args)
    extract_features(dataset, net, args.trfs, pooling=args.pooling, gemp=args.gemp, detailed=args.detailed,
                     threads=args.threads, dbg=args.dbg, whiten=whiten, output=args.output)
