"""CPU oracle for the descriptor-extraction + retrieval hot path.  TEST INFRASTRUCTURE ONLY.

This file restates, function by function, what the reference (naver/deep-image-retrieval,
``dirtorch``) computes on the one hot path this repository accelerates: image ->
ResNet-50/101 trunk -> GeM -> FC -> L2 descriptor -> multi-scale pool -> PCA whitening ->
dot-product scores -> ranking / top-k -> alpha query expansion -> average precision.
Each function cites the reference file:line it follows.  It is plain fp32/fp64 CPU
arithmetic (torch CPU functional ops for conv/BN/pool, numpy for everything else).

Who may import this: ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs - as the checker or the timed CPU baseline,
never from the product package (``deep-image-retrieval_b200/`` and ``dirtorch/`` do not
import it, and fail loudly without the CUDA library).

Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4 / 8c), so this
oracle is pinned against outputs of the *unmodified reference itself*, imported from
``/root/reference`` in the build container by ``tests/golden/make_golden.py`` and committed
as ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks every function here
against those vectors.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

BLOCKS = {"resnet50": [3, 4, 6, 3], "resnet101": [3, 4, 23, 3], "resnet152": [3, 8, 36, 3]}  # rmac_resnet.py:78-88
BASIC_BLOCKS = {"resnet18": [2, 2, 2, 2]}   # rmac_resnet.py:74-76 (BasicBlock, expansion 1) - oracle only so far, see DESIGN.md
BN_EPS = 1e-5  # torch.nn.BatchNorm2d default, used by resnet.py:57,60,63,117,140


# --------------------------------------------------------------------------- trunk
def _bn(x, sd, name):
    """Eval-mode BatchNorm2d (running statistics), resnet.py:57,60,63,117."""
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"],
                        sd[name + ".weight"], sd[name + ".bias"], False, 0.0, BN_EPS)


def stem(x, sd):
    """conv 7x7/s2/p3 -> BN -> ReLU -> maxpool 3x3/s2/p1, resnet.py:115-119,158-161."""
    x = F.conv2d(x, sd["conv1.weight"], None, stride=2, padding=3)
    x = F.relu(_bn(x, sd, "bn1"))
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)


def bottleneck(x, sd, prefix, stride, has_down):
    """1x1 -> BN -> ReLU -> 3x3(stride, pad 1) -> BN -> ReLU -> 1x1 -> BN, + (downsampled) x, ReLU.
    resnet.py:67-87 (stride sits on conv2, resnet.py:58)."""
    out = F.relu(_bn(F.conv2d(x, sd[prefix + "conv1.weight"]), sd, prefix + "bn1"))
    out = F.relu(_bn(F.conv2d(out, sd[prefix + "conv2.weight"], None, stride=stride, padding=1), sd, prefix + "bn2"))
    out = _bn(F.conv2d(out, sd[prefix + "conv3.weight"]), sd, prefix + "bn3")
    if has_down:  # resnet.py:136-141
        x = _bn(F.conv2d(x, sd[prefix + "downsample.0.weight"], None, stride=stride), sd, prefix + "downsample.1")
    return F.relu(out + x)


def basic_block(x, sd, prefix, stride, has_down):
    """3x3(stride, pad 1) -> BN -> ReLU -> 3x3 -> BN, + (downsampled) x, ReLU.  resnet.py:14-43."""
    out = F.relu(_bn(F.conv2d(x, sd[prefix + "conv1.weight"], None, stride=stride, padding=1), sd, prefix + "bn1"))
    out = _bn(F.conv2d(out, sd[prefix + "conv2.weight"], None, padding=1), sd, prefix + "bn2")
    if has_down:
        x = _bn(F.conv2d(x, sd[prefix + "downsample.0.weight"], None, stride=stride), sd, prefix + "downsample.1")
    return F.relu(out + x)


def trunk(x, sd, arch="resnet50", return_stages=False):
    """ResNet.forward without the classifier, resnet.py:157-168; layer strides 1,2,2,2 (resnet.py:120-123).
    A projection shortcut exists where the stride or the width changes (resnet.py:136-141): block 0 of every layer
    for Bottleneck trunks, block 0 of layers 2-4 for BasicBlock trunks."""
    name = arch.split("_")[0]
    basic = name in BASIC_BLOCKS
    blocks = BASIC_BLOCKS[name] if basic else BLOCKS[name]
    stages = {}
    x = stem(x, sd)
    stages["stem"] = x
    for li, nblk in enumerate(blocks, start=1):
        for b in range(nblk):
            stride = 2 if (li > 1 and b == 0) else 1
            if basic:
                x = basic_block(x, sd, "layer%d.%d." % (li, b), stride=stride, has_down=(b == 0 and li > 1))
            else:
                x = bottleneck(x, sd, "layer%d.%d." % (li, b), stride=stride, has_down=(b == 0))
        stages["layer%d" % li] = x
    return (x, stages) if return_stages else x


# --------------------------------------------------------------------------- head
def gem(x, p, eps=1e-6):
    """(mean_hw clamp(x,eps)^p)^(1/p), pooling.py:38-40.  x: (B,C,H,W) -> (B,C)."""
    p = float(p)
    return x.clamp(min=eps).pow(p).mean(dim=(2, 3)).pow(1.0 / p)


def center_bias_map(b, h, w, dtype=torch.float32):
    """1 + bilinear(align_corners=True) resize to (h, w) of the 4x4 map with b on its central 2x2, rmac_resnet.py:52-55."""
    m = torch.zeros(1, 1, 4, 4, dtype=dtype)
    m[0, 0, 1:3, 1:3] = float(b)
    return F.interpolate(1 + m, size=(h, w), mode="bilinear", align_corners=True)


def head(feat, sd, pooling="gem", norm_features=False, without_fc=False, squeeze=True, center_bias=0):
    """(center bias) -> global pooling -> (L2 over C) -> squeeze -> fc -> L2, rmac_resnet.py:52-69."""
    if center_bias > 0:
        feat = feat * center_bias_map(center_bias, feat.shape[2], feat.shape[3])
    if pooling == "max":
        x = feat.amax(dim=(2, 3))
    elif pooling == "avg":
        x = feat.mean(dim=(2, 3))
    elif pooling.startswith("gem"):
        x = gem(feat, sd["adpool.p"].item())
    else:
        raise ValueError(pooling)
    if norm_features:
        x = F.normalize(x, p=2, dim=1)
    if not without_fc:
        x = F.linear(x, sd["fc.weight"], sd["fc.bias"])
    x = F.normalize(x, p=2, dim=-1)
    if squeeze and x.shape[0] == 1:  # x.squeeze_() drops the batch dim at B=1, rmac_resnet.py:64
        x = x[0]
    return x


@torch.no_grad()
def extract_fpn(x, sd, arch="resnet50_fpn_rmac", mode=1, norm_features=False, without_fc=False, squeeze=True):
    """ResNet_RMAC_FPN.forward, rmac_resnet_fpn.py:52-90: (layer3, layer4) maps; mode 1 adds the 1x1-reduced,
    nearest-upsampled layer4 map to layer3 and smooths with a 3x3 conv (no BN, ReLU after each); one GeM per map
    (own p each), concatenation [x4 | x5], (L2), fc, L2.  Oracle only so far (DESIGN.md section 6)."""
    _, stages = trunk(x, sd, arch.replace("_fpn0", "").replace("_fpn", ""), return_stages=True)
    x4, x5 = stages["layer3"], stages["layer4"]
    if mode == 1:
        c5 = F.interpolate(x5, size=x4.shape[-2:], mode="nearest")
        c5 = F.relu(F.conv2d(c5, sd["conv1x5.weight"]))
        x4 = F.relu(F.conv2d(x4 + c5, sd["conv3c4.weight"], None, padding=1))
    v = torch.cat([gem(x4, sd["adpoolc4.p"].item()), gem(x5, sd["adpoolx5.p"].item())], dim=1)
    if norm_features:
        v = F.normalize(v, p=2, dim=1)
    if not without_fc:
        v = F.linear(v, sd["fc.weight"], sd["fc.bias"])
    v = F.normalize(v, p=2, dim=-1)
    return v[0] if (squeeze and v.shape[0] == 1) else v


@torch.no_grad()
def extract(x, sd, arch="resnet50_rmac", **head_kw):
    """net(imgs): NCHW fp32 normalised images -> L2-normalised descriptors, rmac_resnet.py:39-69."""
    return head(trunk(x, sd, arch), sd, **head_kw)


# --------------------------------------------------------------------------- post-processing
def pool_scales(xs, pooling="mean", gemp=3):
    """common.pool, common.py:41-55: across transform chains; S=1 is the identity."""
    if len(xs) == 1:
        return xs[0]
    x = np.stack([np.asarray(v, dtype=np.float32) for v in xs], axis=0)
    if pooling == "mean":
        return x.mean(axis=0)
    if pooling == "gem":
        def sympow(v, p, eps=1e-6):
            s = np.sign(v)
            return np.power(np.maximum(v * s, eps), p).astype(np.float32) * s
        return sympow(sympow(x, gemp).mean(axis=0), 1.0 / gemp)
    raise ValueError("Bad pooling mode: " + str(pooling))


def l2n(x, eps=1e-12):
    """F.normalize(p=2, dim=1), test_dir.py:121-122."""
    x = np.asarray(x)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), eps)


def whiten_features(X, pca, l2norm=True, whitenp=0.5, whitenv=None, whitenm=1.0):
    """common.transform + whiten_features, common.py:221-239 (sklearn branch)."""
    X = np.asarray(X)
    if pca.mean_ is not None:
        X = X - pca.mean_
    Y = np.dot(X, pca.components_[:whitenv].T)
    if pca.whiten:
        Y = Y / (whitenm * np.power(pca.explained_variance_[:whitenv], whitenp))
    if l2norm:
        Y = Y / np.expand_dims(np.linalg.norm(Y, axis=1), axis=1)
    return Y


def scores_exact(Q, DB):
    """common.matmul, common.py:30-38: A . B^T.  Accumulated in fp64 so that the ordering it
    induces does not depend on a BLAS summation order (the reference's fp32 np.dot agrees with
    it to ~1e-7 absolute)."""
    return np.dot(np.asarray(Q, dtype=np.float64), np.asarray(DB, dtype=np.float64).T)


def rank_desc(scores_row):
    """Full descending order of one score row, ties -> lower index first.
    Reference: np.argsort(scores)[::-1] (generic.py:207,221) / (-scores).argsort() (dataset.py:100);
    those are unstable under exact ties, so the oracle fixes the tie order."""
    s = np.asarray(scores_row)
    return np.lexsort((np.arange(s.shape[0]), -s))


def topk(Q, DB, k, chunk=64):
    """Top-k by exact score, (score desc, index asc).  Returns (scores fp64 [Q,k], idx int64 [Q,k])."""
    Q = np.asarray(Q)
    n = DB.shape[0]
    k = min(k, n)
    out_s = np.empty((Q.shape[0], k), dtype=np.float64)
    out_i = np.empty((Q.shape[0], k), dtype=np.int64)
    for s0 in range(0, Q.shape[0], chunk):
        sc = scores_exact(Q[s0:s0 + chunk], DB)
        for r in range(sc.shape[0]):
            row = sc[r]
            if k < n:
                kth = np.partition(row, n - k)[n - k]
                cand = np.nonzero(row >= kth)[0]
            else:
                cand = np.arange(n)
            order = cand[np.lexsort((cand, -row[cand]))][:k]
            out_i[s0 + r] = order
            out_s[s0 + r] = row[order]
    return out_s, out_i


def merge_topk(shard_scores, shard_idx, k):
    """Merge per-shard top-k lists (global indices) into the global top-k, same order rule."""
    s = np.concatenate(shard_scores, axis=1)
    i = np.concatenate(shard_idx, axis=1)
    out_s = np.empty((s.shape[0], k), dtype=s.dtype)
    out_i = np.empty((s.shape[0], k), dtype=i.dtype)
    for r in range(s.shape[0]):
        order = np.lexsort((i[r], -s[r]))[:k]
        out_s[r], out_i[r] = s[r][order], i[r][order]
    return out_s, out_i


def expand_descriptors(descs, db=None, alpha=0, k=0):
    """alpha query expansion / database augmentation, test_dir.py:24-44.
    q' = normalize(mean([q] + [db_j * sim_ij^alpha for j in top-k(i)]))."""
    if k == 0:
        return descs
    descs = np.asarray(descs)
    n = descs.shape[0]
    dbd = np.asarray(db if db is not None else descs)
    sim = np.dot(descs, dbd.T)
    if db is None:
        sim[np.diag_indices(n)] = 0
    out = np.zeros_like(descs)
    for i in range(n):
        idx = rank_desc(sim[i])[:k]           # the reference takes an unordered argpartition; the mean is order-free
        rows = [descs[i]] + [dbd[j, :] * sim[i, j] ** alpha for j in idx]
        new_q = np.mean(np.vstack(rows), axis=0)
        out[i] = new_q / np.linalg.norm(new_q)
    return out


# --------------------------------------------------------------------------- evaluation
def average_precision(positive_ranks):
    """Trapezoidal AP over zero-based ranks of the positives, evaluation.py:46-82."""
    n = len(positive_ranks)
    if n == 0:
        return 0.0
    ap = 0.0
    for i, rank in enumerate(positive_ranks):
        left = 1.0 if rank == 0 else i / rank
        right = (i + 1) / (rank + 1)
        ap += (left + right) / (2.0 * n)
    return ap


def eval_query_ap(scores_row, ok, junk):
    """ImageListRelevants.eval_query_AP (classic mode), generic.py:196-209: drop junk, sort, AP."""
    n = scores_row.shape[0]
    gt = -np.ones(n, dtype=np.int8)
    gt[list(ok)] = 1
    gt[list(junk)] = 0
    keep = gt != 0
    gt, sc = gt[keep], np.asarray(scores_row)[keep]
    gt_sorted = gt[rank_desc(sc)]
    return average_precision(np.where(gt_sorted == 1)[0])


def ap_from_positive_ranks(pos_ranks_with_junk_removed):
    """AP when the (junk-free) ranks of the positives are already known (top-k engines)."""
    return average_precision(np.sort(np.asarray(pos_ranks_with_junk_removed)))


def rank_counts(Q, DB, t_off, t_rows):
    """What the ranking of generic.py:207,221 says about the labelled rows only: for target t of query q the exact
    score and the number of database rows that come before it in rank_desc (score desc, ties -> lower index)."""
    sc_out = np.zeros(len(t_rows), dtype=np.float64)
    above = np.zeros(len(t_rows), dtype=np.int64)
    for q in range(len(t_off) - 1):
        row = scores_exact(np.asarray(Q)[q:q + 1], DB)[0]
        for t in range(t_off[q], t_off[q + 1]):
            r = int(t_rows[t])
            s = row[r]
            sc_out[t] = s
            above[t] = int((row > s).sum() + (row[:r] == s).sum())
    return sc_out, above


def mean_ap(scores, gnd):
    """test_dir.py:153-159: mean over queries with AP >= 0."""
    aps = [eval_query_ap(scores[q], g["ok"], g["junk"]) for q, g in enumerate(gnd)]
    return float(np.mean([a for a in aps if a >= 0])), aps
