"""Spherical k-means of unit descriptors on the GPU (extension; DESIGN.md section 4.9, rules K1-K7).

Centres are unit rows and the similarity is the library's exact score e(x, c) (the fp64 score of ``ops.Index.search``).
Each iteration assigns every row to its best centre (the exact top-1 of ``Index(C).search(X, 1)``, ties to the smallest
centre), gives each empty cluster the worst-placed row of a cluster that can spare one, and replaces every centre by the
normalised fp64 sum of its rows, summed in a fixed order.  Every step is deterministic, so a fit is bit-identical from
run to run, and ``tests/kmeans_model.py`` restates it in numpy.

``python -m dirtorch.cluster_features`` is the command-line front end (``cluster_features_main``).
"""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import torch

from . import inputs, lib, ops
from .duplicates import add_input_args, check_input_args, load_input

MAX_ROWS = (1 << 29) - 1   # k-means++ weights are up to 2^34 units of 2^-32 each; their int64 total holds 2^29 rows
INITS = ("k-means++", "random")


NEAREST_MAX_K = 16384      # measured on an H100 (results/h100_kmeans.json): nearest() beats search(X, 1) up to 16384 centres
                           # and loses at 65536, where the group maxima leave more candidate groups per row


def assign(x, centres, stats=None):
    """Rules K2 / K3: (labels int64 (N,), scores fp64 (N,)) = the exact nearest centre of each row, the top-1 of
    Index(centres).search(x, 1) bit for bit: by Index.nearest up to NEAREST_MAX_K centres, by that search beyond.
    stats: a dict whose band_rows / full_rescores are incremented by the nearest path."""
    idx = ops.Index(centres, check_norms=False)
    try:
        if centres.shape[0] > NEAREST_MAX_K:
            sc, lab = idx.search(x, 1)
            return lab[:, 0].contiguous(), sc[:, 0].contiguous()
        lab, sc = idx.nearest(x)
        if stats is not None:
            st = idx.nearest_stats()
            stats["band_rows"] += st["band_rows"]
            stats["full_rescores"] += st["full_rescores"]
    finally:
        idx.close()
    return lab, sc


def kmeans_pp_rows(x, k, seed):
    """Rule K7's D^2 sampling -> the k rows drawn (int64 host array).  ValueError when fewer than k rows are distinct."""
    n, d = x.shape
    rs = np.random.RandomState(seed)
    first = int(rs.randint(n))
    u = np.ascontiguousarray(rs.random_sample(k - 1), dtype=np.float64)
    chosen = torch.empty(k, dtype=torch.int64, device=x.device)
    ws = ops.workspace(lib.raw("dirb200_kmeans_pp_workspace_bytes")(n, k), x.device)
    lib.call("dirb200_kmeans_pp", ops._ptr(x), n, d, first, u.ctypes.data_as(C.c_void_p), k, ops._ptr(ws), ops._ptr(chosen),
             ops._stream())
    rows = chosen.cpu().numpy()
    if (rows < 0).any():
        raise ValueError("k-means++ ran out of weight: the rows hold fewer than %d distinct descriptors" % k)
    return rows


class SphericalKMeans:
    """Spherical k-means with exact scores and deterministic centre updates.

    n_clusters: K >= 1.  init: 'k-means++' (D^2 sampling from RandomState(seed)), 'random' (the rows
    RandomState(seed).permutation(N)[:K]) or a (K, D) array of unit rows.  max_iter: iterations of assign, relocate,
    update; the fit stops earlier when an assignment repeats the previous one.

    After fit(X): cluster_centers_ (K, D) fp32, labels_ int64 (N,), scores_ fp64 (N,) (CUDA tensors; the labels and
    scores are those of the returned centres), n_iter_ (iterations run), objective_ (the sum of scores_, summed in
    units of 2^-32) and stats_ = {band_rows: row assignments with more than one candidate group of centres,
    full_rescores: row assignments re-scored over all centres (both summed over the assignments), relocations: rows
    moved into empty clusters, zero_sums: centres kept because their rows summed to zero}."""

    def __init__(self, n_clusters, init="k-means++", max_iter=20, seed=0):
        self.n_clusters = n_clusters
        self.init = init
        self.max_iter = max_iter
        self.seed = seed

    def _params(self, n, d):
        k = inputs.check_int(self.n_clusters, "n_clusters")
        if k > n:
            raise ValueError("n_clusters = %d exceeds the number of rows (%d)" % (k, n))
        if n > MAX_ROWS:
            raise ValueError("at most %d rows can be clustered (got %d)" % (MAX_ROWS, n))
        if d % 64:
            raise ValueError("the descriptor dimension must be a multiple of 64 (got %d)" % d)
        inputs.check_int(self.max_iter, "max_iter", 0)
        return k

    def _initial_centres(self, x, k):
        n, d = x.shape
        init = self.init
        if isinstance(init, str):
            if init == "k-means++":
                rows = kmeans_pp_rows(x, k, self.seed)
            elif init == "random":
                rows = np.random.RandomState(self.seed).permutation(n)[:k]
            else:
                raise ValueError("init must be one of %s or a (K, D) array (got %r)" % (INITS, init))
            return x[torch.from_numpy(np.asarray(rows, np.int64)).to(x.device)].contiguous()
        c = inputs.rows(init, x.device, "init")
        if tuple(c.shape) != (k, d):
            raise ValueError("init must have shape (%d, %d) (got %s)" % (k, d, tuple(c.shape)))
        inputs.check_unit(c, "init")
        return c.clone()

    def fit(self, X, device=None):
        """X: (N, D) unit descriptors - a CUDA fp32 tensor, a host array / tensor / memmap or a DescriptorStore."""
        x = inputs.rows(X, device, "X")
        n, d = x.shape
        k = self._params(n, d)
        inputs.check_unit(x, "X")
        centres = self._initial_centres(x, k)
        dev = x.device
        counts = torch.empty(k, dtype=torch.int32, device=dev)
        ws_stats = ops.workspace(lib.raw("dirb200_kmeans_stats_workspace_bytes")(n, k), dev)
        ws_upd = ops.workspace(lib.raw("dirb200_kmeans_update_workspace_bytes")(n, k, d), dev)
        ws_rel = None
        out = (C.c_int64 * 3)()
        one = C.c_int64()
        prev, n_iter = None, 0
        stats = dict(band_rows=0, full_rescores=0, relocations=0, zero_sums=0)
        while True:
            labels, scores = assign(x, centres, stats)
            lib.call("dirb200_kmeans_stats", ops._ptr(labels), ops._ptr(scores), ops._ptr(prev), n, k, ops._ptr(ws_stats),
                     ops._ptr(counts), out, ops._stream())
            changed, objective, empty = out[0], out[1], out[2]
            if (prev is not None and changed == 0) or n_iter == self.max_iter:
                break
            if empty:
                if ws_rel is None:
                    ws_rel = ops.workspace(lib.raw("dirb200_kmeans_relocate_workspace_bytes")(n), dev)
                lib.call("dirb200_kmeans_relocate", ops._ptr(labels), ops._ptr(scores), n, k, ops._ptr(counts),
                         ops._ptr(ws_rel), C.byref(one), ops._stream())
                stats["relocations"] += one.value
            lib.call("dirb200_kmeans_update", ops._ptr(x), n, d, ops._ptr(labels), ops._ptr(counts), k, ops._ptr(centres),
                     ops._ptr(ws_upd), C.byref(one), ops._stream())
            stats["zero_sums"] += one.value
            prev = labels
            n_iter += 1
        self.cluster_centers_ = centres
        self.labels_ = labels
        self.scores_ = scores
        self.n_iter_ = n_iter
        self.objective_ = objective / 2.0 ** 32
        self.stats_ = stats
        return self

    def predict(self, X, device=None):
        """Rule K2 against the fitted centres -> labels int64 (N,) (CUDA)."""
        if not hasattr(self, "cluster_centers_"):
            raise ValueError("fit() first")
        x = inputs.rows(X, self.cluster_centers_.device if device is None else torch.device(device), "X")
        if x.shape[1] != self.cluster_centers_.shape[1]:
            raise ValueError("X has dimension %d, the centres %d" % (x.shape[1], self.cluster_centers_.shape[1]))
        inputs.check_unit(x, "X")
        if x.shape[0] == 0:
            return torch.empty(0, dtype=torch.int64, device=x.device)
        return assign(x, self.cluster_centers_.to(x.device))[0]


def parse_args(argv=None):
    import argparse
    p = argparse.ArgumentParser(description="Cluster descriptors with exact spherical k-means")
    p.add_argument("--n-clusters", type=int, required=True, help="number of clusters K")
    p.add_argument("--init", type=str, default="k-means++", help="k-means++, random, or an .npy of K unit rows")
    p.add_argument("--max-iter", type=int, default=20, help="most assign / relocate / update iterations")
    p.add_argument("--seed", type=int, default=0, help="seed of the initialisation")
    add_input_args(p)
    p.add_argument("--output", type=str, default="", help=".npz receiving labels, scores and centres")
    p.add_argument("--out-json", type=str, default="", help="json receiving the clusters (image keys with --dataset)")
    p.add_argument("--gpu", type=int, default=0, help="GPU id")
    args = p.parse_args(argv)
    check_input_args(p, args)
    if args.n_clusters < 1:
        p.error("--n-clusters must be >= 1")
    if args.max_iter < 0:
        p.error("--max-iter must be >= 0")
    if args.init not in INITS and not args.init.endswith(".npy"):
        p.error("--init must be k-means++, random or an .npy file")
    return args


def cluster_features_main(argv=None):
    """python -m dirtorch.cluster_features (extension): spherical k-means of a descriptor set."""
    args = parse_args(argv)
    torch.cuda.set_device(args.gpu)
    dataset, X = load_input(args)
    init = args.init if args.init in INITS else np.load(args.init)
    km = SphericalKMeans(args.n_clusters, init=init, max_iter=args.max_iter, seed=args.seed).fit(X)
    labels = km.labels_.cpu().numpy()
    sizes = np.bincount(labels, minlength=args.n_clusters)
    print(">> %d rows in %d clusters after %d iterations: objective %.6f, sizes %d .. %d, %d relocations, %d zero sums" % (
        len(labels), args.n_clusters, km.n_iter_, km.objective_, sizes.min(), sizes.max(), km.stats_["relocations"],
        km.stats_["zero_sums"]))
    res = dict(labels=labels, scores=km.scores_.cpu().numpy(), centres=km.cluster_centers_.cpu().numpy())
    if args.output:
        np.savez(args.output, **res)
        print("saved to " + args.output)
    if args.out_json:
        order = np.argsort(labels, kind="stable")
        bounds = np.concatenate([[0], np.cumsum(sizes)])
        clusters = [order[bounds[c]:bounds[c + 1]].tolist() for c in range(args.n_clusters)]
        if dataset is not None:
            clusters = [[dataset.get_key(i) for i in m] for m in clusters]
        with open(args.out_json, "w") as f:
            json.dump({"n_clusters": args.n_clusters, "n_iter": km.n_iter_, "objective": km.objective_,
                       "clusters": clusters}, f, indent=1)
        print("saved to " + args.out_json)
    return res
