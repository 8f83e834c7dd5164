"""Near-duplicate detection and set overlap by exact range search (extension; DESIGN.md section 4.8, rules J1-J6).

``near_duplicates(descs, tau)`` finds every pair of rows (i, j), i < j, whose exact score e(x_i, x_j) (the fp64 score of
the search) reaches tau, with the triangular self-join of ``ops.Index.self_join``, then the connected components of that
pair graph: label(i) is the smallest row of i's component, and a group is a component of at least two rows.
``overlap(qdescs, bdescs, tau)`` lists, for every row of the first set, the rows of the second with e >= tau
(``ops.Index.range_search``).  Both are exact for any tau: nothing is dropped when many rows match.

``python -m dirtorch.find_duplicates`` is the command-line front end (``find_duplicates_main``).
"""
from __future__ import annotations

import json
import math
import os
import tempfile
from typing import NamedTuple

import numpy as np
import torch

from . import inputs, ops
from .store import DescriptorStore


class Duplicates(NamedTuple):
    """off / cols / scores: the pairs as a CSR by the first row (off int64 (N+1,), partners j > i int64, exact scores
    fp64, each row's partners by (score desc, j asc)); labels int64 (N,); groups = (group offsets int64 (G+1,), members
    int64): group g is members[off[g]:off[g+1]], groups by ascending label, members ascending.  CUDA tensors."""
    off: torch.Tensor
    cols: torch.Tensor
    scores: torch.Tensor
    labels: torch.Tensor
    groups: tuple

    def group_lists(self):
        """The groups as Python lists of row indices."""
        goff, mem = (t.cpu().numpy() for t in self.groups)
        return [mem[goff[g]:goff[g + 1]].tolist() for g in range(len(goff) - 1)]


def check_tau(tau):
    try:
        t = float(tau)
    except (TypeError, ValueError):
        raise ValueError("tau must be a finite number (got %r)" % (tau,))
    if not math.isfinite(t):
        raise ValueError("tau must be finite (got %r)" % (tau,))
    return t


def _index(x, eps16):
    idx = ops.Index(x, check_norms=False)
    if eps16 is not None:
        e = float(eps16)
        if not (math.isfinite(e) and e > 0):
            raise ValueError("eps16 must be a positive finite number (got %r)" % (eps16,))
        idx.set_option("eps16", e)
    return idx


def near_duplicates(descs, tau, eps16=None, row_block=None, device=None) -> Duplicates:
    """Every pair i < j of rows with exact score >= tau, its connected components and the groups they form.
    descs: (N, D) descriptors - a CUDA tensor, a host array / tensor or a DescriptorStore.  Rows must be unit-norm
    unless eps16 (the bound on |fp16-path score - exact score|, ops.Index's recipe) is given.  row_block: rows joined
    per tensor-core launch sequence (a multiple of 128; the result does not depend on it)."""
    tau = check_tau(tau)
    x = inputs.rows(descs, device, "descs")
    if eps16 is None:
        inputs.check_norm_at_most_1(x, "descs")
    n = x.shape[0]
    if n == 0:
        z = torch.zeros(1, dtype=torch.int64, device=x.device)
        e = torch.empty(0, dtype=torch.int64, device=x.device)
        return Duplicates(z, e, torch.empty(0, dtype=torch.float64, device=x.device), e, (z, e))
    idx = _index(x, eps16)
    try:
        off, cols, scores = idx.self_join(tau, row_block=row_block)
    finally:
        idx.close()
    labels = ops.join_components(off, cols, n)
    return Duplicates(off, cols, scores, labels, ops.join_groups(labels))


def overlap(qdescs, bdescs, tau, eps16=None, device=None):
    """For every row q of the first set, the rows r of the second with exact score e(q, r) >= tau, ordered by (score
    desc, r asc) -> CSR (offsets int64 (Q+1,), rows int64, scores fp64), CUDA tensors.  Same inputs as near_duplicates;
    both sets must have the same dimension."""
    tau = check_tau(tau)
    dev = inputs.device(device)
    q = inputs.rows(qdescs, dev, "qdescs")
    b = inputs.rows(bdescs, dev, "bdescs")
    if q.shape[1] != b.shape[1]:
        raise ValueError("the two sets have different dimensions (%d and %d)" % (q.shape[1], b.shape[1]))
    if eps16 is None:
        inputs.check_norm_at_most_1(q, "qdescs")
        inputs.check_norm_at_most_1(b, "bdescs")
    if q.shape[0] == 0:
        return (torch.zeros(1, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int64, device=dev),
                torch.empty(0, dtype=torch.float64, device=dev))
    idx = _index(b, eps16)
    try:
        return idx.range_search(q, tau)
    finally:
        idx.close()


def pairs_from_csr(off, cols):
    """CSR (offsets, partners) -> (P, 2) int64 host array of (row, partner)."""
    off = off.cpu().numpy()
    first = np.repeat(np.arange(len(off) - 1, dtype=np.int64), np.diff(off))
    return np.stack([first, cols.cpu().numpy()], 1) if len(first) else np.zeros((0, 2), np.int64)


def _load_set(path):
    if DescriptorStore.is_store(path):
        return DescriptorStore(path)
    if os.path.isfile(path):
        return np.load(path, mmap_mode="r")
    raise ValueError("%s is neither a descriptor store nor an .npy file" % path)


def add_input_args(p):
    """The descriptor-set inputs shared by the command lines that read one set: an .npy, a store, or a dataset to extract
    with a checkpoint and the usual extraction and whitening flags."""
    p.add_argument("--load-feats", type=str, default="", help=".npy of descriptors")
    p.add_argument("--store", type=str, default="", help="descriptor store")
    p.add_argument("--dataset", "-d", type=str, default="", help="command to load the dataset to extract")
    p.add_argument("--checkpoint", type=str, default="", help="path to weights (with --dataset)")
    p.add_argument("--trfs", type=str, required=False, default="", nargs="+", help="test transforms (can be several)")
    p.add_argument("--pooling", type=str, default="gem", help="pooling scheme if several trf chains")
    p.add_argument("--gemp", type=int, default=3, help="GeM pooling power")
    p.add_argument("--whiten", type=str, default=None, help="applies whitening")
    p.add_argument("--whitenp", type=float, default=0.5, help="whitening power")
    p.add_argument("--whitenv", type=int, default=None, help="number of components, default is None (all)")
    p.add_argument("--whitenm", type=float, default=1.0, help="whitening multiplier")
    p.add_argument("--threads", type=int, default=8, help="number of thread workers")


def check_input_args(p, args):
    if sum(bool(s) for s in (args.dataset, args.load_feats, args.store)) != 1:
        p.error("exactly one of --dataset, --load-feats and --store is required")
    if args.dataset and not args.checkpoint:
        p.error("--dataset needs --checkpoint")


def load_input(args):
    """(dataset or None, descriptors) of the inputs add_input_args declares."""
    if args.dataset:
        return _extract(args)
    if args.load_feats:
        return None, _load_set(args.load_feats)
    return None, DescriptorStore(args.store)


def parse_args(argv=None):
    import argparse
    p = argparse.ArgumentParser(description="Find near-duplicate descriptors (every pair with exact score >= T) and "
                                            "their groups, or the overlap of two sets")
    p.add_argument("--threshold", type=float, required=True, help="score threshold T (inclusive)")
    add_input_args(p)
    p.add_argument("--against", type=str, default="", help=".npy or store: report, for each row of the first set, "
                                                           "the rows of this set with score >= T")
    p.add_argument("--eps16", type=float, default=None, help="score error bound for rows that are not unit-norm")
    p.add_argument("--output", type=str, default="", help=".npz receiving pairs, scores (and labels)")
    p.add_argument("--out-json", type=str, default="", help="json receiving the groups (image keys with --dataset)")
    p.add_argument("--gpu", type=int, default=0, help="GPU id")
    args = p.parse_args(argv)
    check_input_args(p, args)
    if not math.isfinite(args.threshold):
        p.error("--threshold must be finite")
    if args.eps16 is not None and not (math.isfinite(args.eps16) and args.eps16 > 0):
        p.error("--eps16 must be a positive number")
    if args.out_json and args.against:
        p.error("--out-json lists duplicate groups; it does not apply to --against")
    return args


def _extract(args):
    """Descriptors of the dataset's database images, as extract_features writes them."""
    from . import datasets
    from .pipeline import _select_pca, extract_features, load_model
    dataset = datasets.create(args.dataset)
    print("Dataset:", dataset)
    net = load_model(args.checkpoint, True)
    whiten = _select_pca(net, args)
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "feats.npy")
        extract_features(dataset, net, args.trfs, pooling=args.pooling, gemp=args.gemp, whiten=whiten,
                         threads=args.threads, output=out)
        if not os.path.exists(out):            # a dataset with its own query list: database rows only
            out = os.path.join(tmp, "feats.dbdescs.npy")
        return dataset, np.load(out)


def find_duplicates_main(argv=None):
    """python -m dirtorch.find_duplicates (extension): every pair of rows with exact score >= --threshold and their
    groups (connected components), or with --against the rows of a second set that each row reaches."""
    args = parse_args(argv)
    torch.cuda.set_device(args.gpu)
    dataset, X = load_input(args)
    if args.against:
        off, rows, scores = overlap(X, _load_set(args.against), args.threshold, eps16=args.eps16)
        pairs = pairs_from_csr(off, rows)
        hit = np.diff(off.cpu().numpy()) > 0
        print(">> %d rows against %d: %d pairs with score >= %g, %d rows with a match" % (
            len(off) - 1, len(_load_set(args.against)), len(pairs), args.threshold, int(hit.sum())))
        res = dict(pairs=pairs, scores=scores.cpu().numpy())
    else:
        d = near_duplicates(X, args.threshold, eps16=args.eps16)
        pairs = pairs_from_csr(d.off, d.cols)
        groups = d.group_lists()
        largest = max((len(g) for g in groups), default=0)
        print(">> %d rows: %d pairs with score >= %g, %d groups, largest group %d rows" % (
            len(d.labels), len(pairs), args.threshold, len(groups), largest))
        res = dict(pairs=pairs, scores=d.scores.cpu().numpy(), labels=d.labels.cpu().numpy(), groups=groups)
        if args.out_json:
            named = [[dataset.get_key(i) for i in g] for g in groups] if dataset is not None else groups
            with open(args.out_json, "w") as f:
                json.dump({"threshold": args.threshold, "groups": named}, f, indent=1)
            print("saved to " + args.out_json)
    if args.output:
        np.savez(args.output, **{k: v for k, v in res.items() if k != "groups"})
        print("saved to " + args.output)
    return res
