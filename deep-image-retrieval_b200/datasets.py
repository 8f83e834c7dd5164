"""Minimal dataset layer behind the CLIs: image lists and Oxford-style retrieval ground truth.

Mirrors the parts of ``dirtorch/datasets`` the evaluation path touches: ``ImageList`` (generic.py:13-30),
``ImageListLabels`` / ``ImageListLabelsQ`` with the label-based AP and top-k of ``Dataset`` (generic.py:33-121,
dataset.py:69-101), ``ImageListRelevants`` + ``eval_query_AP`` (generic.py:120-224), ``ImageListROIs`` (generic.py:226-250),
the Oxford/Paris wrappers (oxford.py, paris.py) and ``create`` (create.py:19-24).  AP arithmetic follows
``utils/evaluation.py:46-82``.  File bookkeeping only - nothing here is on the GPU hot path.
"""
from __future__ import annotations

import os
import os.path as osp
import pickle

import numpy as np


def compute_average_precision(positive_ranks):
    """Trapezoidal AP over sorted zero-based ranks of the positives (Revisited Oxford/Paris convention)."""
    n = len(positive_ranks)
    if not n:
        return 0.0
    ap = 0.0
    for i, rank in enumerate(positive_ranks):
        left = 1.0 if not rank else i / rank
        right = (i + 1) / (rank + 1)
        ap += (left + right) / (2.0 * n)
    return ap


class Dataset:
    root = ""
    img_dir = ""
    nimg = 0
    nquery = 0

    def __len__(self):
        return self.nimg

    def get_key(self, i):
        raise NotImplementedError()

    def get_filename(self, i, root=None):
        return os.path.join(root or self.root, self.img_dir, self.get_key(i))

    def get_image(self, i, resize=None):
        from PIL import Image
        img = Image.open(self.get_filename(i)).convert("RGB")
        if resize:
            img = img.resize(resize, Image.LANCZOS if np.prod(resize) < np.prod(img.size) else Image.BICUBIC)
        return img

    def get_image_source(self, i):
        """(file name, crop box or None) that get_image(i) decodes: lets the extraction decode the file itself."""
        return self.get_filename(i), None

    def get_label(self, i, toint=False):
        raise NotImplementedError()

    def get_query_db(self):
        raise NotImplementedError()

    def eval_query_AP(self, query_idx, scores):
        raise NotImplementedError()

    def eval_query_top(self, query_idx, scores, k=(1, 5, 10, 20, 50, 100)):
        raise NotImplementedError()

    def __repr__(self):
        return "Dataset: %s\n  %d images, %d queries" % (type(self).__name__, self.nimg, self.nquery)


class ImageList(Dataset):
    """A list of images (text file, one path per row, or an explicit list)."""

    def __init__(self, img_list_path=None, root="", imgs=None):
        self.root = root
        self.imgs = list(imgs) if imgs is not None else [e.strip() for e in open(img_list_path) if e.strip()]
        self.nimg = len(self.imgs)

    def get_key(self, i):
        return self.imgs[i]


class ImageListLabels(Dataset):
    """Images with one class label each; every image is also a query and its positives are the other images of its
    class (generic.py:44-77; ground truth and AP: dataset.py:69-92 with sklearn's average_precision_score,
    evaluation.py:41-43).

    Input: a text file with ``<image path> <label>`` per row, a json ``{path: label}``, or explicit lists."""

    def __init__(self, img_list_path=None, root=None, imgs=None, labels=None, cls_idx=None):
        self.root = root or ""
        if imgs is None:
            if osp.splitext(img_list_path)[1] == ".json":
                import json
                with open(img_list_path) as f:
                    pairs = list(json.load(f).items())
            else:
                with open(img_list_path) as f:
                    pairs = [row.split(" ")[:2] for row in (e.strip() for e in f) if row]
            imgs, labels = [p[0] for p in pairs], [p[1] for p in pairs]
        assert len(imgs) == len(labels), "one label per image"
        self.imgs, self.labels = list(imgs), list(labels)
        self.nimg = len(self.imgs)
        self._index_classes(self.labels, cls_idx)

    def _index_classes(self, all_labels, cls_idx=None):
        # class ids in order of first appearance (callers may pin some ids through cls_idx)
        self.cls_idx = dict(cls_idx or {})
        free = (i for i in range(len(set(all_labels) | set(self.cls_idx))) if i not in set(self.cls_idx.values()))
        for lab in all_labels:
            if lab not in self.cls_idx:
                self.cls_idx[lab] = next(free)
        self.classes = [c for c, _ in sorted(self.cls_idx.items(), key=lambda kv: kv[1])]
        self.nclass = len(self.classes)
        self.c_relevant_idx = {}
        for i, lab in enumerate(self.labels):
            self.c_relevant_idx.setdefault(lab, []).append(i)

    def get_key(self, i):
        return self.imgs[i]

    def get_label(self, i, toint=False):
        return self.cls_idx[self.labels[i]] if toint else self.labels[i]

    def get_query_db(self):
        return self

    def get_query_groundtruth(self, query_idx, what="AP"):
        qdb = self.get_query_db()
        qlabel = qdb.get_label(query_idx)
        if what == "label":
            return qlabel
        if what != "AP":
            raise ValueError("Unknown ground-truth type: %s" % what)
        gt = -np.ones(self.nimg, dtype=np.int8)                  # negatives
        gt[self.c_relevant_idx.get(qlabel, [])] = 1              # same class
        if qdb is self:
            gt[query_idx] = 0                                    # the query itself is ignored
        return gt

    def eval_query_AP(self, query_idx, scores):
        from sklearn.metrics import average_precision_score
        gt = self.get_query_groundtruth(query_idx, "AP")
        scores = np.asarray(scores)
        assert gt.shape == scores.shape, "scores should have shape %s" % str(gt.shape)
        keep = gt != 0
        if not (gt[keep] > 0).any():
            return -1                                            # no relevant image: excluded from the mean
        return average_precision_score(gt[keep] > 0, scores[keep])

    def eval_query_top(self, query_idx, scores, k=(1, 5, 10, 20, 50, 100)):
        qlabel = self.get_query_groundtruth(query_idx, "label")
        correct = np.array([lab == qlabel for lab in self.labels], dtype=bool)[np.argsort(-np.asarray(scores))]
        return {k_: float(correct[:k_].any()) for k_ in k if k_ < len(correct)}

    # ---- the same AP / top-k from threshold counts (dirb200_index_count_ge) and a ranked prefix, no score row
    def _class_ids(self):
        """(class id of every database row, class id of every query); -1 for a query label absent from the database."""
        if getattr(self, "_ids", None) is None:
            qdb = self.get_query_db()
            db_ids = np.array([self.cls_idx[l] for l in self.labels], dtype=np.int64)
            present = set(self.labels)
            q_ids = np.array([self.cls_idx[l] if l in present else -1 for l in qdb.labels], dtype=np.int64)
            self._ids = (db_ids, q_ids)
        return self._ids

    def label_targets(self, queries=None):
        """Positives of the given queries (default: all), built at once and grouped by class: database rows with the
        query's label, the query's own row excluded when the queries are the database (get_query_groundtruth marks it
        0).  -> (t_off int64 (Q+1,), t_rows int64 (T,) ascending within each query, skip_row int64 (Q,), -1 = none)."""
        db_ids, q_ids = self._class_ids()
        queries = np.arange(len(q_ids), dtype=np.int64) if queries is None else np.asarray(queries, dtype=np.int64)
        qc = q_ids[queries]
        by_class = np.argsort(db_ids, kind="stable")                       # rows grouped by class, ascending inside
        nclass = int(max(db_ids.max(initial=-1), q_ids.max(initial=-1))) + 1
        size = np.bincount(db_ids, minlength=nclass)
        start = np.concatenate([[0], np.cumsum(size)[:-1]])
        n = np.where(qc >= 0, size[np.maximum(qc, 0)], 0)
        first = np.where(qc >= 0, start[np.maximum(qc, 0)], 0)
        off = np.concatenate([[0], np.cumsum(n)])
        pos = np.arange(off[-1], dtype=np.int64) - np.repeat(off[:-1] - first, n)
        rows = by_class[pos]
        skip = queries.copy() if self.get_query_db() is self else -np.ones(len(queries), dtype=np.int64)
        keep = rows != np.repeat(skip, n)
        n = n - (skip >= 0)                                  # a self-query's own row is always in its class
        return np.concatenate([[0], np.cumsum(n)]).astype(np.int64), rows[keep].astype(np.int64), skip

    def eval_query_AP_from_ge_counts(self, query_idx, thr, counts):
        """AP of `eval_query_AP` from the fp32 scores of the query's positives in descending order (thr) and, for each,
        the number of rows other than the query's own with a score >= it (counts, dirb200_index_count_ge):
        AP = (1/|P|) sum_t TP_t / c_t, TP_t = positives scoring >= thr[t] (tied positives share TP and c)."""
        thr = np.asarray(thr, dtype=np.float32)
        if thr.shape[0] == 0:
            return -1                                            # no relevant image: excluded from the mean
        tp = np.searchsorted(-thr, -thr, side="right")
        return float(np.sum(tp / np.asarray(counts, dtype=np.float64)) / thr.shape[0])

    def eval_query_top_from_ranking(self, query_idx, ranked_idx, k=(1, 5, 10, 20, 50, 100)):
        """`eval_query_top` from the database indices of the best-ranked rows (at least min(max(k), N - 1) of them)."""
        db_ids, q_ids = self._class_ids()
        correct = db_ids[np.asarray(ranked_idx, dtype=np.int64)] == q_ids[query_idx]
        return {k_: float(correct[:k_].any()) for k_ in k if k_ < self.nimg}


class ImageListLabelsQ(ImageListLabels):
    """Labelled database + a separate labelled query list (generic.py:80-105)."""

    def __init__(self, img_list_path, query_list_path, root=None):
        with open(query_list_path) as f:
            qpairs = [row.split(" ")[:2] for row in (e.strip() for e in f) if row]
        self.qimgs, self.qlabels = [p[0] for p in qpairs], [p[1] for p in qpairs]
        ImageListLabels.__init__(self, img_list_path, root=root)
        self.nquery = len(self.qimgs)

    def _index_classes(self, all_labels, cls_idx=None):
        ImageListLabels._index_classes(self, list(all_labels) + list(self.qlabels), cls_idx)

    def get_query_db(self):
        if getattr(self, "_qdb", None) is None:
            self._qdb = ImageListLabels(root=self.root, imgs=self.qimgs, labels=self.qlabels, cls_idx=self.cls_idx)
        return self._qdb


class ImageListROIs(Dataset):
    def __init__(self, root, img_dir, imgs, rois):
        self.root, self.img_dir, self.imgs, self.rois = root, img_dir, imgs, rois
        self.nimg = len(imgs)

    def get_key(self, i):
        return self.imgs[i]

    def get_image(self, i, resize=None):
        from PIL import Image
        img = Image.open(self.get_filename(i)).convert("RGB").crop(self.rois[i])
        if resize:
            img = img.resize(resize, Image.LANCZOS if np.prod(resize) < np.prod(img.size) else Image.BICUBIC)
        return img

    def get_image_source(self, i):
        return self.get_filename(i), tuple(self.rois[i])


class ImageListRelevants(Dataset):
    """Images + query list + per-query relevant / junk indices from an Oxford-format pickle."""

    def __init__(self, gt_file, root=None, img_dir="jpg", ext=".jpg"):
        self.root, self.img_dir = root, img_dir
        with open(gt_file, "rb") as f:
            gt = pickle.load(f)
        fix = lambda e: osp.splitext(e)[0] + (osp.splitext(e)[1] or ext)
        self.imgs = [fix(e) for e in gt["imlist"]]
        self.qimgs = [fix(e) for e in gt["qimlist"]]
        self.qroi = [tuple(e["bbx"]) for e in gt["gnd"]]
        if "ok" in gt["gnd"][0]:
            self.relevants = [e["ok"] for e in gt["gnd"]]
        else:
            self.relevants = None
            self.easy = [e["easy"] for e in gt["gnd"]]
            self.hard = [e["hard"] for e in gt["gnd"]]
        self.junk = [e["junk"] for e in gt["gnd"]]
        self.nimg, self.nquery = len(self.imgs), len(self.qimgs)

    def get_key(self, i):
        return self.imgs[i]

    def get_query_key(self, i):
        return self.qimgs[i]

    def get_query_db(self):
        return ImageListROIs(self.root, self.img_dir, self.qimgs, self.qroi)

    def get_relevants(self, q, mode="classic"):
        return {"classic": lambda: self.relevants[q], "easy": lambda: self.easy[q],
                "medium": lambda: self.easy[q] + self.hard[q], "hard": lambda: self.hard[q]}[mode]()

    def get_junk(self, q, mode="classic"):
        return {"classic": lambda: self.junk[q], "easy": lambda: self.junk[q] + self.hard[q],
                "medium": lambda: self.junk[q], "hard": lambda: self.junk[q] + self.easy[q]}[mode]()

    def get_query_groundtruth(self, q, what="AP", mode="classic"):
        res = -np.ones(self.nimg, dtype=np.int8)
        res[self.get_relevants(q, mode)] = 1
        res[self.get_junk(q, mode)] = 0
        return res

    def _ap(self, q, scores, mode):
        gt = self.get_query_groundtruth(q, "AP", mode)
        assert gt.shape == scores.shape, "scores should have shape %s" % str(gt.shape)
        keep = gt != 0
        if mode != "classic" and (gt[keep] > 0).sum() == 0:
            return -1
        gt, sc = gt[keep], scores[keep]
        order = np.lexsort((np.arange(sc.shape[0]), -sc))          # descending, ties -> lower index
        return compute_average_precision(np.where(gt[order] == 1)[0])

    def eval_query_AP(self, query_idx, scores):
        scores = np.asarray(scores)
        if self.relevants:
            return self._ap(query_idx, scores, "classic")
        return {m: self._ap(query_idx, scores, m) for m in ("easy", "medium", "hard")}

    # ---- the same AP from a ranked PREFIX (top-k engine) instead of a full score row
    def _ap_from_ranking(self, q, ranked_idx, mode):
        rel = set(int(i) for i in self.get_relevants(q, mode))
        junk = set(int(i) for i in self.get_junk(q, mode))
        rel -= junk                                  # a label set to 0 (junk) after 1 wins, as in get_query_groundtruth
        if mode != "classic" and not rel:
            return -1
        ranks, pos, found = [], 0, 0
        for i in ranked_idx:
            i = int(i)
            if i < 0 or i in junk:
                continue
            if i in rel:
                ranks.append(pos)
                found += 1
                if found == len(rel):
                    break
            pos += 1
        if found < len(rel):
            return None                              # prefix too short: some positive ranks are unknown
        return compute_average_precision(ranks)

    def eval_query_AP_from_ranking(self, query_idx, ranked_idx):
        """AP of `eval_query_AP` computed from the first entries of the ranking (database indices, best first).
        Returns None (or a dict containing None) when the prefix does not reach every positive."""
        if self.relevants:
            return self._ap_from_ranking(query_idx, ranked_idx, "classic")
        return {m: self._ap_from_ranking(query_idx, ranked_idx, m) for m in ("easy", "medium", "hard")}


    # ---- the same AP from rank COUNTS of the labelled rows (dirb200_index_rank_count) instead of a full score row
    def rank_targets(self, q):
        """Labelled rows of query q for the counting kernel: (rows int64 sorted, flags uint8); flag 1 = the row is a
        positive in some evaluation mode (its rank is needed), 0 = junk only (its score suffices)."""
        if self.relevants:
            pos, junk = set(int(i) for i in self.relevants[q]), set(int(i) for i in self.junk[q])
        else:
            pos = set(int(i) for i in self.easy[q]) | set(int(i) for i in self.hard[q])
            junk = set(int(i) for i in self.junk[q])
        rows = np.array(sorted(pos | junk), dtype=np.int64)
        flags = np.array([1 if int(r) in pos else 0 for r in rows], dtype=np.uint8)
        return rows, flags

    def _ap_from_counts(self, q, rows, scores, above, mode, inside=None):
        rel = set(int(i) for i in self.get_relevants(q, mode))
        junk = set(int(i) for i in self.get_junk(q, mode))
        rel -= junk                                  # a label set to 0 (junk) after 1 wins, as in get_query_groundtruth
        if mode != "classic" and not rel:
            return -1
        at = {int(r): i for i, r in enumerate(rows)}
        jidx = np.array(sorted(junk), dtype=np.int64)
        js = np.array([scores[at[int(j)]] for j in jidx], dtype=np.float64)
        ranks = []
        for p in rel:
            sp = scores[at[p]]
            if inside is None:
                before = int(((js > sp) | ((js == sp) & (jidx < p))).sum()) if len(jidx) else 0   # junk rows ranked before p
            else:                                                 # (inside R_q, value, index) order of truncation
                ip = bool(inside[at[p]])
                ji = np.array([bool(inside[at[int(j)]]) for j in jidx], dtype=bool)
                before = int(((ji & (not ip)) | ((ji == ip) & ((js > sp) | ((js == sp) & (jidx < p))))).sum()) \
                    if len(jidx) else 0
            ranks.append(int(above[at[p]]) - before)
        return compute_average_precision(np.sort(np.array(ranks, dtype=np.int64)))

    def eval_query_AP_from_truncated_counts(self, query_idx, rows, inside, values, above):
        """eval_query_AP_from_counts for truncated diffusion: the rows of R_q (inside) rank before all others, so a
        junk row ranks before a positive by (inside, value, index) - f' inside R_q, the exact score outside."""
        if self.relevants:
            return self._ap_from_counts(query_idx, rows, values, above, "classic", inside)
        return {m: self._ap_from_counts(query_idx, rows, values, above, m, inside) for m in ("easy", "medium", "hard")}

    def eval_query_AP_from_counts(self, query_idx, rows, scores, above):
        """AP of `eval_query_AP` from the exact scores of the labelled rows and, for each positive, the number of
        database rows ranking before it (score desc, ties -> lower index): position among the non-junk rows =
        that count minus the junk rows that rank before it."""
        if self.relevants:
            return self._ap_from_counts(query_idx, rows, scores, above, "classic")
        return {m: self._ap_from_counts(query_idx, rows, scores, above, m) for m in ("easy", "medium", "hard")}


def _db_root():
    return os.environ["DB_ROOT"]


def _oxford_like(name, gnd):
    class _DS(ImageListRelevants):
        def __init__(self):
            ImageListRelevants.__init__(self, os.path.join(_db_root(), name, gnd), root=os.path.join(_db_root(), name))
    return _DS


Oxford5K = _oxford_like("oxford5k", "gnd_oxford5k.pkl")
ROxford5K = _oxford_like("oxford5k", "gnd_roxford5k.pkl")
Paris6K = _oxford_like("paris6k", "gnd_paris6k.pkl")
RParis6K = _oxford_like("paris6k", "gnd_rparis6k.pkl")
for _n, _c in (("Oxford5K", Oxford5K), ("ROxford5K", ROxford5K), ("Paris6K", Paris6K), ("RParis6K", RParis6K)):
    _c.__name__ = _n


def create(dataset_cmd):
    """datasets.create: evaluate a dataset expression such as ``ImageList("list.txt", "imgs")`` (create.py:19-24)."""
    if "(" not in dataset_cmd:
        dataset_cmd += "()"
    names = {k: v for k, v in globals().items() if isinstance(v, type) and issubclass(v, Dataset)}
    try:
        return eval(dataset_cmd, {"__builtins__": {}}, names)
    except NameError:
        import sys
        print("Error: unknown dataset %s\nAvailable datasets: %s" % (dataset_cmd.replace("()", ""), ", ".join(sorted(names))),
              file=sys.stderr)
        sys.exit(1)
