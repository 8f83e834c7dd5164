"""GPU-backed equivalents of the helpers in ``dirtorch/utils/common.py`` that sit on the hot path
(``tonumpy, matmul, pool, transform, whiten_features``) plus the runtime glue the CLIs call
(``torch_set_gpu, torch_set_seed, load_checkpoint, switch_model_to_cuda, variables``).

Same names, argument meaning and error behaviour as the reference; the arithmetic runs in libdirb200
on the current CUDA device.  There is no CPU execution path: ``torch_set_gpu([-1])`` raises.
"""
from __future__ import annotations

import os
import sys
from collections import OrderedDict

import numpy as np
import torch

from . import inputs, ops


def typename(x):
    return type(x).__module__


def tonumpy(x):
    """common.py:23-27."""
    if typename(x) == torch.__name__:
        return x.cpu().numpy()
    return x


def matmul(A, B):
    """scores = A . B^T as a host ndarray (common.py:30-38); fp64-accumulated on the GPU, fp32 out."""
    if typename(A) == np.__name__:
        B = tonumpy(B)
    elif typename(B) != torch.__name__:
        raise TypeError("matrices must be either numpy or torch type")
    return ops.scores_exact(inputs.rows(A), inputs.rows(B)).cpu().numpy()


def pool(x, pooling="mean", gemp=3):
    """Pool descriptors of several transform chains (common.py:41-55).  x: list of (N,D) torch tensors."""
    if len(x) == 1:
        return x[0]
    if pooling not in ("mean", "gem"):
        raise ValueError("Bad pooling mode: " + str(pooling))
    return ops.pool_scales([inputs.rows(v) for v in x], pooling, gemp, l2=False)


def torch_set_gpu(gpus, seed=None, randomize=True):
    """common.py:58-81.  Only CUDA execution exists here."""
    if type(gpus) is int:
        gpus = [gpus]
    assert gpus, "error: empty gpu list, use --gpu N N ..."
    cuda = all(gpu >= 0 for gpu in gpus)
    if not cuda:
        raise RuntimeError("dirb200 has no CPU execution path (--gpu %s): the hot path runs only on an sm_90 (H100) GPU" % gpus)
    if any(gpu >= 1000 for gpu in gpus):
        visible = [int(g) for g in os.environ["CUDA_VISIBLE_DEVICES"].split(",")]
        os.environ["CUDA_VISIBLE_DEVICES"] = ",".join(str(visible[g - 1000]) for g in gpus)
    else:
        os.environ["CUDA_VISIBLE_DEVICES"] = ",".join(str(g) for g in gpus)
    assert torch.cuda.is_available(), "%s has GPUs %s unavailable" % (
        os.environ.get("HOSTNAME", "?"), os.environ["CUDA_VISIBLE_DEVICES"])
    ops.require_gpu(0)
    print("Launching on GPUs " + os.environ["CUDA_VISIBLE_DEVICES"])
    torch_set_seed(seed, cuda, randomize=randomize)
    return cuda


def torch_set_seed(seed, cuda, randomize=True):
    if randomize and not seed:
        seed = int.from_bytes(os.urandom(4), byteorder="little", signed=False)
    if seed:
        np.random.seed(seed % (2 ** 32))
        torch.manual_seed(seed)
        if cuda:
            torch.cuda.manual_seed(seed)


def save_checkpoint(state, is_best, filename):
    """common.py:100-112: write the checkpoint dict ({state_dict, model_options, preprocess?, pca?, ...}); a copy named
    ``<filename>.best`` when is_best.  Errors are reported, not raised, like the reference."""
    import shutil
    try:
        folder = os.path.split(filename)[0]
        if folder and not os.path.isdir(folder):
            os.makedirs(folder)
        torch.save(state, filename)
        if is_best:
            shutil.copyfile(filename, filename + ".best")
            filename += ".best"
        print("saving to " + filename)
    except Exception:
        print("Error: Could not save checkpoint at %s, skipping" % filename)


def model_size(model):
    """common.py:178-184: number of parameters (all state-dict tensors)."""
    return int(sum(int(np.prod(tuple(w.shape))) for w in model.state_dict().values()))


def load_checkpoint(filename, iscuda=False):
    """common.py:117-147: torch.load of {state_dict, model_options, preprocess?, pca?}, 'module.' stripped."""
    if not filename:
        return None
    assert os.path.isfile(filename), "=> no checkpoint found at '%s'" % filename
    checkpoint = torch.load(filename, map_location="cpu", weights_only=False)   # the dict pickles an sklearn PCA
    print("=> loading checkpoint '%s'" % filename, end="")
    for key in ["epoch", "iter", "current_iter"]:
        if key in checkpoint:
            print(" (%s %d)" % (key, checkpoint[key]), end="")
    print()
    new_dict = OrderedDict()
    for k, v in list(checkpoint["state_dict"].items()):
        new_dict[k[7:] if k.startswith("module.") else k] = v
    checkpoint["state_dict"] = new_dict
    return checkpoint


def switch_model_to_cuda(model, iscuda=True, checkpoint=None):
    """common.py:150-175.  The reference wraps the model in nn.DataParallel; here one process drives one GPU
    (multi-GPU = one process per GPU, dirb200.dist), so the model is returned as is."""
    if not iscuda:
        raise RuntimeError("dirb200 has no CPU execution path")
    model.cuda()
    model.isasync = True
    model.iscuda = iscuda
    return model


def variables(inputs, iscuda, not_on_gpu=[]):
    """common.py:205-218: move tensors to the GPU."""
    out = []
    for i, x in enumerate(inputs):
        if i not in not_on_gpu and not isinstance(x, (tuple, list)) and iscuda:
            x = x.cuda(non_blocking=True)
        out.append(x)
    return out


def _pca_arrays(pca, whitenp, whitenv, whitenm, use_sklearn):
    if use_sklearn:
        comp = np.asarray(pca.components_[:whitenv], dtype=np.float64)
        mean = None if pca.mean_ is None else np.asarray(pca.mean_, dtype=np.float64)
        cs = None
        if pca.whiten:
            cs = 1.0 / (whitenm * np.power(np.asarray(pca.explained_variance_[:whitenv], dtype=np.float64), whitenp))
    else:
        comp = np.asarray(pca["W"], dtype=np.float64).T
        mean = np.asarray(pca["means"], dtype=np.float64)
        cs = None
    f = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).to(inputs.device())
    return f(comp), f(mean), f(cs)


def transform(pca, X, whitenp=0.5, whitenv=None, whitenm=1.0, use_sklearn=True):
    """common.py:221-232 (projection + whitening scale, no L2)."""
    comp, mean, cs = _pca_arrays(pca, whitenp, whitenv, whitenm, use_sklearn)
    return ops.whiten(inputs.rows(X), comp, mean, cs, l2norm=False).cpu().numpy()


def whiten_features(X, pca, l2norm=True, whitenp=0.5, whitenv=None, whitenm=1.0, use_sklearn=True):
    """common.py:235-239."""
    comp, mean, cs = _pca_arrays(pca, whitenp, whitenv, whitenm, use_sklearn)
    return ops.whiten(inputs.rows(X), comp, mean, cs, l2norm=l2norm).cpu().numpy()


def whiten_features_gpu(X, pca, l2norm=True, whitenp=0.5, whitenv=None, whitenm=1.0, want_f16=False):
    """Device-resident variant (no host round trip) for the search pipeline."""
    comp, mean, cs = _pca_arrays(pca, whitenp, whitenv, whitenm, True)
    return ops.whiten(inputs.rows(X), comp, mean, cs, l2norm=l2norm, want_f16=want_f16)
