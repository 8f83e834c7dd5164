"""The table of stream cases: one small call of every public entry point that launches work.

Each case is a function `build(mk)` that prepares its inputs on the default stream and returns `run`, a function of no
arguments that makes the call and returns its outputs (tensors, numbers, lists, tuples and dicts of them).  `mk(t)`
hands a device tensor the call reads to the case: tests/test_gpu_streams.py passes either the tensor itself or a buffer
filled with poison that is only filled with `t` on the caller's side stream, behind a gate.  `covers` names the C entry
points the case must reach (checked on the GPU by recording every `lib.call`); tests/test_stream_cases.py checks on the
CPU that every export of include/dirb200.h is covered here or listed in EXEMPT with its reason.

Imports of the package stay inside the cases, so that this module loads without a GPU."""
from __future__ import annotations

import functools
from typing import Callable, NamedTuple

import numpy as np
import torch


class Case(NamedTuple):
    name: str
    covers: tuple
    build: Callable
    options: dict        # global options (dirb200_set_global_option) held for both runs of the case


STREAM_CASES = []


def case(name, covers, options=None):
    def reg(fn):
        STREAM_CASES.append(Case(name, tuple("dirb200_" + c for c in covers), fn, dict(options or {})))
        return fn
    return reg


# Exports the table does not reach, each with its reason: none of them takes the caller's stream.
EXEMPT = {
    "dirb200_version": "host only: the ABI version",
    "dirb200_last_error": "host only: the thread's last message",
    "dirb200_device_check": "host only: device properties",
    "dirb200_set_global_option": "host setting; the cases run with both values of 'pdl', 'halo' and 'head_fused'",
    "dirb200_get_global_option": "host only",
    "dirb200_net_create": "handle creation, no device work",
    "dirb200_net_set_option": "host setting of a handle",
    "dirb200_net_set_tensor": "host copy of a weight into the handle",
    "dirb200_net_destroy": "handle destruction",
    "dirb200_net_forward_host": "_host forward: its own stream and synchronisation by design",
    "dirb200_net_forward_host_u8": "_host forward: its own stream and synchronisation by design",
    "dirb200_net_profile": "host read of the profile; synchronises the device itself",
    "dirb200_net_profile_table": "host read of the profile; synchronises the device itself",
    "dirb200_net_last_launches": "host counters of the last forward",
    "dirb200_resize_coeffs": "host only: PIL's coefficient table",
    "dirb200_jpeg_probe": "host only: header parse",
    "dirb200_jpeg_decoder_create": "handle creation",
    "dirb200_jpeg_decoder_set_option": "host setting of a handle",
    "dirb200_jpeg_decoder_destroy": "handle destruction",
    "dirb200_stem_workspace_bytes": "size query",
    "dirb200_stem_pack_weight": "host only: weight repack",
    "dirb200_head_workspace_floats": "size query",
    "dirb200_index_create": "handle creation",
    "dirb200_index_set_db": "host setting of a handle (pointers only)",
    "dirb200_index_set_option": "host setting of a handle",
    "dirb200_index_last_profile": "host read of CUDA-event timings of the last search",
    "dirb200_index_destroy": "handle destruction",
    "dirb200_exchange_ipc_handle": "CUDA IPC between processes: needs one process per rank",
    "dirb200_exchange_open": "CUDA IPC between processes: needs one process per rank",
    "dirb200_exchange_destroy": "handle destruction",
    "dirb200_diffusion_graph_workspace_bytes": "size query",
    "dirb200_diffusion_solve_workspace_bytes": "size query",
    "dirb200_diffusion_rank_count_workspace_bytes": "size query",
    "dirb200_diffusion_topk_workspace_bytes": "size query",
    "dirb200_diffusion_trunc_build_workspace_bytes": "size query",
    "dirb200_diffusion_trunc_solve_workspace_bytes": "size query",
    "dirb200_diffusion_trunc_topk_workspace_bytes": "size query",
    "dirb200_join_components_workspace_bytes": "size query",
    "dirb200_join_groups_workspace_bytes": "size query",
    "dirb200_kmeans_stats_workspace_bytes": "size query",
    "dirb200_kmeans_relocate_workspace_bytes": "size query",
    "dirb200_kmeans_update_workspace_bytes": "size query",
    "dirb200_kmeans_pp_workspace_bytes": "size query",
    "dirb200_pq_search_ws_bytes": "size query",
    "dirb200_graph_search_smem_bytes": "size query",
}


# ---------------------------------------------------------------------------------------------------------- inputs
def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def randn(*shape, seed=0, dtype=torch.float32, scale=1.0):
    a = np.random.RandomState(seed).standard_normal(shape) * scale
    return torch.from_numpy(a.astype(np.float32)).to(dtype).cuda()


def unit(n, d, seed=0):
    a = np.random.RandomState(seed).standard_normal((n, d))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    return torch.from_numpy(a.astype(np.float32)).cuda()


def clustered(n, d, centres=16, seed=0):
    """Unit rows around a few directions: k-means, IVF and graph builds have structure to find."""
    r = np.random.RandomState(seed)
    c = r.standard_normal((centres, d))
    a = c[r.randint(centres, size=n)] + 0.6 * r.standard_normal((n, d))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    return torch.from_numpy(a.astype(np.float32)).cuda()


def index(mk, db, offset=0):
    """An ops.Index over rows the search reads from buffers handed out by mk."""
    return _ops().Index(mk(db), index_offset=offset, db16=mk(db.half()), check_norms=False)


@functools.lru_cache(maxsize=None)
def _state_dict(arch):
    import synthdata as synth
    return synth.make_state_dict(arch, seed=1)


def model(arch="resnet50_rmac"):
    from dirb200 import nets
    net = nets.create_model(arch)
    net.load_state_dict(_state_dict(arch))
    return net.eval()


@functools.lru_cache(maxsize=None)
def shared_model():
    """One network for every forward case: its weights are uploaded once."""
    return model()


def images_u8(b, h, w, seed=0):
    import synthdata as synth
    return torch.from_numpy(synth.make_images_u8(b, h, w, seed=seed)).cuda()


def images(b, h, w, seed=0):
    import synthdata as synth
    return synth.make_images(b, h, w, seed=seed).cuda()


def conv_weights(cout, cin, k, seed):
    ops = _ops()
    r = np.random.RandomState(seed)
    w = torch.from_numpy((r.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32))
    scale = torch.from_numpy(r.uniform(0.5, 1.5, cout).astype(np.float32)).cuda()
    shift = torch.from_numpy((0.2 * r.standard_normal(cout)).astype(np.float32)).cuda()
    return ops.pack_conv_weight(w).cuda(), scale, shift, w


def targets(nq, n, per_q, seed):
    """A host CSR of per_q target rows per query, every other one flagged."""
    r = np.random.RandomState(seed)
    off = np.arange(nq + 1, dtype=np.int64) * per_q
    rows = np.concatenate([r.choice(n, per_q, replace=False) for _ in range(nq)]).astype(np.int64)
    flags = (np.arange(rows.shape[0]) % 2 == 0).astype(np.uint8)
    return off, rows, flags


# -------------------------------------------------------------------------------------------- network and extraction
@case("nchw_to_nhwc8", ["nchw_to_nhwc8"])
def _(mk):
    x = mk(images(2, 37, 53, seed=1))
    return lambda: _ops().nchw_to_nhwc8(x)


def _conv_case(mk, b, h, w, cin, cout, k, stride, pad, res, seed):
    wp, scale, shift, _ = conv_weights(cout, cin, k, seed)
    x = mk(randn(b, h, w, cin, seed=seed, dtype=torch.float16))
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    r = mk(randn(b, ho, wo, cout, seed=seed + 1, dtype=torch.float16)) if res else None
    wp, scale, shift = mk(wp), mk(scale), mk(shift)
    return lambda: _ops().conv_bn_act(x, wp, cout, k, k, stride, pad, scale, shift, res=r)


@case("conv_bn_act_1x1", ["conv_bn_act"])
def _(mk):
    return _conv_case(mk, 2, 14, 14, 256, 64, 1, 1, 0, False, seed=2)


@case("conv_bn_act_3x3_halo", ["conv_bn_act"], options={"halo": 1})
def _(mk):
    return _conv_case(mk, 2, 17, 9, 128, 128, 3, 1, 1, False, seed=3)


@case("conv_bn_act_3x3_taps", ["conv_bn_act"], options={"halo": 0})
def _(mk):
    return _conv_case(mk, 2, 17, 9, 128, 128, 3, 1, 1, False, seed=3)


@case("conv_bn_act_residual", ["conv_bn_act"])
def _(mk):
    return _conv_case(mk, 1, 24, 20, 64, 256, 1, 1, 0, True, seed=4)


@case("conv_c23", ["conv_c23"])
def _(mk):
    cm = 64
    w2p, s2, h2, _ = conv_weights(cm, cm, 3, 5)
    w3p, s3, h3, _ = conv_weights(4 * cm, cm, 1, 6)
    t1 = mk(torch.relu(randn(2, 16, 9, cm, seed=7)).half())
    res = mk(randn(2, 16, 9, 4 * cm, seed=8, dtype=torch.float16))
    w2p, w3p = mk(w2p), mk(w3p)
    return lambda: _ops().conv_c23(t1, w2p, s2, h2, w3p, s3, h3, res)


@case("conv_c31", ["conv_c31"])
def _(mk):
    cm = 64
    w3p, s3, h3, _ = conv_weights(4 * cm, cm, 1, 9)
    w1p, s1, h1, _ = conv_weights(cm, 4 * cm, 1, 10)
    t2 = mk(torch.relu(randn(2, 40, 3, cm, seed=11)).half())
    x = mk(torch.relu(randn(2, 40, 3, 4 * cm, seed=12)).half())
    w3p, w1p = mk(w3p), mk(w1p)
    return lambda: _ops().conv_c31(t2, w3p, s3, h3, x, w1p, s1, h1)


def _stem_args(mk):
    import layer_model as LM
    sd = _state_dict("resnet50_rmac")
    s, sh = LM.bn_fold(sd, "bn1", 64)
    return sd["conv1.weight"], mk(torch.from_numpy(s).cuda()), mk(torch.from_numpy(sh).cuda())


@case("stem_pool", ["stem_pool"])
def _(mk):
    w, s, sh = _stem_args(mk)
    x = mk(images(2, 63, 65, seed=13))
    return lambda: _ops().stem_pool(x, w, s, sh, stem_map=True)


@case("stem_pool_u8", ["stem_pool"])
def _(mk):
    w, s, sh = _stem_args(mk)
    x = mk(images_u8(2, 50, 71, seed=14))
    ms = ([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
    return lambda: _ops().stem_pool(x, w, s, sh, mean_std=ms)


@case("stem_conv", ["stem_conv"])
def _(mk):
    w, s, sh = _stem_args(mk)
    x = mk(images(2, 64, 96, seed=15))
    return lambda: _ops().stem_conv(x, w, s, sh)


@case("maxpool_3x3s2", ["maxpool_3x3s2"])
def _(mk):
    x = mk(randn(2, 33, 20, 64, seed=16, dtype=torch.float16))
    return lambda: _ops().maxpool_3x3s2(x)


def _head_case(mk):
    feat = mk(randn(3, 7, 9, 2048, seed=17).abs().half())
    fc_w = mk(randn(2048, 2048, seed=18, scale=1 / 45.0))
    fc_b = mk(randn(2048, seed=19, scale=0.01))
    return lambda: _ops().head_pool_fc_l2(feat, pooling="gem", p=3.0, eps=1e-6, fc_w=fc_w, fc_b=fc_b, want_f16=True)


@case("head_pool_fc_l2_fused", ["head_pool_fc_l2"], options={"head_fused": 1})
def _(mk):
    return _head_case(mk)


@case("head_pool_fc_l2_phases", ["head_pool_fc_l2"], options={"head_fused": 0})
def _(mk):
    return _head_case(mk)


@case("center_bias", ["center_bias"])
def _(mk):
    x = mk(randn(2, 13, 11, 256, seed=20, dtype=torch.float16))
    return lambda: _ops().center_bias(x, 0.75)


def _forward_cases():
    for pdl in (1, 0):
        @case("net_forward_pdl%d" % pdl, ["net_forward"], options={"pdl": pdl})
        def _(mk):
            net, x = shared_model(), mk(images(2, 96, 128, seed=21))
            return lambda: net(x, want_f16=True)

        @case("net_forward_u8_pdl%d" % pdl, ["net_forward_u8"], options={"pdl": pdl})
        def _(mk):
            net, x = shared_model(), mk(images_u8(2, 112, 80, seed=22))
            return lambda: net.forward_u8(x)

        @case("net_forward_ragged_u8_pdl%d" % pdl, ["net_forward_ragged_u8"], options={"pdl": pdl})
        def _(mk):
            net = shared_model()
            imgs = [mk(images_u8(1, h, w, seed=23 + i)[0]) for i, (h, w) in enumerate([(97, 33), (64, 48), (33, 65)])]
            return lambda: net.forward_ragged_u8(imgs)

        @case("net_forward_ragged_pdl%d" % pdl, ["net_forward_ragged"], options={"pdl": pdl})
        def _(mk):
            net = shared_model()
            imgs = [mk(images(1, h, w, seed=26 + i)[0]) for i, (h, w) in enumerate([(65, 33), (40, 72)])]
            return lambda: net.forward_ragged(imgs)


_forward_cases()


@case("net_debug_stage", ["net_finalize", "net_forward", "net_debug_stage"])
def _(mk):
    net = model()
    net.set_backend_option("debug_taps", 1)
    x = mk(images(1, 64, 64, seed=28))

    def run():
        d = net(x)                                      # the handle is created and finalized here, then used at once
        return d, net.debug_stage("layer1"), net.debug_stage("stem")
    return run


@case("resize_bilinear_u8", ["resize_bilinear_u8"])
def _(mk):
    x = mk(images_u8(2, 77, 51, seed=29))
    return lambda: _ops().resize_bilinear_u8(x, (40, 97))


@case("jpeg_decode", ["jpeg_decoder_decode", "jpeg_debug_coefficients"])
def _(mk):
    from test_jpeg_host import encode, make_image
    files = [encode(make_image(37, 53, "smooth", seed=3), quality=90, subsampling=2, restart_marker_blocks=2),
             encode(make_image(33, 17, "noise", seed=4), quality=100, subsampling=1),
             encode(make_image(40, 24, "smooth", seed=5), gray=True, quality=50),
             encode(make_image(120, 90, "noise", seed=6), quality=95, subsampling=0),
             b"not a jpeg"]
    dec = _ops().JpegDecoder(subseq_bits=64)           # short subsequences: several synchronisation rounds

    def run():
        imgs, ok = dec.decode(files)
        return [im for im, good in zip(imgs, ok) if good], ok, dec.last_rounds, dec.debug_coefficients(1)
    return run


# ------------------------------------------------------------------------------------------------- post-processing
@case("l2_normalize", ["l2_normalize"])
def _(mk):
    x = mk(randn(300, 2048, seed=30))
    return lambda: _ops().l2_normalize(x, want_f16=True)


@case("f32_to_f16", ["f32_to_f16"])
def _(mk):
    x = mk(randn(1001, 33, seed=31))
    return lambda: _ops().f32_to_f16(x)


@case("pool_scales", ["pool_scales"])
def _(mk):
    xs = [mk(randn(50, 2048, seed=32 + i).abs()) for i in range(3)]
    return lambda: (_ops().pool_scales(xs, "gem", 3, l2=True), _ops().pool_scales(xs, "mean", l2=False))


def _whiten_case(mk, n, d, dout, seed):
    x = mk(unit(n, d, seed=seed))
    comp = mk(randn(dout, d, seed=seed + 1, scale=d ** -0.5))
    mean = mk(randn(d, seed=seed + 2, scale=0.01))
    cs = mk(randn(dout, seed=seed + 3).abs() + 0.5)
    return lambda: _ops().whiten(x, comp, mean, cs, l2norm=True, want_f16=True)


@case("whiten_simt", ["whiten"])
def _(mk):
    return _whiten_case(mk, 40, 2048, 512, seed=40)          # N < 64: the SIMT kernel


@case("whiten_tensor_cores", ["whiten"])
def _(mk):
    return _whiten_case(mk, 700, 512, 384, seed=44)          # D % 64 == 0, N >= 64: the wgmma hi/lo kernel


@case("col_sums_f64", ["col_sums_f64"])
def _(mk):
    x = mk(randn(5000, 130, seed=48))
    return lambda: _ops().col_sums_f64(x)


@case("gram_f64", ["gram_f64"])
def _(mk):
    x = mk(randn(3000, 256, seed=49))
    mean = mk(randn(256, seed=50, dtype=torch.float64, scale=0.1))
    return lambda: _ops().gram_f64(x, mean)


def _neighbours(n, nq, k, seed):
    r = np.random.RandomState(seed)
    idx = torch.from_numpy(np.stack([r.choice(n, k, replace=False) for _ in range(nq)]).astype(np.int64)).cuda()
    sc = torch.from_numpy(np.sort(r.uniform(0.1, 0.9, (nq, k)))[:, ::-1].copy()).cuda()
    return idx, sc


@case("aqe_expand", ["aqe_expand"])
def _(mk):
    q, db = mk(unit(12, 256, seed=51)), mk(unit(900, 256, seed=52))
    idx, sc = _neighbours(900, 12, 10, seed=53)
    idx, sc = mk(idx), mk(sc)
    return lambda: _ops().aqe_expand(q, db, idx, sc, 3.0)


@case("aqe_expand_partial", ["aqe_expand"])
def _(mk):
    q, db = mk(unit(12, 256, seed=51)), mk(unit(900, 256, seed=52))
    idx, sc = _neighbours(900, 12, 10, seed=53)
    idx, sc = mk(idx), mk(sc)
    return lambda: _ops().aqe_expand(q, db[300:600], idx, sc, 0.5, partial=True, row_offset=300, n_rows=300)


@case("topk_merge", ["topk_merge"])
def _(mk):
    r = np.random.RandomState(54)
    g, nq, k = 3, 9, 40
    sc = torch.from_numpy(-np.sort(-r.uniform(-1, 1, (g, nq, k)), axis=2)).cuda()
    ix = torch.from_numpy(r.permutation(g * nq * k).reshape(g, nq, k).astype(np.int64)).cuda()
    sc, ix = mk(sc), mk(ix)
    return lambda: _ops().topk_merge(sc, ix, k)


@case("topk_merge_packed", ["topk_merge"])
def _(mk):
    r = np.random.RandomState(55)
    g, nq, k = 4, 5, 30
    sc = torch.from_numpy(-np.sort(-r.uniform(-1, 1, (g, nq, k)), axis=2)).cuda()
    ix = torch.from_numpy(r.permutation(g * nq * k).reshape(g, nq, k).astype(np.int64)).cuda()
    packed = mk(torch.stack([sc.view(torch.int64), ix], 1).contiguous())
    return lambda: _ops().topk_merge_packed(packed, k)


@case("scores_exact", ["scores_exact"])
def _(mk):
    q, db = mk(randn(7, 130, seed=56)), mk(randn(1000, 130, seed=57))
    return lambda: _ops().scores_exact(q, db)


# ------------------------------------------------------------------------------------------ index, search, ranking
def _stats(ix):
    st = ix.stats()
    st.pop("launches")                      # a process-wide counter, not a result
    return st


@case("index_search_k10", ["index_search", "index_last_stats"])
def _(mk):
    ix, q = index(mk, unit(5000, 256, seed=60)), mk(unit(20, 256, seed=61))
    return lambda: (ix.search(q, 10), _stats(ix))


@case("index_search_deep", ["index_search", "index_last_stats"])
def _(mk):
    ix, q = index(mk, unit(6000, 128, seed=62)), mk(unit(5, 128, seed=63))
    return lambda: (ix.search(q, 1500), _stats(ix))


@case("index_search_forced_retry", ["index_search", "index_last_stats"])
def _(mk):
    ix, q = index(mk, unit(20000, 128, seed=64)), mk(unit(8, 128, seed=65))
    ix.set_option("sample_rows", 32)        # a loose seed bound: thousands of candidates per query
    ix.set_option("cand_cap", 1)            # lists of 256: the first filter pass overflows, the retry passes refill them
    ix.set_option("retries", 4)

    def run():
        # the retry threshold is the k-th best of the entries that won the race into the full list, so the counts of
        # candidates and survivors depend on scheduling; the result and the number of retry passes do not
        out = ix.search(q, 50)
        st = _stats(ix)
        return out, {k: st[k] for k in ("dense_rows", "retries")}
    return run


@case("index_deferred_check_overflow", ["index_search", "index_check"])
def _(mk):
    ix, q = index(mk, unit(20000, 128, seed=64)), mk(unit(8, 128, seed=65))
    ix.set_option("sample_rows", 32)
    ix.set_option("cand_cap", 1)
    ix.set_option("retries", 0)             # no retry left: the status block reports the overflow
    ix.set_option("deferred_check", 1)
    from dirb200 import lib

    def run():
        ix.search(q, 50)
        try:
            ix.check()
            return "ok"
        except lib.DirbError as e:
            return e.status
    return run


@case("index_search_begin_finish", ["index_search_begin", "index_search_finish", "index_search_max_queries"])
def _(mk):
    ix, q = index(mk, unit(4000, 192, seed=66)), mk(unit(11, 192, seed=67))

    def run():
        sel = ix.search_begin(q, 30, 30)
        return sel, ix.search_finish(q, 30, sel), ix.search_max_queries(30)
    return run


SHARDS = (1400, 37, 2563)


def _shards(mk, x):
    bounds = np.concatenate([[0], np.cumsum(SHARDS)])
    out = [index(mk, x[a:b].contiguous(), offset=int(a)) for a, b in zip(bounds[:-1], bounds[1:])]
    for sh in out:
        sh.n_global = int(bounds[-1])
    return out


@case("sharded_collective", ["index_search_begin", "index_search_finish", "topk_merge"])
def _(mk):
    from dirb200.dist import shard_quota
    shards, q = _shards(mk, unit(sum(SHARDS), 128, seed=68)), mk(unit(9, 128, seed=69))
    k = 40
    c = shard_quota(k, list(SHARDS))

    def run():
        sels = [sh.search_begin(q, k, c) for sh in shards]
        sel = torch.stack(sels).min(dim=0).values.contiguous()
        outs = [sh.search_finish(q, k, sel) for sh in shards]
        for sh in shards:
            sh.check()
        return _ops().topk_merge(torch.stack([o[0] for o in outs]).contiguous(),
                                 torch.stack([o[1] for o in outs]).contiguous(), k)
    return run


@case("sharded_peer_memory", ["exchange_create", "exchange_open_local", "index_search_sharded_phase",
                              "exchange_close_peers", "index_check"])
def _(mk):
    from dirb200.dist import shard_quota
    shards, q = _shards(mk, unit(sum(SHARDS), 128, seed=68)), mk(unit(9, 128, seed=69))
    k = 40
    c = shard_quota(k, list(SHARDS))
    for sh in shards:
        sh.set_option("deferred_check", 1)
    ops = _ops()

    def run():
        xs = [ops.Exchange(0, len(shards), g, 64, 64) for g in range(len(shards))]   # windows used at once
        ops.Exchange.open_local(xs)
        try:
            for ph in (1, 2, 3):
                for sh, x in zip(shards, xs):
                    sh.search_sharded(x, q, k, c, phase=ph)
            res = [sh.search_sharded(x, q, k, c, phase=4) for sh, x in zip(shards, xs)]
            for sh in shards:
                sh.check()
            return res
        finally:
            torch.cuda.current_stream().synchronize()
            for x in xs:
                x.close_peers()
            for x in xs:
                x.close()
    return run


@case("sharded_world_of_one", ["exchange_create", "index_search_sharded", "index_check"])
def _(mk):
    ix, q = index(mk, unit(3000, 128, seed=70)), mk(unit(6, 128, seed=71))
    ix.set_option("deferred_check", 1)
    ops = _ops()

    def run():
        x = ops.Exchange(0, 1, 0, 16, 64)
        ops.Exchange.open_local([x])
        try:
            out = ix.search_sharded(x, q, 25, 25)
            ix.check()
            return out
        finally:
            torch.cuda.current_stream().synchronize()
            x.close_peers()
            x.close()
    return run


@case("rank_counts", ["index_target_scores", "index_rank_count"])
def _(mk):
    n = 4000
    ix, q = index(mk, unit(n, 128, seed=72)), mk(unit(6, 128, seed=73))
    off, rows, flags = targets(6, n, 9, seed=74)
    return lambda: ix.rank_counts(q, off, rows, flags)


def _count_case(mk, band_cap):
    n, nq = 5000, 5
    db = unit(n, 128, seed=75)
    ix, q = index(mk, db), mk(unit(nq, 128, seed=76))
    ix.set_option("count_eps", 1e-3)        # many pairs within the band: re-scored exactly
    if band_cap is not None:
        ix.set_option("band_cap", band_cap)  # the band overflows: the queries are counted again over all rows
    r = np.random.RandomState(77)
    thr = np.sort(r.uniform(-0.2, 0.3, (nq, 12)))[:, ::-1].reshape(-1).astype(np.float32)
    thr_off = mk(torch.arange(nq + 1, dtype=torch.int32).cuda() * 12)
    thr = mk(torch.from_numpy(thr.copy()).cuda())
    skip = mk(torch.tensor([-1, 3, 17, -1, 4000], dtype=torch.int64).cuda())
    return lambda: (ix.count_ge(q, thr_off, thr, skip), _stats(ix))


@case("count_ge", ["index_count_ge", "index_last_stats"])
def _(mk):
    return _count_case(mk, None)


@case("count_ge_band_recount", ["index_count_ge", "index_last_stats"])
def _(mk):
    return _count_case(mk, 4)


def _join_stats(ix):
    st = ix.join_stats()
    return {k: v for k, v in st.items() if not k.endswith("_ms")}


@case("range_search", ["index_range_search", "index_join_fetch", "index_join_stats"])
def _(mk):
    ix, q = index(mk, unit(3000, 64, seed=78)), mk(unit(7, 64, seed=79))
    return lambda: (ix.range_search(q, 0.25), _join_stats(ix))


@case("self_join", ["index_self_join", "index_join_fetch", "index_join_stats"])
def _(mk):
    ix = index(mk, clustered(1500, 64, seed=80))
    ix.set_option("join_cap", 1)            # every list overflows: re-run at the exact count
    return lambda: (ix.self_join(0.5, row_block=512), _join_stats(ix))


@case("join_components_and_groups", ["join_components", "join_groups"])
def _(mk):
    r = np.random.RandomState(81)
    n = 700
    a, b = r.randint(n, size=500), r.randint(n, size=500)
    src, dst = np.concatenate([a, b]), np.concatenate([b, a])
    order = np.argsort(src, kind="stable")
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=off[1:])
    off, cols = mk(torch.from_numpy(off).cuda()), mk(torch.from_numpy(dst[order].astype(np.int64)).cuda())
    ops = _ops()

    def run():
        labels = ops.join_components(off, cols, n)
        return labels, ops.join_groups(labels)
    return run


@case("nearest", ["index_nearest", "index_nearest_stats"])
def _(mk):
    ix, q = index(mk, unit(3000, 128, seed=82)), mk(unit(500, 128, seed=83))
    return lambda: (ix.nearest(q), ix.nearest_stats())


def _allow_case(mk, per_query):
    ops = _ops()
    n, nq = 5000, 7
    ix, q = index(mk, unit(n, 128, seed=84)), mk(unit(nq, 128, seed=85))
    r = np.random.RandomState(86)
    mask = torch.from_numpy(r.rand(nq, n) < 0.3 if per_query else r.rand(n) < 0.2).cuda()
    words = mk(ops.allow_rows(mask))
    return lambda: (ix.search(q, 20, allow=words), _stats(ix))


@case("filtered_search_shared", ["index_set_allow", "index_search"])
def _(mk):
    return _allow_case(mk, False)


@case("filtered_search_per_query", ["index_set_allow", "index_search"])
def _(mk):
    return _allow_case(mk, True)


@case("allow_exclude", ["allow_exclude"])
def _(mk):
    ops = _ops()
    n = 3000
    base = mk(ops.allow_rows(torch.from_numpy(np.random.RandomState(87).rand(n) < 0.7).cuda()))
    rows = [[0, 5, 2999], [], [31, 32, 33, 64], [1000]]
    return lambda: ops.allow_exclude(base, len(rows), rows)


# ---------------------------------------------------------------------------------- approximate and iterative indexes
def _kmeans_result(km):
    return (km.cluster_centers_, km.labels_, km.scores_, km.n_iter_, km.objective_, km.stats_)


@case("kmeans_fit_relocate", ["kmeans_stats", "kmeans_relocate", "kmeans_update", "index_nearest",
                              "index_nearest_stats"])
def _(mk):
    from dirb200.cluster import SphericalKMeans
    x = clustered(3000, 128, centres=8, seed=88)
    init = x[:12].clone()
    init[11] = -x.mean(0) / x.mean(0).norm()            # no row is nearest to it: the first update relocates into it
    x, init = mk(x), mk(init)
    return lambda: _kmeans_result(SphericalKMeans(12, init=init, max_iter=6).fit(x))


@case("kmeans_fit_pp", ["kmeans_pp", "kmeans_stats", "kmeans_update"])
def _(mk):
    from dirb200.cluster import SphericalKMeans
    x = mk(clustered(2000, 64, centres=6, seed=89))
    return lambda: _kmeans_result(SphericalKMeans(10, init="k-means++", max_iter=4, seed=3).fit(x))


def _centres(x, k, seed):
    return x[torch.from_numpy(np.random.RandomState(seed).choice(x.shape[0], k, replace=False)).cuda()].contiguous()


@case("ivf", ["index_set_lists", "index_search_lists", "index_lists_stats"])
def _(mk):
    from dirb200.ivf import IVFIndex
    x = clustered(4000, 128, seed=90)
    c = _centres(x, 16, seed=91)
    x, c, q = mk(x), mk(c), mk(clustered(9, 128, seed=92))

    def run():
        ivf = IVFIndex(x, c)
        out = ivf.search(q, 20, 3)
        st = {k: v for k, v in ivf.stats().items() if not k.endswith("_ms")}
        return out, st, ivf.labels_, ivf.perm_
    return run


def _ivfpq_case(mk, rows):
    from dirb200.ivfpq import IVFPQIndex
    x = clustered(3000, 128, seed=93)
    c = _centres(x, 8, seed=94)
    x, c, q = mk(x), mk(c), mk(clustered(7, 128, seed=95))

    def run():
        pq = IVFPQIndex(x, c, 16, train_size=1000, pq_iter=3, rows=rows, chunk_rows=1024)
        out = pq.search(q, 15, 3)
        return out, pq.stats(), pq.codes_, pq.codebooks_, pq.empty_codewords_
    return run


@case("ivfpq_device_rows", ["pq_assign", "pq_update", "pq_tables", "pq_search"])
def _(mk):
    return _ivfpq_case(mk, "device")


@case("ivfpq_host_rows", ["pq_assign", "pq_update", "pq_tables", "pq_search"])
def _(mk):
    return _ivfpq_case(mk, "host")


@case("graph", ["graph_prune", "graph_merge", "graph_search", "join_components"])
def _(mk):
    from dirb200.graph import GraphIndex
    x, q = mk(clustered(2500, 128, seed=96)), mk(clustered(8, 128, seed=97))

    def run():
        g = GraphIndex(x, degree=16, build_k=32, n_entry=256)
        out = g.search(q, 10, itopk=64, max_iter=32)
        return out, g.graph_, g.n_components_, g.stats()
    return run


@case("diffusion", ["diffusion_graph", "diffusion_seeds", "diffusion_solve", "diffusion_topk",
                    "diffusion_rank_count"])
def _(mk):
    from dirb200.diffusion import Diffusion
    n = 1500
    x, q = mk(clustered(n, 128, seed=98)), mk(clustered(6, 128, seed=99))
    off, rows, flags = targets(6, n, 5, seed=100)

    def run():
        d = Diffusion(x, k=20)
        return d.search(q, 30, kq=5, iters=15), d.rank_counts(q, off, rows, flags, kq=5, iters=15), d.graph
    return run


@case("diffusion_truncated", ["diffusion_graph_weights", "diffusion_trunc_build", "diffusion_trunc_solve",
                              "diffusion_trunc_topk", "diffusion_trunc_rank_count"])
def _(mk):
    from dirb200.diffusion import Diffusion
    n = 1500
    x, q = mk(clustered(n, 128, seed=101)), mk(clustered(6, 128, seed=102))
    off, rows, flags = targets(6, n, 5, seed=103)

    def run():
        d = Diffusion(x, k=20, truncation=True)
        return (d.search(q, 30, kq=5, iters=15, truncate=200),
                d.rank_counts_truncated(q, off, rows, flags, 200, kq=5, iters=15), d.weights)
    return run


# ---------------------------------------------------------------------------------------------------------- AP loss
@case("aploss", ["aploss_forward", "aploss_backward"])
def _(mk):
    from dirb200.loss import quantizer_table
    nq = 20
    r = np.random.RandomState(104)
    x = mk(torch.from_numpy(r.uniform(-1, 1, (6, 300)).astype(np.float32)).cuda())
    lab = mk(torch.from_numpy((r.rand(6, 300) < 0.1).astype(np.uint8)).cuda())
    table = mk(quantizer_table(nq, -1, 1).cuda())
    g = mk(torch.from_numpy(r.standard_normal(6).astype(np.float32)).cuda())
    ops = _ops()

    def run():
        h, G, ap = ops.aploss_forward(x, lab, nq, table, "tap")
        return h, G, ap, ops.aploss_backward(x, lab, nq, table, G, g)
    return run
