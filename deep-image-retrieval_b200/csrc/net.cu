// ResNet-50/101 + GeM + FC + L2 descriptor network on one GPU: weight packing and the launch schedule.
//
// Reference: dirtorch/nets/backbones/resnet.py:46-87 (Bottleneck), :102-168 (ResNet.__init__/forward),
//            dirtorch/nets/rmac_resnet.py:12-69 (head), dirtorch/nets/layers/pooling.py:38-54 (GeM).
// Data layout in HBM: activations NHWC fp16; conv weights [Cout][KH][KW][Cin] fp16 (K-major rows, the B operand
// of the implicit GEMM); BatchNorm folded to per-channel fp32 (scale, shift) applied in the conv epilogue together
// with the residual add and ReLU; head weights fp32.  A batch is processed in chunks of `chunk` images so that
// the activations of consecutive layers stay L2-resident.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "conv.h"

using namespace dirb;

namespace {

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
};

struct ConvLayer {
  std::string conv, bn;          // state-dict prefixes
  int Cin, Cout, K, stride, pad;
  int CinPad, Kpad;              // packed layout
  __half* w = nullptr;
  float* scale = nullptr;
  float* shift = nullptr;
};

struct Block {
  ConvLayer c1, c2, c3, down;
  bool has_down = false;
  // block 0 of a layer: conv3 + projection shortcut as ONE GEMM over K = [conv2 output | block input]:
  // wcat[o] = [scale3[o] * W3[o][:], scale_d[o] * Wd[o][:]] (fp16), shift = shift3 + shift_d, scale = 1.
  __half* wcat = nullptr;
  float* cat_shift = nullptr;
  float* ones = nullptr;
};

}  // namespace

// Per-launch CUDA-event timing of one forward (option "profile"): class 0 = wgmma conv, 1 = stem conv (mma.sync),
// 2 = layout/maxpool, 3 = head.  Events sit on the launch stream, so they time exactly the kernels between them.
struct Profiler {
  struct Rec { cudaEvent_t a, b; int cls; double flops, bytes; std::string tag; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  cudaEvent_t get() {
    if (used == pool.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      pool.push_back(e);
    }
    return pool[used++];
  }
  void reset() { recs.clear(); used = 0; }
  ~Profiler() { for (auto e : pool) cudaEventDestroy(e); }
};

struct dirb200_net {
  int device = 0;
  std::string arch;
  std::vector<int> nblocks;
  // options
  int pooling = 0, norm_features = 0, without_fc = 0, out_dim = 2048, chunk = 0, conv_impl = 0;
  float gem_p = 3.0f, gem_eps = 1e-6f;
  float center_bias = 0.0f;       // rmac_resnet.py:52-56
  // host state dict
  std::map<std::string, HostTensor> sd;
  bool finalized = false;
  // device weights
  ConvLayer stem;
  __half* stem_w2 = nullptr;      // [64][256] space-to-depth tap layout of the stem
  std::vector<Block> blocks;      // flattened over layer1..4
  std::vector<int> layer_end;     // index (exclusive) of the last block of each layer
  float* fc_w = nullptr;
  float* fc_b = nullptr;
  unsigned int* head_bar = nullptr;   // grid-barrier words of the fused head kernel (zero once, self-resetting)
  std::vector<void*> owned;
  // workspace
  void* ws = nullptr;
  size_t ws_bytes = 0;
  // staging for forward_host
  float* h2d = nullptr;
  size_t h2d_bytes = 0;
  float* d_desc = nullptr;
  size_t d_desc_bytes = 0;
  cudaStream_t own_stream = nullptr;
  // debug taps of the last chunk (copies, only when the "debug_taps" option is set)
  struct Tap { __half* ptr; size_t cap; int n, h, w, c; };
  std::map<std::string, Tap> taps;
  int debug_taps = 0;
  int64_t last_launches = 0;
  double last_flops = 0;
  int profile = 0;
  Profiler prof;
  float mean_std[6] = {0.485f, 0.456f, 0.406f, 0.229f, 0.224f, 0.225f};   // preprocess of resnet.py:110-111
  int fuse_ds = 1;                // fuse the projection shortcut into conv3 of block 0 (wgmma path only)
  int fuse_stem = 1;              // stem conv + maxpool as one kernel reading the images (conv_impl 0 / 2)
  int fuse_c23 = 0;               // conv2 + conv3 (+ residual) of the identity blocks as one kernel (conv_c23.cuh):
                                  // 0 off, 1 where every SM gets several tiles, 2 wherever the kernel supports the shape
  // trunk / head variants (rmac_resnet.py:74-88, rmac_resnet_fpn.py:92-110)
  bool basic = false;             // BasicBlock trunk (resnet18): two 3x3 convolutions per block, expansion 1
  int expansion = 4;
  int stage_ch[5] = {64, 256, 512, 1024, 2048};   // channels of the output of stage 0..4
  int fpn = 0;                    // FPN head: GeM of layer3 (after the lateral merge in mode 1) and of layer4, concatenated
  int fpn_mode = 1;               // rmac_resnet_fpn.py:27-30,55-62: 1 = lateral 1x1 + upsample-add + 3x3 smoothing, 0 = none
  float gem_p4 = 3.0f;            // adpoolc4.p (layer3 map); gem_p holds adpoolx5.p (layer4 map) for FPN heads
  ConvLayer fpn_lat, fpn_smooth;  // conv1x5 (1x1, C4 -> C3), conv3c4 (3x3, C3 -> C3): no BN, ReLU after each
  int feat_in() const { return fpn ? stage_ch[3] + stage_ch[4] : stage_ch[4]; }     // fc.in_features
  int desc_dim() const { return without_fc ? feat_in() : out_dim; }
  // ragged entry points: device copy of the extent table (see RG_LD)
  int* ext_dev = nullptr;
  size_t ext_bytes = 0;
  // pipelined host entry point
  cudaStream_t copy_stream = nullptr;
  std::vector<cudaEvent_t> pipe_events;
  int host_chunk = 16;
};

struct ProfScope {
  dirb200_net* n; cudaStream_t st; bool on;
  ProfScope(dirb200_net* n_, cudaStream_t st_, int cls, double flops, double bytes, const std::string& tag = std::string())
      : n(n_), st(st_), on(n_->profile != 0) {
    if (on) {
      Profiler::Rec r{n->prof.get(), n->prof.get(), cls, flops, bytes, tag};
      cudaEventRecord(r.a, st);
      n->prof.recs.push_back(r);
    }
  }
  ~ProfScope() { if (on) cudaEventRecord(n->prof.recs.back().b, st); }
};

static int dev_alloc(dirb200_net* n, void** p, size_t bytes) {
  DIRB_CUDA(cudaMalloc(p, bytes));
  n->owned.push_back(*p);
  return 0;
}

// keep a copy of an intermediate activation (the rotating buffers are overwritten by later layers)
static int record_tap(dirb200_net* n, const std::string& name, const __half* src, int nb, int h, int w, int c,
                      cudaStream_t stream) {
  if (!n->debug_taps) return 0;
  const size_t bytes = static_cast<size_t>(nb) * h * w * c * 2;
  auto& t = n->taps[name];
  DIRB_TRY(grow_device(reinterpret_cast<void**>(&t.ptr), &t.cap, bytes));
  t.n = nb; t.h = h; t.w = w; t.c = c;
  DIRB_CUDA(cudaMemcpyAsync(t.ptr, src, bytes, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

static int get_tensor(dirb200_net* n, const std::string& name, const HostTensor** out, size_t expect) {
  auto it = n->sd.find(name);
  DIRB_REQUIRE(it != n->sd.end(), DIRB200_EKEY, "missing state-dict tensor '%s'", name.c_str());
  DIRB_REQUIRE(it->second.data.size() == expect, DIRB200_EINVAL, "tensor '%s' has %zu elements, expected %zu",
               name.c_str(), it->second.data.size(), expect);
  *out = &it->second;
  return 0;
}

// OIHW fp32 -> [Cout][KH][KW][CinPad] fp16 rows padded to Kpad; BN -> (scale, shift), also returned through
// sc_host / sh_host when given.  An empty BN prefix (the FPN convolutions) means scale 1, shift 0.
static int pack_conv(dirb200_net* n, ConvLayer& L, std::vector<float>* sc_host = nullptr,
                     std::vector<float>* sh_host = nullptr) {
  const HostTensor* w;
  const size_t kk = static_cast<size_t>(L.K) * L.K;
  DIRB_TRY(get_tensor(n, L.conv + ".weight", &w, static_cast<size_t>(L.Cout) * L.Cin * kk));
  std::vector<float> sc(L.Cout, 1.0f), sh(L.Cout, 0.0f);
  if (!L.bn.empty()) {
    const HostTensor *g, *b, *m, *v;
    DIRB_TRY(get_tensor(n, L.bn + ".weight", &g, L.Cout));
    DIRB_TRY(get_tensor(n, L.bn + ".bias", &b, L.Cout));
    DIRB_TRY(get_tensor(n, L.bn + ".running_mean", &m, L.Cout));
    DIRB_TRY(get_tensor(n, L.bn + ".running_var", &v, L.Cout));
    for (int o = 0; o < L.Cout; ++o) {
      // BatchNorm2d eval: y = (x - mean) / sqrt(var + 1e-5) * gamma + beta   (eps: torch default, resnet.py:57)
      const float s = g->data[o] / sqrtf(v->data[o] + 1e-5f);
      sc[o] = s;
      sh[o] = b->data[o] - m->data[o] * s;
    }
  }
  L.CinPad = (L.Cin % 8 == 0) ? L.Cin : ((L.Cin + 7) / 8 * 8);
  const int Ktot = L.K * L.K * L.CinPad;
  L.Kpad = (Ktot + 31) / 32 * 32;
  std::vector<__half> hw(static_cast<size_t>(L.Cout) * L.Kpad, __float2half(0.f));
  for (int o = 0; o < L.Cout; ++o)
    for (int c = 0; c < L.Cin; ++c)
      for (int kh = 0; kh < L.K; ++kh)
        for (int kw = 0; kw < L.K; ++kw)
          hw[static_cast<size_t>(o) * L.Kpad + (static_cast<size_t>(kh) * L.K + kw) * L.CinPad + c] =
              __float2half_rn(w->data[((static_cast<size_t>(o) * L.Cin + c) * L.K + kh) * L.K + kw]);
  DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&L.w), hw.size() * sizeof(__half)));
  DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&L.scale), L.Cout * sizeof(float)));
  DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&L.shift), L.Cout * sizeof(float)));
  DIRB_CUDA(cudaMemcpy(L.w, hw.data(), hw.size() * sizeof(__half), cudaMemcpyHostToDevice));
  DIRB_CUDA(cudaMemcpy(L.scale, sc.data(), L.Cout * sizeof(float), cudaMemcpyHostToDevice));
  DIRB_CUDA(cudaMemcpy(L.shift, sh.data(), L.Cout * sizeof(float), cudaMemcpyHostToDevice));
  if (sc_host) *sc_host = std::move(sc);
  if (sh_host) *sh_host = std::move(sh);
  return 0;
}

static ConvLayer make_layer(const std::string& conv, const std::string& bn, int cin, int cout, int k, int stride,
                            int pad) {
  ConvLayer L;
  L.conv = conv; L.bn = bn; L.Cin = cin; L.Cout = cout; L.K = k; L.stride = stride; L.pad = pad;
  L.CinPad = cin; L.Kpad = 0;
  return L;
}

static int run_conv(dirb200_net* n, const ConvLayer& L, const __half* in, int B, int H, int W, const __half* res,
                    int relu, __half* out, cudaStream_t stream, int force_mma = 0, const ConvExt* ext = nullptr) {
  ConvShape s{B, H, W, L.CinPad, L.Cout, L.K, L.K, L.stride, L.pad};
  const double flops = 2.0 * B * s.Ho() * s.Wo() * static_cast<double>(L.Cout) * L.K * L.K * L.Cin;
  // algorithmic bytes: input + output (+ residual) activations once, weights once
  const double bytes = 2.0 * (static_cast<double>(B) * H * W * L.CinPad + static_cast<double>(B) * s.Ho() * s.Wo() * L.Cout * (res ? 2 : 1) +
                              static_cast<double>(L.Cout) * L.K * L.K * L.CinPad);
  n->last_flops += flops;
  const bool mma = force_mma || n->conv_impl == 1 || L.CinPad % 64 != 0;
  std::string tag;
  if (n->profile) {
    char buf[96];
    snprintf(buf, sizeof(buf), "%dx%d%s %d->%d%s @%dx%d", L.K, L.K, L.stride == 2 ? "/s2" : "", L.Cin, L.Cout, res ? " +res" : "", s.Ho(), s.Wo());
    tag = buf;
  }
  ProfScope ps(n, stream, mma ? 1 : 0, flops, bytes, tag);
  DIRB_REQUIRE(!(mma && ext), DIRB200_ENOTSUP, "ragged batches need the wgmma convolutions (conv_impl 0 or 2)");
  if (mma)
    return conv_mma(s, in, L.w, L.Kpad, L.scale, L.shift, res, relu, out, stream);
  if (n->conv_impl == 2) return conv_tc_np(s, in, L.w, L.scale, L.shift, res, relu, out, stream, ext);
  return conv_tc(s, in, L.w, L.scale, L.shift, res, relu, out, stream, ext);
}

extern "C" {

int dirb200_net_create(const char* arch, int device, dirb200_net** out) {
  DIRB_REQUIRE(arch && out, DIRB200_EINVAL, "null argument");
  DIRB_TRY(dirb200_device_check(device));
  auto* n = new dirb200_net();
  n->device = device;
  n->arch = arch;
  // "<trunk>_rmac" (rmac_resnet.py:74-88), "<trunk>_fpn_rmac" / "resnet101_fpn0_rmac" (rmac_resnet_fpn.py:92-110)
  std::string trunk = n->arch;
  const char* suffixes[3] = {"_fpn0_rmac", "_fpn_rmac", "_rmac"};
  int which = -1;
  for (int i = 0; i < 3 && which < 0; ++i) {
    const std::string suf(suffixes[i]);
    if (trunk.size() > suf.size() && trunk.compare(trunk.size() - suf.size(), suf.size(), suf) == 0) {
      trunk = trunk.substr(0, trunk.size() - suf.size());
      which = i;
    }
  }
  n->fpn = (which == 0 || which == 1) ? 1 : 0;
  n->fpn_mode = (which == 0) ? 0 : 1;
  if (trunk == "resnet18") { n->nblocks = {2, 2, 2, 2}; n->basic = true; }        // rmac_resnet.py:76
  else if (trunk == "resnet50") n->nblocks = {3, 4, 6, 3};                         // rmac_resnet.py:80
  else if (trunk == "resnet101") n->nblocks = {3, 4, 23, 3};                       // rmac_resnet.py:84
  else if (trunk == "resnet152") n->nblocks = {3, 8, 36, 3};                       // rmac_resnet.py:88
  const bool known = which >= 0 && !n->nblocks.empty() && !(which == 0 && trunk != "resnet101");
  if (!known) {
    delete n;
    DIRB_REQUIRE(false, DIRB200_ENOTSUP,
                 "unknown model architecture '%s' (supported: resnet{18,50,101,152}_rmac, resnet{18,50,101,152}_fpn_rmac, "
                 "resnet101_fpn0_rmac)", arch);
  }
  n->expansion = n->basic ? 1 : 4;
  for (int s = 1; s < 5; ++s) n->stage_ch[s] = (64 << (s - 1)) * n->expansion;
  *out = n;
  return 0;
}

static bool is_global_option(const std::string& k) {
  return k == "halo" || k == "pdl" || k == "head_fused";
}

int dirb200_set_global_option(const char* key, double value) {
  DIRB_REQUIRE(key, DIRB200_EINVAL, "null argument");
  const std::string k(key);
  if (k == "halo") set_conv_halo(value != 0);
  else if (k == "pdl") g_use_pdl = value != 0;
  else if (k == "head_fused") set_head_fused(static_cast<int>(value));
  else DIRB_REQUIRE(false, DIRB200_EKEY, "unknown global option '%s'", key);
  return 0;
}

int dirb200_get_global_option(const char* key, double* value) {
  DIRB_REQUIRE(key && value, DIRB200_EINVAL, "null argument");
  const std::string k(key);
  if (k == "halo") *value = get_conv_halo();
  else if (k == "pdl") *value = g_use_pdl;
  else if (k == "head_fused") *value = get_head_fused();
  else DIRB_REQUIRE(false, DIRB200_EKEY, "unknown global option '%s'", key);
  return 0;
}

int dirb200_net_set_option(dirb200_net* n, const char* key, double value) {
  DIRB_REQUIRE(n && key, DIRB200_EINVAL, "null argument");
  const std::string k(key);
  // options that decide which tensors dirb200_net_finalize reads / packs cannot change afterwards
  const bool structural = (k == "pooling" || k == "without_fc" || k == "out_dim" || k == "fpn_mode");
  DIRB_REQUIRE(!(structural && n->finalized), DIRB200_ESTATE, "option '%s' must be set before dirb200_net_finalize", key);
  if (k == "pooling") n->pooling = static_cast<int>(value);
  else if (k == "norm_features") n->norm_features = value != 0;
  else if (k == "without_fc") n->without_fc = value != 0;
  else if (k == "out_dim") n->out_dim = static_cast<int>(value);
  else if (k == "fpn_mode") {
    DIRB_REQUIRE(n->fpn && (value == 0 || value == 1), DIRB200_EINVAL, "fpn_mode is 0 or 1 and only applies to *_fpn_rmac networks");
    n->fpn_mode = static_cast<int>(value);
  }
  else if (k == "chunk") n->chunk = static_cast<int>(value);
  else if (k == "conv_impl") n->conv_impl = static_cast<int>(value);
  else if (k == "gem_eps") n->gem_eps = static_cast<float>(value);
  else if (k == "center_bias") n->center_bias = static_cast<float>(value);
  else if (k == "debug_taps") n->debug_taps = value != 0;
  else if (k == "profile") {             // 1 = time every launch of the NEXT forward; 2 = accumulate over forwards
    n->profile = static_cast<int>(value);
    n->prof.reset();
  }
  else if (k == "fuse_ds") n->fuse_ds = value != 0;
  else if (k == "fuse_c23") n->fuse_c23 = static_cast<int>(value);
  else if (k == "fuse_stem") n->fuse_stem = value != 0;
  else if (is_global_option(k)) return dirb200_set_global_option(key, value);   // process-wide kernel selectors
  else if (k.size() == 5 && k.compare(0, 4, "mean") == 0 && k[4] >= '0' && k[4] <= '2') n->mean_std[k[4] - '0'] = static_cast<float>(value);
  else if (k.size() == 4 && k.compare(0, 3, "std") == 0 && k[3] >= '0' && k[3] <= '2') n->mean_std[3 + k[3] - '0'] = static_cast<float>(value);
  else if (k == "host_chunk") n->host_chunk = std::max(1, static_cast<int>(value));
  else DIRB_REQUIRE(false, DIRB200_EKEY, "unknown net option '%s'", key);
  return 0;
}

int dirb200_net_set_tensor(dirb200_net* n, const char* name, const float* host_data, const int64_t* shape, int ndim) {
  DIRB_REQUIRE(n && name && (host_data || ndim == 0) && ndim >= 0 && ndim <= 4, DIRB200_EINVAL, "bad tensor argument");
  DIRB_REQUIRE(!n->finalized, DIRB200_ESTATE, "network already finalized");
  std::string key(name);
  if (key.rfind("module.", 0) == 0) key = key.substr(7);  // DataParallel prefix, common.py:128-133
  const char* nbt = "num_batches_tracked";
  if (key.size() >= strlen(nbt) && key.compare(key.size() - strlen(nbt), strlen(nbt), nbt) == 0) return 0;
  HostTensor t;
  size_t numel = 1;
  for (int i = 0; i < ndim; ++i) {
    t.shape.push_back(shape[i]);
    numel *= static_cast<size_t>(shape[i]);
  }
  t.data.assign(host_data, host_data + numel);
  n->sd[key] = std::move(t);
  return 0;
}

int dirb200_net_finalize(dirb200_net* n) {
  DIRB_REQUIRE(n, DIRB200_EINVAL, "null");
  DIRB_REQUIRE(!n->finalized, DIRB200_ESTATE, "network already finalized");
  DIRB_CUDA(cudaSetDevice(n->device));
  n->stem = make_layer("conv1", "bn1", 3, 64, 7, 2, 3);          // resnet.py:115-117
  DIRB_TRY(pack_conv(n, n->stem));
  {
    const HostTensor* w;
    DIRB_TRY(get_tensor(n, "conv1.weight", &w, 64 * 3 * 7 * 7));
    std::vector<__half> w2(64 * 256);
    pack_stem_w2(w->data.data(), w2.data());
    DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&n->stem_w2), w2.size() * sizeof(__half)));
    DIRB_CUDA(cudaMemcpy(n->stem_w2, w2.data(), w2.size() * sizeof(__half), cudaMemcpyHostToDevice));
  }
  int inplanes = 64;
  const int planes_per_layer[4] = {64, 128, 256, 512};           // resnet.py:120-123
  for (int li = 0; li < 4; ++li) {
    const int planes = planes_per_layer[li];
    for (int b = 0; b < n->nblocks[li]; ++b) {
      const std::string p = "layer" + std::to_string(li + 1) + "." + std::to_string(b) + ".";
      const int stride = (li > 0 && b == 0) ? 2 : 1;
      Block blk;
      const int cout = planes * n->expansion;
      if (n->basic) {                                                              // resnet.py:15-44
        blk.c1 = make_layer(p + "conv1", p + "bn1", inplanes, planes, 3, stride, 1);
        blk.c2 = make_layer(p + "conv2", p + "bn2", planes, planes, 3, 1, 1);
        blk.has_down = (b == 0) && (stride != 1 || inplanes != cout);              // resnet.py:136-141
        DIRB_TRY(pack_conv(n, blk.c1));
        DIRB_TRY(pack_conv(n, blk.c2));
        if (blk.has_down) {
          blk.down = make_layer(p + "downsample.0", p + "downsample.1", inplanes, cout, 1, stride, 0);
          DIRB_TRY(pack_conv(n, blk.down));
        }
        n->blocks.push_back(blk);
        inplanes = cout;
        continue;
      }
      blk.c1 = make_layer(p + "conv1", p + "bn1", inplanes, planes, 1, 1, 0);
      blk.c2 = make_layer(p + "conv2", p + "bn2", planes, planes, 3, stride, 1);     // stride on conv2, resnet.py:58
      blk.c3 = make_layer(p + "conv3", p + "bn3", planes, planes * 4, 1, 1, 0);
      blk.has_down = (b == 0);                                                     // resnet.py:136-141
      std::vector<float> s3, sh3;
      DIRB_TRY(pack_conv(n, blk.c1));
      DIRB_TRY(pack_conv(n, blk.c2));
      DIRB_TRY(pack_conv(n, blk.c3, &s3, &sh3));
      if (blk.has_down) {
        blk.down = make_layer(p + "downsample.0", p + "downsample.1", inplanes, planes * 4, 1, stride, 0);
        std::vector<float> sd, shd;
        DIRB_TRY(pack_conv(n, blk.down, &sd, &shd));
        // K-concatenated, BN-scaled weights for the fused conv3 + shortcut
        const HostTensor *w3, *wd;
        const int kcat = planes + inplanes;
        DIRB_TRY(get_tensor(n, p + "conv3.weight", &w3, static_cast<size_t>(cout) * planes));
        DIRB_TRY(get_tensor(n, p + "downsample.0.weight", &wd, static_cast<size_t>(cout) * inplanes));
        std::vector<__half> wc(static_cast<size_t>(cout) * kcat);
        std::vector<float> shc(cout), one(cout, 1.0f);
        for (int o = 0; o < cout; ++o) {
          for (int c = 0; c < planes; ++c) wc[static_cast<size_t>(o) * kcat + c] = __float2half_rn(s3[o] * w3->data[static_cast<size_t>(o) * planes + c]);
          for (int c = 0; c < inplanes; ++c) wc[static_cast<size_t>(o) * kcat + planes + c] = __float2half_rn(sd[o] * wd->data[static_cast<size_t>(o) * inplanes + c]);
          shc[o] = sh3[o] + shd[o];
        }
        DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&blk.wcat), wc.size() * sizeof(__half)));
        DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&blk.cat_shift), cout * 4));
        DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&blk.ones), cout * 4));
        DIRB_CUDA(cudaMemcpy(blk.wcat, wc.data(), wc.size() * sizeof(__half), cudaMemcpyHostToDevice));
        DIRB_CUDA(cudaMemcpy(blk.cat_shift, shc.data(), cout * 4, cudaMemcpyHostToDevice));
        DIRB_CUDA(cudaMemcpy(blk.ones, one.data(), cout * 4, cudaMemcpyHostToDevice));
      }
      n->blocks.push_back(blk);
      inplanes = planes * 4;
    }
    n->layer_end.push_back(static_cast<int>(n->blocks.size()));
  }
  if (n->fpn) {
    // rmac_resnet_fpn.py:36-43: only the 'gem' branch creates the two pooling layers forward() uses
    DIRB_REQUIRE(n->pooling == 0, DIRB200_ENOTSUP, "FPN heads support pooling='gem' only (rmac_resnet_fpn.py:36-43,76-77)");
    const HostTensor *p5, *p4;
    DIRB_TRY(get_tensor(n, "adpoolx5.p", &p5, 1));
    DIRB_TRY(get_tensor(n, "adpoolc4.p", &p4, 1));
    n->gem_p = p5->data[0];
    n->gem_p4 = p4->data[0];
    DIRB_REQUIRE(n->gem_p > 0 && n->gem_p4 > 0, DIRB200_EINVAL, "GeM p must be positive");
    if (n->fpn_mode == 1) {                                                       // rmac_resnet_fpn.py:27-30
      n->fpn_lat = make_layer("conv1x5", "", n->stage_ch[4], n->stage_ch[3], 1, 1, 0);
      n->fpn_smooth = make_layer("conv3c4", "", n->stage_ch[3], n->stage_ch[3], 3, 1, 1);
      DIRB_TRY(pack_conv(n, n->fpn_lat));
      DIRB_TRY(pack_conv(n, n->fpn_smooth));
    }
  } else if (n->pooling == 0) {
    const HostTensor* p;
    DIRB_TRY(get_tensor(n, "adpool.p", &p, 1));                  // pooling.py:54
    n->gem_p = p->data[0];
    DIRB_REQUIRE(n->gem_p > 0, DIRB200_EINVAL, "GeM p must be positive");
  }
  if (!n->without_fc) {
    const HostTensor *w, *b;
    DIRB_TRY(get_tensor(n, "fc.weight", &w, static_cast<size_t>(n->out_dim) * n->feat_in()));   // rmac_resnet.py:34, rmac_resnet_fpn.py:46
    DIRB_TRY(get_tensor(n, "fc.bias", &b, n->out_dim));
    DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&n->fc_w), w->data.size() * 4));
    DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&n->fc_b), b->data.size() * 4));
    DIRB_CUDA(cudaMemcpy(n->fc_w, w->data.data(), w->data.size() * 4, cudaMemcpyHostToDevice));
    DIRB_CUDA(cudaMemcpy(n->fc_b, b->data.data(), b->data.size() * 4, cudaMemcpyHostToDevice));
  }
  DIRB_TRY(dev_alloc(n, reinterpret_cast<void**>(&n->head_bar), 128));
  DIRB_CUDA(cudaMemset(n->head_bar, 0, 128));
  // The memset and the pageable copies above run on the legacy stream and may still be in flight when they return;
  // a forward on a non-blocking stream is not ordered after them.  Finish them before the network is usable.
  DIRB_CUDA(cudaStreamSynchronize(cudaStreamLegacy));
  n->sd.clear();
  n->finalized = true;
  return 0;
}

static int auto_chunk(int B, int H, int W) {
  // Large chunks keep every launch at many tiles per SM (the persistent kernels lose ~1/waves to the tail);
  // bound the activation workspace to ~24 GB of the 80 GB HBM.
  const double per_img = 2.0 * (static_cast<double>(H) * W * 8 + (H / 2.0) * (W / 2.0) * 64 + 5.0 * (H / 4.0) * (W / 4.0) * 256);
  int c = static_cast<int>(24e9 / per_img);
  if (c < 1) c = 1;
  if (c > 64) c = 64;
  if (c > B) c = B;
  return c;
}

// Resolution levels of the network: 0 = input, 1 = stem convolution output, 2 + s = output of stage s (0 maxpool,
// 1..4 layer1..4).  The workspace, the launch schedule and the extent table of ragged batches all take their sizes
// from level_sizes, which is what makes a ragged batch bit-identical to B = 1 forwards.
constexpr int RG_LEVELS = 7, RG_LD = 4 * RG_LEVELS;

namespace {
struct LevelSizes {
  int h[RG_LEVELS], w[RG_LEVELS];
};

// Activation buffers of one pass of the network over up to `chunk` images; every stage runs over the whole pass.
struct Workspace {
  __half* stem_ws;        // s2d / nhwc8 staging of the stem input (unfused stem only, else null)
  __half* stem_out;       // stem conv output (before the maxpool; unfused stem or debug taps only, else null)
  __half* stage_out[4];   // outputs of stage 0..3
  __half* scratch[4];     // rotating tensors inside a stage
  float* head_ws;
  int chunk;
  LevelSizes sz;          // of the slot shape H x W
};
}  // namespace

static LevelSizes level_sizes(int H, int W) {
  LevelSizes z;
  z.h[0] = H;
  z.w[0] = W;
  for (int l = 1; l < RG_LEVELS; ++l) {
    int h = z.h[l - 1], w = z.w[l - 1];
    if (l == 1) { h = (h + 6 - 7) / 2 + 1; w = (w + 6 - 7) / 2 + 1; }           // stem conv 7x7/s2/p3
    else if (l != 3) { h = (h + 2 - 3) / 2 + 1; w = (w + 2 - 3) / 2 + 1; }     // maxpool, layer2..4 (layer1: stride 1)
    z.h[l] = h;
    z.w[l] = w;
  }
  return z;
}

// Ragged batches: B pictures of sizes (h_i, w_i) in the top-left corners of B slots of one shape (H, W).  Every kernel
// writes 0 outside a picture (what zero padding feeds its border) and the head pools over the picture's own pixels,
// so each descriptor equals, bit for bit, the one of a B = 1 forward of the picture at its own size.  The extent table
// holds per picture and resolution level one row {h, w, plain, block}: plain / block = the K order (1 = HALO order,
// 0 = tap by tap) that a B = 1 forward gives a 3x3 stride-1 convolution at that level, standalone / as conv2 of an
// identity Bottleneck (which fuse_c23 may take).  Where a pass's pictures disagree with the slot's kernel choice, that
// convolution runs image by image in each picture's own order (ConvExt::kc_major).
namespace {
struct Ragged {
  const int* dev = nullptr;    // table rows of the pass's pictures (device)
  const int* host = nullptr;   // the same rows on the host
  bool on() const { return dev != nullptr; }
  ConvExt at(int lvl, int nb, int slot_w) const { return ConvExt{dev + 4 * lvl, RG_LD, nb, nullptr, slot_w}; }
  bool all(int lvl, int col, int nb, int v) const {
    for (int i = 0; i < nb; ++i)
      if (host[static_cast<size_t>(i) * RG_LD + 4 * lvl + col] != v) return false;
    return true;
  }
};
}  // namespace

// The HALO mode's choice of conv_pers_any for a 3x3 stride-1 convolution at h x w (conv_impl 2 never takes it).
static bool halo_order_plain(const dirb200_net* n, int h, int w) {
  return get_conv_halo() && n->conv_impl == 0 && h >= 16 && w >= 8;
}

// Whether an identity Bottleneck of B images at h x w with Cm mid channels runs as the fused conv_c23 kernel.
static bool c23_taken(const dirb200_net* n, int B, int h, int w, int Cm) {
  return !n->basic && n->fuse_c23 && n->conv_impl == 0 &&
         (n->fuse_c23 == 2 ? conv_c23_supported(h, w, Cm) : conv_c23_profitable(B, h, w, Cm));
}

// Whether identity Bottleneck b's conv3 and the conv1 of the block after it (next; null at the end of a stage) run as
// the fused conv_c31 kernel for B images at h x w: both blocks stride-1 identity Bottlenecks, at most 256 mid channels
// and a tile for every SM.  Layer4's 512 mid channels would need 256 accumulator registers per thread for conv1 alone.
static bool c31_taken(const dirb200_net* n, const Block& b, const Block* next, int B, int h, int w) {
  return !n->basic && n->conv_impl == 0 && next != nullptr && !b.has_down && b.c2.stride == 1 && !next->has_down &&
         next->c2.stride == 1 && conv_c31_profitable(B, h, w, b.c3.Cin);
}

static void ragged_table(const dirb200_net* n, const int* hw, int B, std::vector<int>* t) {
  t->assign(static_cast<size_t>(B) * RG_LD, 0);
  for (int i = 0; i < B; ++i) {
    int* r = t->data() + static_cast<size_t>(i) * RG_LD;
    const LevelSizes z = level_sizes(hw[2 * i], hw[2 * i + 1]);
    for (int l = 0; l < RG_LEVELS; ++l) {
      const int Cm = 64 << std::max(0, l - 3);   // mid channels of the identity blocks at level l (layer1 at 2 and 3)
      r[4 * l] = z.h[l];
      r[4 * l + 1] = z.w[l];
      r[4 * l + 2] = halo_order_plain(n, z.h[l], z.w[l]) ? 1 : 0;
      r[4 * l + 3] = (c23_taken(n, 1, z.h[l], z.w[l], Cm) || r[4 * l + 2]) ? 1 : 0;
    }
  }
}

// Whether the stem and its maxpool run as one kernel (stem_pool); the mma.sync stem of conv_impl 1 has no fused form.
static bool stem_fused(const dirb200_net* n) { return n->fuse_stem && n->conv_impl != 1; }

static int setup_workspace(dirb200_net* n, int chunk, int H, int W, Workspace* w) {
  w->chunk = chunk;
  w->sz = level_sizes(H, W);
  const int* h = w->sz.h;
  const int* wd = w->sz.w;
  const size_t c = chunk;
  // the fused stem reads the images and writes the pooled map: neither intermediate exists
  const bool unfused = !stem_fused(n);
  const size_t sws = unfused ? std::max(c * H * W * 8, stem_workspace_bytes(chunk, H, W) / 2) : 0;
  const size_t stem = unfused || n->debug_taps ? c * h[1] * wd[1] * 64 : 0;
  size_t scr = 0;   // largest tensor inside any stage: conv1 output at the stage's input resolution, or a block output
  for (int s = 1; s < 5; ++s) {
    scr = std::max(scr, c * h[1 + s] * wd[1 + s] * (n->stage_ch[s] / 4));
    scr = std::max(scr, c * h[2 + s] * wd[2 + s] * n->stage_ch[s]);
  }
  if (n->fpn)   // the merged / smoothed layer3 map of the FPN head lives in a scratch tensor
    scr = std::max(scr, c * h[5] * wd[5] * n->stage_ch[3]);
  size_t head_floats = head_workspace_floats(chunk, h[6] * wd[6], n->stage_ch[4], n->out_dim);
  if (n->fpn) {
    const size_t partial = std::max(head_partial_floats(chunk, h[5] * wd[5], n->stage_ch[3]),
                                    head_partial_floats(chunk, h[6] * wd[6], n->stage_ch[4]));
    head_floats = partial + c * (n->feat_in() + std::max(n->out_dim, n->feat_in()));
  }
  auto layout = [&](void* base) {
    Carver cv(base, 1024);
    __half* stem_ws = cv.take<__half>(sws);
    __half* stem_out = cv.take<__half>(stem);
    w->stem_ws = unfused ? stem_ws : nullptr;
    w->stem_out = unfused || n->debug_taps ? stem_out : nullptr;
    for (int s = 0; s < 4; ++s) w->stage_out[s] = cv.take<__half>(c * h[2 + s] * wd[2 + s] * n->stage_ch[s]);
    for (int i = 0; i < 4; ++i) w->scratch[i] = cv.take<__half>(scr);
    w->head_ws = cv.take<float>(head_floats);
    return cv.used;
  };
  DIRB_TRY(grow_device(&n->ws, &n->ws_bytes, layout(nullptr)));
  layout(n->ws);
  return 0;
}

// One pass of the network over cb <= w.chunk images on the device (NCHW fp32 imgs, or HWC uint8 imgs_u8) -> cb
// descriptors.
static int run_chunk(dirb200_net* n, const Workspace& w, const float* imgs, const uint8_t* imgs_u8, int cb, int H, int W,
                     float* desc_dev, __half* desc16_dev, cudaStream_t stream, const Ragged& rg) {
  const int D = n->desc_dim();
  const int* lh = w.sz.h;   // size per level (level_sizes)
  const int* lw = w.sz.w;
  ConvExt e0, e1, e2;   // extents handed to one launch (ragged batches; the launchers read them on the host)
  auto ext = [&](ConvExt& e, int lvl, int slot_w) -> const ConvExt* {
    if (!rg.on()) return nullptr;
    e = rg.at(lvl, cb, slot_w);
    return &e;
  };
  // 3x3 stride-1 convolution whose K order on the slot is slot_order: pictures that a B = 1 forward gives another
  // order (column col of the table) make the launch pick the order image by image
  auto ext3 = [&](ConvExt& e, int lvl, int slot_w, int col, bool slot_order) -> const ConvExt* {
    if (!rg.on()) return nullptr;
    e = rg.at(lvl, cb, slot_w);
    if (!rg.all(lvl, col, cb, slot_order ? 1 : 0)) e.kc_major = e.hw + col;
    return &e;
  };
  // ---------------------------------------------------------------- stage 0: stem + maxpool
  if (stem_fused(n)) {
    const double flops = 2.0 * cb * lh[1] * lw[1] * 64.0 * 147.0;
    n->last_flops += flops;
    // bytes: the images once, the pooled map once, the weights
    const double bytes = static_cast<double>(cb) * ((imgs_u8 ? 3.0 : 12.0) * H * W + 128.0 * lh[2] * lw[2]) + 64.0 * 256 * 2;
    ProfScope ps(n, stream, 1, flops, bytes, "stem 7x7/s2 3->64 + maxpool 3x3/s2 fused");
    DIRB_TRY(stem_pool(imgs, imgs_u8, n->mean_std, cb, H, W, n->stem_w2, n->stem.scale, n->stem.shift, w.stage_out[0],
                       n->debug_taps ? w.stem_out : nullptr, stream, ext(e0, 0, W), ext(e1, 1, lw[1]), ext(e2, 2, lw[2])));
    DIRB_TRY(record_tap(n, "stem_conv", w.stem_out, cb, lh[1], lw[1], 64, stream));
  } else if (n->conv_impl == 1) {
    DIRB_REQUIRE(imgs_u8 == nullptr, DIRB200_ENOTSUP, "uint8 input needs the space-to-depth stem (conv_impl 0)");
    {
      ProfScope ps(n, stream, 2, 0, static_cast<double>(cb) * H * W * (12 + 16));
      DIRB_TRY(nchw_to_nhwc8(imgs, cb, H, W, w.stem_ws, stream));
    }
    DIRB_TRY(run_conv(n, n->stem, w.stem_ws, cb, H, W, nullptr, 1, w.stem_out, stream, /*force_mma=*/1));
  } else {
    const double flops = 2.0 * cb * lh[1] * lw[1] * 64.0 * 147.0;
    n->last_flops += flops;
    ProfScope ps(n, stream, 1, flops, static_cast<double>(cb) * (12.0 * H * W + 2.0 * stem_workspace_bytes(1, H, W) + 128.0 * lh[1] * lw[1]), "stem s2d + 7x7/s2 3->64");
    DIRB_TRY(stem_tc(imgs, cb, H, W, n->stem_w2, n->stem.scale, n->stem.shift, w.stem_ws, w.stem_out, stream, imgs_u8,
                     n->mean_std, ext(e0, 0, W), ext(e1, 1, lw[1])));
  }
  if (!stem_fused(n)) {
    DIRB_TRY(record_tap(n, "stem_conv", w.stem_out, cb, lh[1], lw[1], 64, stream));
    ProfScope ps(n, stream, 2, 0, 2.0 * cb * 64 * (static_cast<double>(lh[1]) * lw[1] + static_cast<double>(lh[2]) * lw[2]), "maxpool 3x3/s2");
    DIRB_TRY(maxpool_3x3s2(w.stem_out, cb, lh[1], lw[1], 64, w.stage_out[0], stream, ext(e0, 2, lw[2])));
  }
  DIRB_TRY(record_tap(n, "stem", w.stage_out[0], cb, lh[2], lw[2], 64, stream));
  // ---------------------------------------------------------------- stages 1..4: layer1..layer4
  const __half* x = w.stage_out[0];
  int first = 0;
  bool t1_ready = false;   // the block's conv1 output was written together with the previous block's output (conv_c31)
  for (int s = 1; s < 5; ++s) {
    const int last = n->layer_end[s - 1];       // blocks [first, last)
    int lvl = 1 + s;                            // level of x
    for (int bi = first; bi < last; ++bi) {
      const Block& blk = n->blocks[bi];
      const int j = bi - first;
      const int lvl_in = lvl;
      if ((n->basic ? blk.c1.stride : blk.c2.stride) == 2) lvl = 2 + s;   // level of the block's output
      const int h = lh[lvl_in], wd = lw[lvl_in], h2 = lh[lvl], w2 = lw[lvl];
      __half* t1 = w.scratch[0];
      __half* t2 = w.scratch[1];
      __half* rs = w.scratch[2];
      __half* y = (j % 2 == 0) ? w.scratch[3] : w.scratch[2];
      if (bi == last - 1 && s < 4) y = w.stage_out[s];
      // debug taps of this block: "layerL.B" (its output) and "layerL.B.conv1" / ".conv2" / ".down" (L = s, B = j, as
      // in the state-dict keys)
      const std::string tp = "layer" + std::to_string(s) + "." + std::to_string(j);
      const int cm = blk.c1.Cout, cout = n->stage_ch[s];
      if (n->basic) {
        // BasicBlock, resnet.py:27-44: 3x3(stride) + BN + ReLU -> 3x3 + BN -> + (projected) x -> ReLU
        DIRB_TRY(run_conv(n, blk.c1, x, cb, h, wd, nullptr, 1, t1, stream, 0,
                          blk.c1.stride == 1 ? ext3(e0, lvl, w2, 2, halo_order_plain(n, h2, w2)) : ext(e0, lvl, w2)));
        DIRB_TRY(record_tap(n, tp + ".conv1", t1, cb, h2, w2, cm, stream));
        const __half* res = x;
        if (blk.has_down) {
          DIRB_TRY(run_conv(n, blk.down, x, cb, h, wd, nullptr, 0, rs, stream, 0, ext(e0, lvl, w2)));
          DIRB_TRY(record_tap(n, tp + ".down", rs, cb, h2, w2, cout, stream));
          res = rs;
        }
        DIRB_TRY(run_conv(n, blk.c2, t1, cb, h2, w2, res, 1, y, stream, 0, ext3(e0, lvl, w2, 2, halo_order_plain(n, h2, w2))));
        DIRB_TRY(record_tap(n, tp, y, cb, h2, w2, cout, stream));
        x = y;
        continue;
      }
      const int st = blk.c2.stride;
      if (!t1_ready) {
        DIRB_TRY(run_conv(n, blk.c1, x, cb, h, wd, nullptr, 1, t1, stream, 0, ext(e0, lvl_in, wd)));
        DIRB_TRY(record_tap(n, tp + ".conv1", t1, cb, h, wd, cm, stream));
      }
      t1_ready = false;
      const bool c23 = !blk.has_down && st == 1 && c23_taken(n, cb, h, wd, blk.c2.Cin);
      // ragged: a stride-1 conv2 in the K order of the slot's kernel choice (the fused kernel has the HALO order)
      const ConvExt* e2 = st == 1 ? ext3(e1, lvl, wd, blk.has_down ? 2 : 3, c23 || halo_order_plain(n, h, wd))
                                  : ext(e1, lvl, w2);
      if (c23 && (e2 == nullptr || e2->kc_major == nullptr)) {
        // identity block: conv2 -> conv3 (+ x) in one kernel, the conv2 output stays in shared memory
        const int Cm = blk.c2.Cin;
        const double flops = 2.0 * cb * h * wd * (9.0 * Cm * Cm + 4.0 * Cm * Cm);
        const double bytes = 2.0 * (static_cast<double>(cb) * h * wd * (Cm + 8.0 * Cm) + 13.0 * Cm * Cm);   // t1 + residual + output, weights
        n->last_flops += flops;
        char tg[96];
        snprintf(tg, sizeof(tg), "3x3 %d->%d + 1x1 ->%d +res fused @%dx%d", Cm, Cm, 4 * Cm, h, wd);
        ProfScope ps(n, stream, 0, flops, bytes, tg);
        DIRB_TRY(conv_c23(cb, h, wd, Cm, t1, blk.c2.w, blk.c2.scale, blk.c2.shift, blk.c3.w, blk.c3.scale, blk.c3.shift, x, y,
                          stream, e2));
        DIRB_TRY(record_tap(n, tp, y, cb, h, wd, cout, stream));
        x = y;
        continue;
      }
      DIRB_TRY(run_conv(n, blk.c2, t1, cb, h, wd, nullptr, 1, t2, stream, 0, e2));
      DIRB_TRY(record_tap(n, tp + ".conv2", t2, cb, h2, w2, cm, stream));
      if (blk.has_down && n->fuse_ds && n->conv_impl == 0 && blk.c3.Cout % 256 == 0) {
        const double flops = 2.0 * cb * h2 * w2 * static_cast<double>(blk.c3.Cout) * (blk.c3.Cin + blk.down.Cin);
        const double bytes = 2.0 * (static_cast<double>(cb) * h2 * w2 * (blk.c3.Cin + blk.c3.Cout) +
                                    static_cast<double>(cb) * h * wd * blk.down.Cin +
                                    static_cast<double>(blk.c3.Cout) * (blk.c3.Cin + blk.down.Cin));
        n->last_flops += flops;
        char tbuf_[96];
        snprintf(tbuf_, sizeof(tbuf_), "1x1 [%d|%d%s]->%d fused-shortcut @%dx%d", blk.c3.Cin, blk.down.Cin, st == 2 ? "/s2" : "", blk.c3.Cout, h2, w2);
        ProfScope ps(n, stream, 0, flops, bytes, tbuf_);
        DIRB_TRY(conv_fused_ds(cb, h2, w2, blk.c3.Cin, t2, h, wd, blk.down.Cin, st, x, blk.wcat, blk.c3.Cout, blk.ones,
                               blk.cat_shift, y, stream, ext(e0, lvl, w2)));
        DIRB_TRY(record_tap(n, tp, y, cb, h2, w2, cout, stream));
        x = y;
        continue;
      }
      if (c31_taken(n, blk, bi + 1 < last ? &n->blocks[bi + 1] : nullptr, cb, h, wd)) {
        // identity block followed by an identity block: conv3 (+ x) and the next block's conv1 in one kernel, the
        // block output feeds conv1 from shared memory; the next block starts at conv2
        const int Cm = blk.c3.Cin;
        const double flops = 2.0 * cb * h * wd * (8.0 * Cm * Cm);
        const double bytes = 2.0 * (static_cast<double>(cb) * h * wd * (2.0 * Cm + 8.0 * Cm) + 8.0 * Cm * Cm);   // t2 + t1, x + y, weights
        n->last_flops += flops;
        char tg[96];
        snprintf(tg, sizeof(tg), "1x1 %d->%d +res + 1x1 ->%d fused @%dx%d", Cm, 4 * Cm, Cm, h, wd);
        ProfScope ps(n, stream, 0, flops, bytes, tg);
        const Block& nx = n->blocks[bi + 1];
        DIRB_TRY(conv_c31(cb, h, wd, Cm, t2, blk.c3.w, blk.c3.scale, blk.c3.shift, x, y, nx.c1.w, nx.c1.scale, nx.c1.shift,
                          t1, stream, ext(e0, lvl, w2)));
        DIRB_TRY(record_tap(n, tp, y, cb, h, wd, cout, stream));
        DIRB_TRY(record_tap(n, "layer" + std::to_string(s) + "." + std::to_string(j + 1) + ".conv1", t1, cb, h, wd, Cm, stream));
        t1_ready = true;
        x = y;
        continue;
      }
      const __half* res = x;
      if (blk.has_down) {
        DIRB_TRY(run_conv(n, blk.down, x, cb, h, wd, nullptr, 0, rs, stream, 0, ext(e0, lvl, w2)));
        DIRB_TRY(record_tap(n, tp + ".down", rs, cb, h2, w2, cout, stream));
        res = rs;
      }
      DIRB_TRY(run_conv(n, blk.c3, t2, cb, h2, w2, res, 1, y, stream, 0, ext(e0, lvl, w2)));
      DIRB_TRY(record_tap(n, tp, y, cb, h2, w2, cout, stream));
      x = y;
    }
    if (s < 4) DIRB_TRY(record_tap(n, "layer" + std::to_string(s), w.stage_out[s], cb, lh[2 + s], lw[2 + s], n->stage_ch[s], stream));
    first = last;
  }
  // ---------------------------------------------------------------- head
  const int C4 = n->stage_ch[4], ho = lh[6], wo = lw[6];
  DIRB_TRY(record_tap(n, "layer4", x, cb, ho, wo, C4, stream));
  if (n->fpn) {
    // ---- FPN head, rmac_resnet_fpn.py:52-90
    const int C3 = n->stage_ch[3], h3 = lh[5], w3 = lw[5], Ct = C3 + C4;
    const __half* x4 = w.stage_out[3];
    if (n->fpn_mode == 1) {
      // relu(conv1x5(upsample(x5))) == upsample(relu(conv1x5(x5))): the 1x1 convolution runs on the small map.
      // x (layer4 output) sits in scratch[2] or [3]; scratch[0] / [1] are free after the last block.
      __half* tbuf = w.scratch[0];
      __half* x4p = w.scratch[1];
      DIRB_TRY(run_conv(n, n->fpn_lat, x, cb, ho, wo, nullptr, 1, tbuf, stream));
      DIRB_TRY(record_tap(n, "fpn_lat", tbuf, cb, ho, wo, C3, stream));
      {
        ProfScope ps(n, stream, 2, 0, 2.0 * cb * (2.0 * h3 * w3 + static_cast<double>(ho) * wo) * C3);
        DIRB_TRY(upsample_add(x4, tbuf, x4p, cb, h3, w3, ho, wo, C3, stream));
      }
      DIRB_TRY(record_tap(n, "fpn_merge", x4p, cb, h3, w3, C3, stream));
      DIRB_TRY(run_conv(n, n->fpn_smooth, x4p, cb, h3, w3, nullptr, 1, tbuf, stream));
      x4 = tbuf;
      DIRB_TRY(record_tap(n, "fpn_c4", x4, cb, h3, w3, C3, stream));
    }
    ProfScope ps(n, stream, 3, n->without_fc ? 0.0 : 2.0 * cb * static_cast<double>(Ct) * n->out_dim,
                 2.0 * cb * (static_cast<double>(ho) * wo * C4 + static_cast<double>(h3) * w3 * C3));
    const size_t partial_floats = std::max(head_partial_floats(w.chunk, h3 * w3, C3), head_partial_floats(w.chunk, ho * wo, C4));
    float* partial = w.head_ws;
    float* g = partial + partial_floats;
    float* yv = g + static_cast<size_t>(w.chunk) * Ct;
    DIRB_TRY(head_pool(x4, cb, h3 * w3, C3, 0, n->gem_p4, n->gem_eps, 0, partial, g, Ct, 0, stream));    // torch.cat((x4, x5), 1)
    DIRB_TRY(head_pool(x, cb, ho * wo, C4, 0, n->gem_p, n->gem_eps, 0, partial, g, Ct, C3, stream));
    if (n->norm_features) DIRB_TRY(l2_normalize(g, cb, Ct, 1e-12f, g, nullptr, stream));
    DIRB_TRY(head_fc_l2(g, cb, Ct, n->without_fc ? nullptr : n->fc_w, n->without_fc ? nullptr : n->fc_b, D, yv, desc_dev,
                        desc16_dev, stream));
    if (!n->without_fc) n->last_flops += 2.0 * cb * static_cast<double>(Ct) * n->out_dim;
    return 0;
  }
  ProfScope ps(n, stream, 3, n->without_fc ? 0.0 : 2.0 * cb * static_cast<double>(C4) * n->out_dim, 2.0 * cb * ho * wo * static_cast<double>(C4), "head pool+fc+l2");
  if (n->center_bias > 0.0f)   // x is a scratch buffer whose only remaining reader is the pooling below
    DIRB_TRY(center_bias(const_cast<__half*>(x), cb, ho, wo, C4, n->center_bias, stream, ext(e0, 6, wo)));
  DIRB_TRY(head_pool_fc_l2(x, cb, ho * wo, C4, n->pooling, n->gem_p, n->gem_eps, n->norm_features,
                           n->without_fc ? nullptr : n->fc_w, n->without_fc ? nullptr : n->fc_b, D, w.head_ws, desc_dev,
                           desc16_dev, stream, n->head_bar, ext(e0, 6, wo)));
  if (!n->without_fc) n->last_flops += 2.0 * cb * static_cast<double>(C4) * n->out_dim;
  return 0;
}

static int check_forward_args(dirb200_net* n, int B, int H, int W) {
  DIRB_REQUIRE(n->finalized, DIRB200_ESTATE, "dirb200_net_finalize has not been called");
  DIRB_REQUIRE(B >= 1 && H >= 32 && W >= 32, DIRB200_ENOTSUP, "need B >= 1 and H, W >= 32 (got %d, %d, %d)", B, H, W);
  return 0;
}

// Bookkeeping of one forward call: its launch and flop counts (dirb200_net_last_launches) and, unless option
// "profile" 2 accumulates over calls, its profile.  begin_forward returns the launch counter end_forward needs.
static int64_t begin_forward(dirb200_net* n) {
  n->last_flops = 0;
  if (n->profile != 2) n->prof.reset();
  return launches_total();
}

static void end_forward(dirb200_net* n, int64_t launches0) { n->last_launches = launches_total() - launches0; }

// Device buffers in and out, on `stream`: B images, NCHW fp32 (f32) or HWC uint8 (u8), -> B descriptors.  hw_host =
// the pictures' sizes of a ragged batch (see Ragged), nullptr for a dense batch.
static int forward_dev(dirb200_net* n, const float* f32, const uint8_t* u8, int B, int H, int W, const int* hw_host,
                       float* desc_dev, __half* desc16_dev, cudaStream_t stream) {
  DIRB_TRY(check_forward_args(n, B, H, W));
  DIRB_CUDA(cudaSetDevice(n->device));
  std::vector<int> table;
  if (hw_host) {
    DIRB_REQUIRE(!n->fpn, DIRB200_ENOTSUP,
                 "ragged batches do not support FPN heads (their upsampling ratio depends on each picture's size)");
    DIRB_REQUIRE(n->conv_impl != 1, DIRB200_ENOTSUP, "ragged batches need the wgmma convolutions (conv_impl 0 or 2)");
    for (int i = 0; i < B; ++i)
      DIRB_REQUIRE(hw_host[2 * i] >= 32 && hw_host[2 * i] <= H && hw_host[2 * i + 1] >= 32 && hw_host[2 * i + 1] <= W,
                   DIRB200_EINVAL, "picture %d: size %dx%d is outside [32, %d] x [32, %d]", i, hw_host[2 * i],
                   hw_host[2 * i + 1], H, W);
    ragged_table(n, hw_host, B, &table);
    const size_t tbytes = table.size() * sizeof(int);
    DIRB_TRY(grow_device(reinterpret_cast<void**>(&n->ext_dev), &n->ext_bytes, tbytes));
    // pageable source: the copy is staged before the call returns, and it is ordered before the kernels that read it
    DIRB_CUDA(cudaMemcpyAsync(n->ext_dev, table.data(), tbytes, cudaMemcpyHostToDevice, stream));
  }
  const int64_t launches0 = begin_forward(n);
  const int chunk = n->chunk > 0 ? std::min(n->chunk, B) : auto_chunk(B, H, W);
  const int D = n->desc_dim();
  Workspace w;
  DIRB_TRY(setup_workspace(n, chunk, H, W, &w));
  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int cb = std::min(chunk, B - b0);
    const size_t img = static_cast<size_t>(b0) * 3 * H * W;
    Ragged rg;
    if (hw_host) {
      rg.dev = n->ext_dev + static_cast<size_t>(b0) * RG_LD;
      rg.host = table.data() + static_cast<size_t>(b0) * RG_LD;
    }
    DIRB_TRY(run_chunk(n, w, f32 ? f32 + img : nullptr, u8 ? u8 + img : nullptr, cb, H, W,
                       desc_dev + static_cast<size_t>(b0) * D, desc16_dev ? desc16_dev + static_cast<size_t>(b0) * D : nullptr,
                       stream, rg));
  }
  end_forward(n, launches0);
  return 0;
}

int dirb200_net_forward(dirb200_net* n, const float* imgs_dev, int B, int H, int W, float* desc_dev, void* desc16_dev,
                        void* stream) {
  DIRB_REQUIRE(n && imgs_dev && desc_dev, DIRB200_EINVAL, "null argument");
  return forward_dev(n, imgs_dev, nullptr, B, H, W, nullptr, desc_dev, static_cast<__half*>(desc16_dev),
                     static_cast<cudaStream_t>(stream));
}

int dirb200_net_forward_u8(dirb200_net* n, const uint8_t* imgs_dev, int B, int H, int W, float* desc_dev, void* desc16_dev,
                           void* stream) {
  DIRB_REQUIRE(n && imgs_dev && desc_dev, DIRB200_EINVAL, "null argument");
  return forward_dev(n, nullptr, imgs_dev, B, H, W, nullptr, desc_dev, static_cast<__half*>(desc16_dev),
                     static_cast<cudaStream_t>(stream));
}

// Ragged batch: B pictures of sizes hw_host[i] in the top-left corners of slots of H x W (see Ragged).
int dirb200_net_forward_ragged_u8(dirb200_net* n, const uint8_t* slots_dev, int B, int H, int W, const int* hw_host,
                                  float* desc_dev, void* desc16_dev, void* stream) {
  DIRB_REQUIRE(n && slots_dev && hw_host && desc_dev, DIRB200_EINVAL, "null argument");
  return forward_dev(n, nullptr, slots_dev, B, H, W, hw_host, desc_dev, static_cast<__half*>(desc16_dev),
                     static_cast<cudaStream_t>(stream));
}

int dirb200_net_forward_ragged(dirb200_net* n, const float* slots_dev, int B, int H, int W, const int* hw_host,
                               float* desc_dev, void* desc16_dev, void* stream) {
  DIRB_REQUIRE(n && slots_dev && hw_host && desc_dev, DIRB200_EINVAL, "null argument");
  return forward_dev(n, slots_dev, nullptr, B, H, W, hw_host, desc_dev, static_cast<__half*>(desc16_dev),
                     static_cast<cudaStream_t>(stream));
}

// Host buffers in, host descriptors out.  The batch is cut into chunks; the H2D copy of chunk i+1 (copy stream)
// overlaps the network pass over chunk i (compute stream), two device input buffers.
static int forward_host_impl(dirb200_net* n, const void* imgs_host_, int is_u8, int B, int H, int W, float* desc_host) {
  const uint8_t* imgs_host = static_cast<const uint8_t*>(imgs_host_);
  DIRB_REQUIRE(n && imgs_host && desc_host, DIRB200_EINVAL, "null argument");
  DIRB_TRY(check_forward_args(n, B, H, W));
  DIRB_CUDA(cudaSetDevice(n->device));
  if (!n->own_stream) DIRB_CUDA(cudaStreamCreateWithFlags(&n->own_stream, cudaStreamNonBlocking));
  if (!n->copy_stream) DIRB_CUDA(cudaStreamCreateWithFlags(&n->copy_stream, cudaStreamNonBlocking));
  // Chunk schedule: small chunks first so that compute starts after a short copy, then doubling sizes (large chunks
  // run the network more efficiently): host_chunk/2, host_chunk/2, host_chunk, 2*host_chunk, ... (option "chunk"
  // forces a uniform size).
  std::vector<int> sizes;
  {
    int left = B;
    if (n->chunk > 0) {
      while (left > 0) { sizes.push_back(std::min(left, n->chunk)); left -= sizes.back(); }
    } else {
      int c = std::max(1, n->host_chunk / 2);
      int reps = 2;
      while (left > 0) {
        const int v = std::min(left, c);
        sizes.push_back(v);
        left -= v;
        if (--reps == 0) { c = std::min(c * 2, 2 * n->host_chunk); reps = 1; }
      }
    }
  }
  const int nchunks = static_cast<int>(sizes.size());
  const int chunk = *std::max_element(sizes.begin(), sizes.end());
  const size_t img_bytes = static_cast<size_t>(3) * H * W * (is_u8 ? 1 : 4);
  const size_t in_bytes = 2 * static_cast<size_t>(chunk) * img_bytes;
  const int D = n->desc_dim();
  const size_t out_bytes = static_cast<size_t>(B) * D * 4;
  DIRB_TRY(grow_device(reinterpret_cast<void**>(&n->h2d), &n->h2d_bytes, in_bytes));
  DIRB_TRY(grow_device(reinterpret_cast<void**>(&n->d_desc), &n->d_desc_bytes, out_bytes));
  while (n->pipe_events.size() < static_cast<size_t>(2 * nchunks)) {
    cudaEvent_t e;
    DIRB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    n->pipe_events.push_back(e);
  }
  const int64_t launches0 = begin_forward(n);
  Workspace w;
  DIRB_TRY(setup_workspace(n, chunk, H, W, &w));
  int b0 = 0;
  for (int c = 0; c < nchunks; ++c) {
    const int cb = sizes[c];
    uint8_t* dst = reinterpret_cast<uint8_t*>(n->h2d) + static_cast<size_t>(c & 1) * chunk * img_bytes;
    cudaEvent_t copied = n->pipe_events[2 * c], done = n->pipe_events[2 * c + 1];
    if (c >= 2) DIRB_CUDA(cudaStreamWaitEvent(n->copy_stream, n->pipe_events[2 * (c - 2) + 1], 0));   // buffer free
    DIRB_CUDA(cudaMemcpyAsync(dst, imgs_host + static_cast<size_t>(b0) * img_bytes, static_cast<size_t>(cb) * img_bytes,
                              cudaMemcpyHostToDevice, n->copy_stream));
    DIRB_CUDA(cudaEventRecord(copied, n->copy_stream));
    DIRB_CUDA(cudaStreamWaitEvent(n->own_stream, copied, 0));
    DIRB_TRY(run_chunk(n, w, is_u8 ? nullptr : reinterpret_cast<const float*>(dst), is_u8 ? dst : nullptr, cb, H, W,
                       n->d_desc + static_cast<size_t>(b0) * D, nullptr, n->own_stream, Ragged()));
    DIRB_CUDA(cudaEventRecord(done, n->own_stream));
    b0 += cb;
  }
  DIRB_CUDA(cudaMemcpyAsync(desc_host, n->d_desc, out_bytes, cudaMemcpyDeviceToHost, n->own_stream));
  DIRB_CUDA(cudaStreamSynchronize(n->own_stream));
  end_forward(n, launches0);
  return 0;
}

int dirb200_net_forward_host(dirb200_net* n, const float* imgs_host, int B, int H, int W, float* desc_host) {
  return forward_host_impl(n, imgs_host, 0, B, H, W, desc_host);
}

int dirb200_net_forward_host_u8(dirb200_net* n, const uint8_t* imgs_host, int B, int H, int W, float* desc_host) {
  return forward_host_impl(n, imgs_host, 1, B, H, W, desc_host);
}

// Aggregated per-class timing of the last forward run with option "profile": out[4][4] = {launches, ms, flops, bytes}
// for class 0 wgmma convs, 1 stem conv, 2 layout + maxpool, 3 head.  Synchronises the device.
int dirb200_net_profile(dirb200_net* n, double* out16) {
  DIRB_REQUIRE(n && out16, DIRB200_EINVAL, "null argument");
  DIRB_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < 16; ++i) out16[i] = 0;
  for (auto& r : n->prof.recs) {
    float ms = 0;
    DIRB_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
    double* o = out16 + 4 * r.cls;
    o[0] += 1; o[1] += ms; o[2] += r.flops; o[3] += r.bytes;
  }
  return 0;
}

// Per launch-type timing of the profiled forward(s) as JSON text: [{"tag","cls","launches","ms","flops","bytes"}, ...]
// in first-launch order.  Returns the number of bytes needed (incl. the terminator) through *needed when buf is too
// small or NULL.  Synchronises the device.
int dirb200_net_profile_table(dirb200_net* n, char* buf, size_t cap, size_t* needed) {
  DIRB_REQUIRE(n, DIRB200_EINVAL, "null argument");
  DIRB_CUDA(cudaDeviceSynchronize());
  struct Row { std::string tag; int cls; double launches, ms, flops, bytes; };
  std::vector<Row> rows;
  std::map<std::string, size_t> at;
  for (auto& r : n->prof.recs) {
    float ms = 0;
    DIRB_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
    auto it = at.find(r.tag);
    if (it == at.end()) {
      at[r.tag] = rows.size();
      rows.push_back(Row{r.tag, r.cls, 0, 0, 0, 0});
      it = at.find(r.tag);
    }
    Row& row = rows[it->second];
    row.launches += 1; row.ms += ms; row.flops += r.flops; row.bytes += r.bytes;
  }
  std::string out = "[";
  for (size_t i = 0; i < rows.size(); ++i) {
    char line[320];
    snprintf(line, sizeof(line), "%s{\"tag\": \"%s\", \"cls\": %d, \"launches\": %.0f, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}",
             i ? ", " : "", rows[i].tag.c_str(), rows[i].cls, rows[i].launches, rows[i].ms, rows[i].flops, rows[i].bytes);
    out += line;
  }
  out += "]";
  if (needed) *needed = out.size() + 1;
  if (buf && cap >= out.size() + 1) memcpy(buf, out.c_str(), out.size() + 1);
  return 0;
}

int dirb200_net_debug_stage(dirb200_net* n, const char* what, void* dst_dev, size_t capacity, int dims[4],
                            void* stream_) {
  DIRB_REQUIRE(n && what && dst_dev && dims, DIRB200_EINVAL, "null argument");
  auto it = n->taps.find(what);
  DIRB_REQUIRE(it != n->taps.end() && it->second.ptr, DIRB200_EKEY,
               "no stage '%s' recorded (set option debug_taps=1 and run a forward first)", what);
  const auto& t = it->second;
  const size_t bytes = static_cast<size_t>(t.n) * t.h * t.w * t.c * 2;
  DIRB_REQUIRE(bytes <= capacity, DIRB200_EINVAL, "stage '%s' needs %zu bytes", what, bytes);
  dims[0] = t.n; dims[1] = t.h; dims[2] = t.w; dims[3] = t.c;
  DIRB_CUDA(cudaMemcpyAsync(dst_dev, t.ptr, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream_)));
  return 0;
}

int dirb200_net_last_launches(dirb200_net* n, int64_t* launches, double* flops) {
  DIRB_REQUIRE(n, DIRB200_EINVAL, "null");
  if (launches) *launches = n->last_launches;
  if (flops) *flops = n->last_flops;
  return 0;
}

int dirb200_net_destroy(dirb200_net* n) {
  if (!n) return 0;
  cudaSetDevice(n->device);
  for (void* p : n->owned) cudaFree(p);
  for (auto& kv : n->taps) if (kv.second.ptr) cudaFree(kv.second.ptr);
  if (n->ws) cudaFree(n->ws);
  if (n->h2d) cudaFree(n->h2d);
  if (n->d_desc) cudaFree(n->d_desc);
  if (n->ext_dev) cudaFree(n->ext_dev);
  if (n->own_stream) cudaStreamDestroy(n->own_stream);
  if (n->copy_stream) cudaStreamDestroy(n->copy_stream);
  for (auto e : n->pipe_events) cudaEventDestroy(e);
  delete n;
  return 0;
}

}  // extern "C"
