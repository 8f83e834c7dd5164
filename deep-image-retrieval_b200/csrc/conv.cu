// Convolution + folded BatchNorm (+ residual) (+ ReLU) on NHWC fp16 activations.
//   impl 0: persistent wgmma implicit GEMM (conv_pers.cuh) - every Bottleneck conv and the stem; 3x3/s1 convolutions
//           load each input patch once per channel block (option "halo")
//   impl 2: the same kernel with one tile per CTA (no persistence), kept as an A/B baseline
//   impl 1: mma.sync implicit GEMM            - the 7x7 stem (Cin padded 3 -> 8) and the validation path
// Reference semantics: dirtorch/nets/backbones/resnet.py:56-63 (convs, bias=False), :70-85 (BN, ReLU, residual add),
// :115-118 (stem).  BatchNorm (eval) is folded by the caller into scale = gamma/sqrt(var+eps), shift = beta-mean*scale.
#include "conv.h"

#include <algorithm>

#include "conv_c23.cuh"
#include "conv_c31.cuh"
#include "conv_pers.cuh"
#include "conv_stem.cuh"

namespace dirb {

// Pick the (tw,th,nb) output patch (tw*th*nb == 128) that minimises the number of tiles (= wasted MMA rows),
// preferring square-ish patches (input reuse in L2) on ties.
static void pick_patch(int B, int Ho, int Wo, int* tw, int* th, int* nb) {
  int64_t best = -1;
  int bt = 16, bh = 8, bb = 1, bscore = 1 << 30;
  for (int w = 1; w <= 128; w *= 2)
    for (int h = 1; w * h <= 128; h *= 2) {
      const int b = 128 / (w * h);
      if (w > 64 || h > 64) continue;  // keeps the TMA box (w*stride, h*stride) <= 256 for stride 2
      const int64_t tiles = ceil_div(Wo, w) * ceil_div(Ho, h) * ceil_div(B, b);
      const int shape_penalty = (w > h ? w / h : h / w) + (b > 1 ? 1 : 0) + (w < 8 ? 4 : 0);
      if (best < 0 || tiles < best || (tiles == best && shape_penalty < bscore)) {
        best = tiles;
        bscore = shape_penalty;
        bt = w;
        bh = h;
        bb = b;
      }
    }
  *tw = bt;
  *th = bh;
  *nb = bb;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Process-wide switch "halo": 3x3 stride-1 convolutions load their input patch once per 64-channel block (1, default)
// or tap by tap (0).
static int g_conv_halo = 1;
void set_conv_halo(int on) { g_conv_halo = on; }
int get_conv_halo() { return g_conv_halo; }

// Ragged batch: the epilogue zeroes every output pixel outside its image's extent (conv_pers.cuh).
static void set_ext(ConvPersParams& p, const ConvExt* ext, int out_h, int out_w) {
  if (ext == nullptr) return;
  p.ext = ext->hw;
  p.kc_major = ext->kc_major;
  p.ext_ld = ext->ld;
  p.ext_n = ext->n;
  p.out_h = out_h;
  p.out_w = out_w;
}

// Ring depth: as many 128 x 64 + BN x 64 operand slots as fit next to the convolution's staging buffers.
template <int BN>
struct PersStages {
  static constexpr int CONV = BN == 128 ? 5 : 7;
  static constexpr int SIM = 6;
};

static int set_total_tiles(ConvPersParams& p, int64_t total) {
  DIRB_REQUIRE(total > 0 && total < (int64_t(1) << 31), DIRB200_ENOTSUP, "tile count %lld out of range", (long long)total);
  p.total_tiles = static_cast<int>(total);
  return 0;
}

template <int BN, int STAGES, bool HALO, bool PP>
static int launch_conv_pers_mode(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmR,
                                 const CUtensorMap& tmO, const ConvPersParams& p, int grid_limit, cudaStream_t stream) {
  if (p.ext != nullptr)
    return conv_pers_launch<BN, STAGES, PERS_EPI_CONV, HALO, true, PP>(tmA, tmB, tmR, tmO, p, grid_limit, stream);
  return conv_pers_launch<BN, STAGES, PERS_EPI_CONV, HALO, false, PP>(tmA, tmB, tmR, tmO, p, grid_limit, stream);
}

// Convolution epilogue on the persistent kernel; the RAGGED instantiation when the launch carries image extents.
// When every CTA gets at least three tiles the consumer warpgroups ping-pong (one's epilogue runs under the other's
// MMAs).  With one tile per CTA ping-pong would leave the whole epilogue to 128 threads; with two there is a single
// overlap per CTA, and on an H100 the B = 1 forwards (layer1 / layer2 at 2-3 tiles per CTA) ran slower than
// cooperative, while B = 64 was as fast as with a threshold of two.  Both modes give bit-identical outputs.
template <int BN, int STAGES, bool HALO>
static int launch_conv_pers(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmR, const CUtensorMap& tmO,
                            ConvPersParams& p, int64_t total, int grid_limit, cudaStream_t stream) {
  DIRB_TRY(set_total_tiles(p, total));
  const int64_t grid = std::min<int64_t>(total, grid_limit);
  if (total >= 3 * grid)
    return launch_conv_pers_mode<BN, STAGES, HALO, true>(tmA, tmB, tmR, tmO, p, grid_limit, stream);
  return launch_conv_pers_mode<BN, STAGES, HALO, false>(tmA, tmB, tmR, tmO, p, grid_limit, stream);
}

template <int CM>
static int launch_c23(const CUtensorMap& tmA, const CUtensorMap& tmB2, const CUtensorMap& tmB3, const CUtensorMap& tmR,
                      const CUtensorMap& tmO, ConvPersParams& p, int64_t total, const float* scale2, const float* shift2,
                      cudaStream_t stream) {
  DIRB_TRY(set_total_tiles(p, total));
  if (p.ext != nullptr)
    return conv_c23_launch<CM, true>(tmA, tmB2, tmB3, tmR, tmO, p, scale2, shift2, num_sms(), stream);
  return conv_c23_launch<CM>(tmA, tmB2, tmB3, tmR, tmO, p, scale2, shift2, num_sms(), stream);
}

template <int BN>
static int conv_pers_bn(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
                        const __half* res, int relu, __half* out, cudaStream_t stream, int grid_limit,
                        const ConvExt* ext) {
  const int Ho = s.Ho(), Wo = s.Wo();
  const int Ktot = s.KH * s.KW * s.Cin;
  ConvPersParams p{};
  p.taps = s.KH * s.KW;
  p.kw_taps = s.KW;
  p.cin_blocks = s.Cin / 64;
  p.stride = s.stride;
  p.pad = s.pad;
  p.n_tiles = s.Cout / BN;
  p.has_res = res != nullptr;
  p.relu = relu;
  p.scale = scale;
  p.shift = shift;
  set_ext(p, ext, Ho, Wo);
  CUtensorMap tmA, tmB, tmR, tmO;
  int64_t m_tiles;
  const bool flat = (s.KH == 1 && s.KW == 1 && s.stride == 1 && s.pad == 0);
  if (flat) {
    const int64_t M = static_cast<int64_t>(s.B) * s.H * s.W;
    p.a_spatial = 0;
    p.tw = 128; p.th = 1; p.nb = 1; p.tiles_w = 1; p.tiles_h = 1;
    m_tiles = ceil_div(M, 128);
    DIRB_TRY(encode_tmap_2d(&tmA, in, s.Cin, M, (uint64_t)s.Cin * 2, 64, 128));
    DIRB_TRY(encode_tmap_2d(&tmO, out, s.Cout, M, (uint64_t)s.Cout * 2, 64, 128));
    if (res) DIRB_TRY(encode_tmap_2d(&tmR, res, s.Cout, M, (uint64_t)s.Cout * 2, 64, 128));
  } else {
    p.a_spatial = 1;
    if (p.kc_major != nullptr) {     // the K order is chosen per image: one image per tile
      p.tw = 8; p.th = 16; p.nb = 1;
    } else {
      pick_patch(s.B, Ho, Wo, &p.tw, &p.th, &p.nb);
    }
    p.tiles_w = (int)ceil_div(Wo, p.tw);
    p.tiles_h = (int)ceil_div(Ho, p.th);
    m_tiles = (int64_t)p.tiles_w * p.tiles_h * ceil_div(s.B, p.nb);
    DIRB_TRY(encode_tmap_nhwc(&tmA, in, s.B, s.H, s.W, s.Cin, p.tw, p.th, p.nb, s.stride));
    DIRB_TRY(encode_tmap_nhwc(&tmO, out, s.B, Ho, Wo, s.Cout, p.tw, p.th, p.nb, 1));
    if (res) DIRB_TRY(encode_tmap_nhwc(&tmR, res, s.B, Ho, Wo, s.Cout, p.tw, p.th, p.nb, 1));
  }
  if (!res) tmR = tmO;   // (never dereferenced without a residual)
  DIRB_TRY(encode_tmap_2d(&tmB, w, Ktot, s.Cout, (uint64_t)Ktot * 2, 64, BN));
  return launch_conv_pers<BN, PersStages<BN>::CONV, false>(tmA, tmB, tmR, tmO, p, m_tiles * p.n_tiles, grid_limit, stream);
}

// 3x3 / stride 1 / pad 1 with the input patch loaded once per 64-channel block (HALO mode of conv_pers.cuh).
template <int BN>
static int conv_halo_bn(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
                        const __half* res, int relu, __half* out, cudaStream_t stream, const ConvExt* ext) {
  ConvPersParams p{};
  p.a_spatial = 1;
  p.taps = 9; p.kw_taps = 3;
  p.cin_blocks = s.Cin / 64;
  p.stride = 1; p.pad = 1;
  p.tw = 8; p.th = 16; p.nb = 1;
  p.tiles_w = (int)ceil_div(s.W, 8);
  p.tiles_h = (int)ceil_div(s.H, 16);
  p.n_tiles = s.Cout / BN;
  p.has_res = res != nullptr;
  p.relu = relu;
  p.scale = scale;
  p.shift = shift;
  set_ext(p, ext, s.H, s.W);
  CUtensorMap tmA, tmB, tmR, tmO;
  DIRB_TRY(encode_tmap_nhwc_halo(&tmA, in, s.B, s.H, s.W, s.Cin));
  DIRB_TRY(encode_tmap_nhwc(&tmO, out, s.B, s.H, s.W, s.Cout, 8, 16, 1, 1));
  if (res) DIRB_TRY(encode_tmap_nhwc(&tmR, res, s.B, s.H, s.W, s.Cout, 8, 16, 1, 1));
  else tmR = tmO;
  DIRB_TRY(encode_tmap_2d(&tmB, w, 9 * s.Cin, s.Cout, (uint64_t)9 * s.Cin * 2, 64, BN));
  return launch_conv_pers<BN, BN == 128 ? 6 : 8, true>(tmA, tmB, tmR, tmO, p, (int64_t)p.tiles_w * p.tiles_h * s.B * p.n_tiles,
                                                       num_sms(), stream);
}

// Tile width (output channels per tile): 128 unless that would leave SMs without a tile - at batch 1-8 a wide tile
// leaves most SMs idle (e.g. layer3 conv1 of ONE 1024x1024 image is 64 tiles of 128 channels), so the tile narrows
// to 64 channels - the reference's default evaluation mode is batch 1 (test_dir.py:52-53,114).
static int conv_pers_any(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
                         const __half* res, int relu, __half* out, cudaStream_t stream, int grid_limit,
                         const ConvExt* ext) {
  DIRB_REQUIRE(s.Cin % 64 == 0 && s.Cout % 64 == 0, DIRB200_ENOTSUP,
               "wgmma conv needs Cin %% 64 == 0 and Cout %% 64 == 0 (got %d, %d)", s.Cin, s.Cout);
  DIRB_REQUIRE(s.stride == 1 || s.stride == 2, DIRB200_ENOTSUP, "stride %d unsupported", s.stride);
  const int64_t m_tiles = ceil_div(static_cast<int64_t>(s.B) * s.Ho() * s.Wo(), 128);
  const bool wide = s.Cout % 128 == 0 && m_tiles * (s.Cout / 128) >= num_sms();
  DIRB_REQUIRE(ext == nullptr || ext->kc_major == nullptr || (s.KH == 3 && s.KW == 3 && s.stride == 1 && s.pad == 1),
               DIRB200_EINVAL, "a per-image K order applies to 3x3 stride-1 convolutions only");
  const bool per_image_order = ext != nullptr && ext->kc_major != nullptr;
  if (g_conv_halo && !per_image_order && grid_limit == num_sms() && s.KH == 3 && s.KW == 3 && s.stride == 1 && s.pad == 1 && s.H >= 16 && s.W >= 8)
    return wide ? conv_halo_bn<128>(s, in, w, scale, shift, res, relu, out, stream, ext)
                : conv_halo_bn<64>(s, in, w, scale, shift, res, relu, out, stream, ext);
  if (wide)
    return conv_pers_bn<128>(s, in, w, scale, shift, res, relu, out, stream, grid_limit, ext);
  return conv_pers_bn<64>(s, in, w, scale, shift, res, relu, out, stream, grid_limit, ext);
}

int conv_tc(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
            const __half* res, int relu, __half* out, cudaStream_t stream, const ConvExt* ext) {
  return conv_pers_any(s, in, w, scale, shift, res, relu, out, stream, num_sms(), ext);
}

int conv_tc_np(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
               const __half* res, int relu, __half* out, cudaStream_t stream, const ConvExt* ext) {
  return conv_pers_any(s, in, w, scale, shift, res, relu, out, stream, 1 << 30, ext);   // one tile per CTA
}

// conv3 (1x1) of block 0 fused with the projection shortcut: out = relu([t2 | x_strided] . [W3*s3 | Wd*sd]^T + shift).
// t2: (B,Ho,Wo,Cmid); x: (B,Hx,Wx,Cx) read with spatial stride `xstride`; wcat: [Cout][Cmid + Cx] fp16.
int conv_fused_ds(int B, int Ho, int Wo, int Cmid, const __half* t2, int Hx, int Wx, int Cx, int xstride,
                  const __half* x, const __half* wcat, int Cout, const float* scale, const float* shift, __half* out,
                  cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(Cmid % 64 == 0 && Cx % 64 == 0 && Cout % 256 == 0, DIRB200_ENOTSUP, "fused shortcut needs 64-multiples");
  constexpr int BN = 128;
  ConvPersParams p{};
  p.a_spatial = 1;
  p.taps = 1; p.kw_taps = 1;
  p.cin_blocks = (Cmid + Cx) / 64;
  p.k_split = Cmid / 64;
  p.a2_stride = xstride;
  p.stride = 1; p.pad = 0;
  pick_patch(B, Ho, Wo, &p.tw, &p.th, &p.nb);
  p.tiles_w = (int)ceil_div(Wo, p.tw);
  p.tiles_h = (int)ceil_div(Ho, p.th);
  p.n_tiles = Cout / BN;
  p.has_res = 0;
  p.relu = 1;
  p.scale = scale;
  p.shift = shift;
  set_ext(p, ext, Ho, Wo);
  CUtensorMap tmA, tmB, tmX, tmO;
  DIRB_TRY(encode_tmap_nhwc(&tmA, t2, B, Ho, Wo, Cmid, p.tw, p.th, p.nb, 1));
  DIRB_TRY(encode_tmap_nhwc(&tmX, x, B, Hx, Wx, Cx, p.tw, p.th, p.nb, xstride));
  DIRB_TRY(encode_tmap_nhwc(&tmO, out, B, Ho, Wo, Cout, p.tw, p.th, p.nb, 1));
  DIRB_TRY(encode_tmap_2d(&tmB, wcat, Cmid + Cx, Cout, (uint64_t)(Cmid + Cx) * 2, 64, BN));
  return launch_conv_pers<BN, PersStages<BN>::CONV, false>(tmA, tmB, tmX, tmO, p,
                                                           (int64_t)p.tiles_w * p.tiles_h * ceil_div(B, p.nb) * p.n_tiles,
                                                           num_sms(), stream);
}

// Bottleneck conv2 (3x3/s1/p1) + BN + ReLU + conv3 (1x1, x4) + BN + residual + ReLU in one kernel (conv_c23.cuh).
// t1: (B,H,W,Cm); w2: [Cm][9*Cm]; w3: [4*Cm][Cm]; res / out: (B,H,W,4*Cm).
bool conv_c23_supported(int H, int W, int Cm) { return (Cm == 64 || Cm == 128 || Cm == 256) && H >= 16 && W >= 8; }
// worth trying only when every SM gets several 128-pixel tiles (each tile walks ALL 4*Cm output channels)
bool conv_c23_profitable(int B, int H, int W, int Cm) {
  return conv_c23_supported(H, W, Cm) && ceil_div(W, 8) * ceil_div(H, 16) * B >= 2 * num_sms();
}

int conv_c23(int B, int H, int W, int Cm, const __half* t1, const __half* w2, const float* scale2, const float* shift2,
             const __half* w3, const float* scale3, const float* shift3, const __half* res, __half* out,
             cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(conv_c23_supported(H, W, Cm), DIRB200_ENOTSUP, "fused conv2+conv3 needs Cm in {64, 128, 256}, H >= 16, W >= 8 (got %d, %d, %d)", Cm, H, W);
  DIRB_REQUIRE(t1 && w2 && w3 && res && out, DIRB200_EINVAL, "null argument");
  ConvPersParams p{};
  p.a_spatial = 1;
  p.tw = 8; p.th = 16; p.nb = 1;
  p.tiles_w = (int)ceil_div(W, 8);
  p.tiles_h = (int)ceil_div(H, 16);
  p.n_tiles = 1;
  p.scale = scale3;
  p.shift = shift3;
  set_ext(p, ext, H, W);
  const int64_t total = (int64_t)p.tiles_w * p.tiles_h * B;
  CUtensorMap tmA, tmB2, tmB3, tmR, tmO;
  DIRB_TRY(encode_tmap_nhwc_halo(&tmA, t1, B, H, W, Cm));
  DIRB_TRY(encode_tmap_2d(&tmB2, w2, 9 * Cm, Cm, (uint64_t)9 * Cm * 2, 64, Cm < 128 ? Cm : 128));
  DIRB_TRY(encode_tmap_2d(&tmB3, w3, Cm, 4 * Cm, (uint64_t)Cm * 2, 64, 128));
  DIRB_TRY(encode_tmap_nhwc(&tmR, res, B, H, W, 4 * Cm, 8, 16, 1, 1));
  DIRB_TRY(encode_tmap_nhwc(&tmO, out, B, H, W, 4 * Cm, 8, 16, 1, 1));
  if (Cm == 256) return launch_c23<256>(tmA, tmB2, tmB3, tmR, tmO, p, total, scale2, shift2, stream);
  if (Cm == 64) return launch_c23<64>(tmA, tmB2, tmB3, tmR, tmO, p, total, scale2, shift2, stream);
  return launch_c23<128>(tmA, tmB2, tmB3, tmR, tmO, p, total, scale2, shift2, stream);
}

// conv3 (1x1, Cm -> 4 Cm) + BN + residual + ReLU of identity Bottleneck b and conv1 (1x1, 4 Cm -> Cm) + BN + ReLU of
// identity Bottleneck b+1 in one kernel (conv_c31.cuh).  t2: (B,H,W,Cm); w3: [4*Cm][Cm]; x / y: (B,H,W,4*Cm) block b's
// input and output; w1: [Cm][4*Cm]; t1: (B,H,W,Cm) block b+1's conv1 output.
bool conv_c31_supported(int Cm) { return Cm == 64 || Cm == 128 || Cm == 256; }
// Each fused tile walks all 4*Cm channels of X: with fewer tiles than SMs some SMs would idle while the unfused
// launches spread narrower tiles over all of them.
bool conv_c31_profitable(int B, int H, int W, int Cm) {
  return conv_c31_supported(Cm) && ceil_div(static_cast<int64_t>(B) * H * W, 128) >= num_sms();
}

int conv_c31(int B, int H, int W, int Cm, const __half* t2, const __half* w3, const float* scale3, const float* shift3,
             const __half* x, __half* y, const __half* w1, const float* scale1, const float* shift1, __half* t1,
             cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(conv_c31_supported(Cm), DIRB200_ENOTSUP, "fused conv3+conv1 needs Cm in {64, 128, 256} (got %d)", Cm);
  DIRB_REQUIRE(t2 && w3 && scale3 && shift3 && x && y && w1 && scale1 && shift1 && t1, DIRB200_EINVAL, "null argument");
  const int64_t M = static_cast<int64_t>(B) * H * W;
  ConvPersParams p{};
  p.a_spatial = 0;
  p.scale = scale3;
  p.shift = shift3;
  set_ext(p, ext, H, W);
  DIRB_TRY(set_total_tiles(p, ceil_div(M, 128)));
  CUtensorMap tmT2, tmW3, tmX, tmY, tmW1, tmT1;   // activations in 64-row boxes: each consumer warpgroup moves its own rows
  DIRB_TRY(encode_tmap_2d(&tmT2, t2, Cm, M, (uint64_t)Cm * 2, 64, 64));
  DIRB_TRY(encode_tmap_2d(&tmW3, w3, Cm, 4 * Cm, (uint64_t)Cm * 2, 64, C31Smem<64>::N3));
  DIRB_TRY(encode_tmap_2d(&tmX, x, 4 * Cm, M, (uint64_t)Cm * 8, 64, 64));
  DIRB_TRY(encode_tmap_2d(&tmY, y, 4 * Cm, M, (uint64_t)Cm * 8, 64, 64));
  DIRB_TRY(encode_tmap_2d(&tmW1, w1, 4 * Cm, Cm, (uint64_t)Cm * 8, 64, Cm < 128 ? Cm : 128));
  DIRB_TRY(encode_tmap_2d(&tmT1, t1, Cm, M, (uint64_t)Cm * 2, 64, 64));
#define DIRB_C31(CM)                                                                                                   \
  return p.ext != nullptr                                                                                              \
             ? conv_c31_launch<CM, true>(tmT2, tmW3, tmX, tmY, tmW1, tmT1, p, scale1, shift1, num_sms(), stream)       \
             : conv_c31_launch<CM, false>(tmT2, tmW3, tmX, tmY, tmW1, tmT1, p, scale1, shift1, num_sms(), stream)
  if (Cm == 256) DIRB_C31(256);
  if (Cm == 128) DIRB_C31(128);
  DIRB_C31(64);
#undef DIRB_C31
}

// ------------------------------------------------------------------------------------------------ stem
// Stem conv 7x7 / stride 2 / pad 3 (3 -> 64 channels) + BN + ReLU (resnet.py:115-118,158-160).  The input is first
// rewritten as a zero-padded "space-to-depth" tensor
//     S[n][Y][X][(dy*2+dx)*4 + c] = img[n][c][2Y+dy-3][2X+dx-3]        (c < 3; channel 3 and the border are 0)
// with 16 fp16 channels per 2x2 pixel block.  The 7x7/s2 convolution over img is then a 4x4/s1 convolution over S:
//     out[ho][wo][co] = sum_{a,b in 0..3} sum_{j<16} S[ho+a][wo+b][j] * W2[co][a][b][j],
//     W2[co][a][b][(dy*2+dx)*4+c] = w[co][c][2a+dy][2b+dx]              (0 where 2a+dy or 2b+dx = 7, or c = 3)
// i.e. an implicit GEMM with K = 16 taps x 16 = 256.  S is stored row-expanded, R[n][Y][X][b*16 + j] = S[n][Y][X+b][j]
// (X < Wo, 64 channels = 128 bytes per pixel), so the stem is a 4x1 convolution over R with Cin = 64 and runs on the
// wgmma kernel (conv_pers.cuh) with the weight layout W2 unchanged (K index = a*64 + b*16 + j).
// NCHW fp32 -> R: one thread per 2x2 block and horizontal neighbour b.
// Ragged batch: ext = the pictures' {h, w} (stride ext_ld); pixels outside them are never read and enter as 0.
__global__ void s2d_kernel(const float* __restrict__ in, __half* __restrict__ out, int H, int W, int Hs, int Wo,
                           int64_t total, const int* __restrict__ ext, int ext_ld) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  const int X = static_cast<int>((i >> 2) % Wo) + static_cast<int>(i & 3);
  const int Y = static_cast<int>(((i >> 2) / Wo) % Hs);
  const int64_t n = (i >> 2) / (static_cast<int64_t>(Wo) * Hs);
  const int hn = ext ? __ldg(ext + n * ext_ld) : H, wn = ext ? __ldg(ext + n * ext_ld + 1) : W;
  const float* img = in + n * 3 * static_cast<int64_t>(H) * W;
  const int64_t plane = static_cast<int64_t>(H) * W;
  uint32_t o[8];
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int y = 2 * Y + dy - 3, x = 2 * X + dx - 3;
      float c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if (y >= 0 && y < hn && x >= 0 && x < wn) {
        const int64_t off = static_cast<int64_t>(y) * W + x;
        c0 = __ldg(img + off);
        c1 = __ldg(img + plane + off);
        c2 = __ldg(img + 2 * plane + off);
      }
      o[(dy * 2 + dx) * 2] = pack_h2(c0, c1);
      o[(dy * 2 + dx) * 2 + 1] = pack_h2(c2, 0.f);
    }
  uint4* dst = reinterpret_cast<uint4*>(out + i * 16);
  dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
  dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

// Same from uint8 HWC pixels (what an image decoder yields): ToTensor (x / 255) and Normalize ((v - mean) / std) of
// dirtorch/utils/transforms.py:27 are applied on the fly in fp32, in torch's order and with true divisions, so the
// fp16 values are bit-identical to those of the fp32-input path.
// Outside a ragged batch's pictures the input is 0 in normalised space (a uint8 0 would normalise to -mean/std).
__global__ void s2d_u8_kernel(const uint8_t* __restrict__ in, __half* __restrict__ out, int H, int W, int Hs, int Wo,
                              int64_t total, float m0, float m1, float m2, float s0, float s1, float s2,
                              const int* __restrict__ ext, int ext_ld) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  const int X = static_cast<int>((i >> 2) % Wo) + static_cast<int>(i & 3);
  const int Y = static_cast<int>(((i >> 2) / Wo) % Hs);
  const int64_t n = (i >> 2) / (static_cast<int64_t>(Wo) * Hs);
  const int hn = ext ? __ldg(ext + n * ext_ld) : H, wn = ext ? __ldg(ext + n * ext_ld + 1) : W;
  const uint8_t* img = in + n * 3 * static_cast<int64_t>(H) * W;
  uint32_t o[8];
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int y = 2 * Y + dy - 3, x = 2 * X + dx - 3;
      float c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if (y >= 0 && y < hn && x >= 0 && x < wn) {
        const uint8_t* px = img + (static_cast<int64_t>(y) * W + x) * 3;
        c0 = __fdiv_rn(__fdiv_rn(static_cast<float>(px[0]), 255.0f) - m0, s0);
        c1 = __fdiv_rn(__fdiv_rn(static_cast<float>(px[1]), 255.0f) - m1, s1);
        c2 = __fdiv_rn(__fdiv_rn(static_cast<float>(px[2]), 255.0f) - m2, s2);
      }
      o[(dy * 2 + dx) * 2] = pack_h2(c0, c1);
      o[(dy * 2 + dx) * 2 + 1] = pack_h2(c2, 0.f);
    }
  uint4* dst = reinterpret_cast<uint4*>(out + i * 16);
  dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
  dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

static void stem_dims(int H, int W, int* Ho, int* Wo, int* Hs, int* Ws) {
  *Ho = (H + 6 - 7) / 2 + 1;
  *Wo = (W + 6 - 7) / 2 + 1;
  *Hs = *Ho + 3;
  *Ws = *Wo + 3;
}

size_t stem_workspace_bytes(int B, int H, int W) {
  int Ho, Wo, Hs, Ws;
  stem_dims(H, W, &Ho, &Wo, &Hs, &Ws);
  (void)Ws;
  return static_cast<size_t>(B) * Hs * Wo * 128;
}

void pack_stem_w2(const float* w, __half* out) {
  for (int co = 0; co < 64; ++co)
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 4; ++b)
        for (int dy = 0; dy < 2; ++dy)
          for (int dx = 0; dx < 2; ++dx)
            for (int c = 0; c < 4; ++c) {
              const int kh = 2 * a + dy, kw = 2 * b + dx;
              float v = 0.f;
              if (c < 3 && kh < 7 && kw < 7) v = w[((co * 3 + c) * 7 + kh) * 7 + kw];
              out[co * 256 + (a * 4 + b) * 16 + (dy * 2 + dx) * 4 + c] = __float2half_rn(v);
            }
}

int stem_tc(const float* imgs, int B, int H, int W, const __half* w2, const float* scale, const float* shift,
            __half* s2d_ws, __half* out, cudaStream_t stream, const uint8_t* imgs_u8, const float* mean_std,
            const ConvExt* in_ext, const ConvExt* out_ext) {
  const int* ext = in_ext ? in_ext->hw : nullptr;
  const int ext_ld = in_ext ? in_ext->ld : 0;
  int Ho, Wo, Hs, Ws;
  stem_dims(H, W, &Ho, &Wo, &Hs, &Ws);
  (void)Ho;
  const int64_t total = static_cast<int64_t>(B) * Hs * Wo * 4;
  if (imgs_u8 != nullptr)
    s2d_u8_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(
        imgs_u8, s2d_ws, H, W, Hs, Wo, total, mean_std[0], mean_std[1], mean_std[2], mean_std[3], mean_std[4], mean_std[5],
        ext, ext_ld);
  else
    s2d_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(imgs, s2d_ws, H, W, Hs, Wo, total, ext, ext_ld);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  const ConvShape s{B, Hs, Wo, 64, 64, 4, 1, 1, 0};      // 4x1 over the row-expanded tensor: Ho = Hs - 3, Wo
  return conv_tc(s, s2d_ws, w2, scale, shift, nullptr, 1, out, stream, out_ext);
}

int stem_pool(const float* imgs, const uint8_t* imgs_u8, const float* mean_std, int B, int H, int W, const __half* w2,
              const float* scale, const float* shift, __half* out, __half* stem_out, cudaStream_t stream,
              const ConvExt* in_ext, const ConvExt* stem_ext, const ConvExt* pool_ext) {
  DIRB_REQUIRE((imgs != nullptr) != (imgs_u8 != nullptr) && (imgs_u8 == nullptr || mean_std != nullptr), DIRB200_EINVAL,
               "the fused stem takes fp32 images or uint8 images with their mean / std");
  DIRB_REQUIRE((in_ext == nullptr) == (stem_ext == nullptr) && (in_ext == nullptr) == (pool_ext == nullptr) &&
                   (in_ext == nullptr || (in_ext->ld == stem_ext->ld && in_ext->ld == pool_ext->ld)),
               DIRB200_EINVAL, "the fused stem needs the extents of all three levels of one table");
  DIRB_REQUIRE(3 * static_cast<int64_t>(H) * W < (int64_t(1) << 31), DIRB200_ENOTSUP, "image of %d x %d pixels too large", H, W);
  StemPoolParams p{};
  p.imgs = imgs;
  p.imgs_u8 = imgs_u8;
  if (imgs_u8 != nullptr) {
    p.m0 = mean_std[0]; p.m1 = mean_std[1]; p.m2 = mean_std[2];
    p.s0 = mean_std[3]; p.s1 = mean_std[4]; p.s2 = mean_std[5];
  }
  p.w2 = w2;
  p.scale = scale;
  p.shift = shift;
  p.out = out;
  p.stem_out = stem_out;
  int Hs, Ws;
  stem_dims(H, W, &p.Ho, &p.Wo, &Hs, &Ws);
  p.H = H;
  p.W = W;
  p.Hp = (p.Ho + 2 - 3) / 2 + 1;
  p.Wp = (p.Wo + 2 - 3) / 2 + 1;
  p.tiles_x = static_cast<int>(ceil_div(p.Wp, SP_PT));
  p.tiles_y = static_cast<int>(ceil_div(p.Hp, SP_PT));
  const int64_t total = static_cast<int64_t>(p.tiles_x) * p.tiles_y * B;
  DIRB_REQUIRE(total > 0 && total < (int64_t(1) << 31), DIRB200_ENOTSUP, "tile count %lld out of range", (long long)total);
  p.total_tiles = static_cast<int>(total);
  if (in_ext != nullptr) {
    p.ext0 = in_ext->hw;
    p.ext1 = stem_ext->hw;
    p.ext2 = pool_ext->hw;
    p.ext_ld = in_ext->ld;
  }
  constexpr int smem = StemPoolSmem::TOTAL;
  auto kern = imgs_u8 != nullptr ? stem_pool_kernel<true> : stem_pool_kernel<false>;
  static std::atomic<uint64_t> attr_done{0};
  if (first_launch_on_device(attr_done)) {
    DIRB_CUDA(cudaFuncSetAttribute(stem_pool_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DIRB_CUDA(cudaFuncSetAttribute(stem_pool_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  const int64_t grid = std::min<int64_t>(total, 2 * num_sms());   // two CTAs per SM (__launch_bounds__ of the kernel)
  DIRB_CUDA(launch_pdl(kern, dim3(static_cast<unsigned>(grid)), dim3(SP_THREADS), smem, stream, p));
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------ mma.sync path
// CTA tile 128 pixels x 64 channels, K chunks of 32, 3-stage cp.async ring, 8 warps (4 x 2), warp tile 32 x 32.
namespace {

constexpr int MM_BM = 128, MM_BN = 64, MM_BK = 32, MM_LD = 40 /* padded row, halfs */, MM_STAGES = 3;

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool pred) {
  const uint32_t d = smem_u32(dst);
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, const uint32_t* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

struct MmaConvParams {
  const __half* in;
  const __half* w;      // [Cout][Kpad]
  const float* scale;
  const float* shift;
  const __half* res;
  __half* out;
  int B, H, W, Cin, Cout, KH, KW, stride, pad, Ho, Wo;
  int Ktot, Kpad, M, relu;
};

__global__ void __launch_bounds__(256) conv_mma_kernel(const MmaConvParams p) {
  __shared__ __align__(16) __half sA[MM_STAGES][MM_BM][MM_LD];
  __shared__ __align__(16) __half sB[MM_STAGES][MM_BN][MM_LD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;          // 4 x 2 warps
  const int m0 = blockIdx.x * MM_BM, n0 = blockIdx.y * MM_BN;
  const int kchunks = p.Kpad / MM_BK;

  // A gather bookkeeping: this thread loads vector `av` (8 halfs) of rows ar0 and ar0+64.
  const int av = tid & 3, ar0 = tid >> 2;
  int a_n[2], a_h[2], a_w[2];
  bool a_ok[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int m = m0 + ar0 + 64 * j;
    a_ok[j] = m < p.M;
    const int mm = a_ok[j] ? m : 0;
    a_w[j] = (mm % p.Wo) * p.stride - p.pad;
    a_h[j] = ((mm / p.Wo) % p.Ho) * p.stride - p.pad;
    a_n[j] = mm / (p.Wo * p.Ho);
  }
  const int bv = tid & 3, br = tid >> 2;  // B: one vector of row br

  auto load_stage = [&](int kc, int st) {
    const int k = kc * MM_BK + av * 8;
    const int tap = k / p.Cin, c = k - tap * p.Cin;
    const int kh = tap / p.KW, kw = tap - kh * p.KW;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int hi = a_h[j] + kh, wi = a_w[j] + kw;
      const bool ok = a_ok[j] && k < p.Ktot && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W;
      const __half* src = ok ? p.in + ((static_cast<int64_t>(a_n[j]) * p.H + hi) * p.W + wi) * p.Cin + c : p.in;
      cp_async16(&sA[st][ar0 + 64 * j][av * 8], src, ok);
    }
    cp_async16(&sB[st][br][bv * 8], p.w + static_cast<int64_t>(n0 + br) * p.Kpad + kc * MM_BK + bv * 8, true);
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
  for (int s = 0; s < MM_STAGES - 1; ++s) {
    if (s < kchunks) load_stage(s, s);
    cp_async_commit();
  }
  for (int kc = 0; kc < kchunks; ++kc) {
    cp_async_wait<MM_STAGES - 2>();
    __syncthreads();
    {
      const int nk = kc + MM_STAGES - 1;
      if (nk < kchunks) load_stage(nk, nk % MM_STAGES);
      cp_async_commit();
    }
    const int st = kc % MM_STAGES;
#pragma unroll
    for (int ks = 0; ks < MM_BK; ks += 16) {
      uint32_t af[2][4], bf[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i)
        ldmatrix_x4(af[i], &sA[st][wm * 32 + i * 16 + (lane & 15)][ks + (lane >> 4) * 8]);
#pragma unroll
      for (int j = 0; j < 2; ++j)
        ldmatrix_x4(bf[j], &sB[st][wn * 32 + j * 16 + ((lane >> 4) << 3) + (lane & 7)][ks + ((lane >> 3) & 1) * 8]);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma16816(acc[i][j], af[i], &bf[j >> 1][(j & 1) * 2]);
    }
  }
  cp_async_wait<0>();

  // epilogue: c0,c1 -> (row g, cols 2t,2t+1); c2,c3 -> (row g+8)
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int m = m0 + wm * 32 + i * 16 + g + hrow * 8;
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = n0 + wn * 32 + j * 8 + t * 2;
        float v0 = fmaf(acc[i][j][hrow * 2 + 0], p.scale[c], p.shift[c]);
        float v1 = fmaf(acc[i][j][hrow * 2 + 1], p.scale[c + 1], p.shift[c + 1]);
        const int64_t off = static_cast<int64_t>(m) * p.Cout + c;
        if (p.res != nullptr) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.res + off));
          v0 += r.x;
          v1 += r.y;
        }
        if (p.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        *reinterpret_cast<__half2*>(p.out + off) = __floats2half2_rn(v0, v1);
      }
    }
}

}  // namespace

int conv_mma(const ConvShape& s, const __half* in, const __half* w, int Kpad, const float* scale, const float* shift,
             const __half* res, int relu, __half* out, cudaStream_t stream) {
  DIRB_REQUIRE(s.Cin % 8 == 0 && s.Cout % 64 == 0, DIRB200_ENOTSUP,
               "mma.sync conv needs Cin %% 8 == 0 and Cout %% 64 == 0 (got %d, %d)", s.Cin, s.Cout);
  MmaConvParams p{};
  p.in = in; p.w = w; p.scale = scale; p.shift = shift; p.res = res; p.out = out;
  p.B = s.B; p.H = s.H; p.W = s.W; p.Cin = s.Cin; p.Cout = s.Cout; p.KH = s.KH; p.KW = s.KW;
  p.stride = s.stride; p.pad = s.pad; p.Ho = s.Ho(); p.Wo = s.Wo();
  p.Ktot = s.KH * s.KW * s.Cin;
  p.Kpad = Kpad;
  DIRB_REQUIRE(Kpad % MM_BK == 0 && Kpad >= p.Ktot, DIRB200_EINVAL, "bad Kpad %d for K %d", Kpad, p.Ktot);
  p.M = s.B * p.Ho * p.Wo;
  p.relu = relu;
  dim3 grid((unsigned)ceil_div(p.M, MM_BM), (unsigned)(s.Cout / MM_BN));
  conv_mma_kernel<<<grid, 256, 0, stream>>>(p);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace dirb
