// extern "C" wrappers of the single operators (include/dirb200.h); the handle-based entry points live next to
// their implementation (net.cu, search.cu, common.cu).
#include "conv.h"

using namespace dirb;

#define ST(s) static_cast<cudaStream_t>(s)
#define H16(p) static_cast<__half*>(p)
#define CH16(p) static_cast<const __half*>(p)

extern "C" {

int dirb200_nchw_to_nhwc8(const float* in_dev, int B, int H, int W, void* out_dev, void* stream) {
  DIRB_REQUIRE(in_dev && out_dev && B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad arguments");
  return nchw_to_nhwc8(in_dev, B, H, W, H16(out_dev), ST(stream));
}

int dirb200_conv_bn_act(const void* in_dev, int B, int H, int W, int Cin, const void* w_dev, int Cout, int KH, int KW,
                        int stride, int pad, const float* scale_dev, const float* shift_dev, const void* res_dev,
                        int relu, int impl, void* out_dev, void* stream) {
  DIRB_REQUIRE(in_dev && w_dev && scale_dev && shift_dev && out_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(B > 0 && H > 0 && W > 0 && KH > 0 && KW > 0 && stride > 0 && pad >= 0, DIRB200_EINVAL, "bad shape");
  ConvShape s{B, H, W, Cin, Cout, KH, KW, stride, pad};
  DIRB_REQUIRE(s.Ho() > 0 && s.Wo() > 0, DIRB200_EINVAL, "empty output");
  if (impl == 0) return conv_tc(s, CH16(in_dev), CH16(w_dev), scale_dev, shift_dev, CH16(res_dev), relu, H16(out_dev), ST(stream));
  if (impl == 2) return conv_tc_np(s, CH16(in_dev), CH16(w_dev), scale_dev, shift_dev, CH16(res_dev), relu, H16(out_dev), ST(stream));
  const int K = KH * KW * Cin;
  return conv_mma(s, CH16(in_dev), CH16(w_dev), (K + 31) / 32 * 32, scale_dev, shift_dev, CH16(res_dev), relu,
                  H16(out_dev), ST(stream));
}

int dirb200_conv_c23(const void* t1_dev, int B, int H, int W, int Cm, const void* w2_dev, const float* scale2_dev,
                     const float* shift2_dev, const void* w3_dev, const float* scale3_dev, const float* shift3_dev,
                     const void* res_dev, void* out_dev, int variant, void* stream) {
  DIRB_REQUIRE(t1_dev && w2_dev && w3_dev && scale2_dev && shift2_dev && scale3_dev && shift3_dev && res_dev && out_dev,
               DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad shape");
  (void)variant;   // CTA-pair variant of the sm_100a build; sm_90a has the single-CTA kernel only
  return conv_c23(B, H, W, Cm, CH16(t1_dev), CH16(w2_dev), scale2_dev, shift2_dev, CH16(w3_dev), scale3_dev, shift3_dev,
                  CH16(res_dev), H16(out_dev), ST(stream));
}

int dirb200_conv_c31(const void* t2_dev, int B, int H, int W, int Cm, const void* w3_dev, const float* scale3_dev,
                     const float* shift3_dev, const void* x_dev, void* y_dev, const void* w1_dev, const float* scale1_dev,
                     const float* shift1_dev, void* t1_dev, void* stream) {
  DIRB_REQUIRE(t2_dev && w3_dev && scale3_dev && shift3_dev && x_dev && y_dev && w1_dev && scale1_dev && shift1_dev && t1_dev,
               DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad shape");
  return conv_c31(B, H, W, Cm, CH16(t2_dev), CH16(w3_dev), scale3_dev, shift3_dev, CH16(x_dev), H16(y_dev), CH16(w1_dev),
                  scale1_dev, shift1_dev, H16(t1_dev), ST(stream));
}

size_t dirb200_stem_workspace_bytes(int B, int H, int W) { return stem_workspace_bytes(B, H, W); }

int dirb200_stem_pack_weight(const float* w_oihw_host, void* w2_host) {
  DIRB_REQUIRE(w_oihw_host && w2_host, DIRB200_EINVAL, "null argument");
  pack_stem_w2(w_oihw_host, static_cast<__half*>(w2_host));
  return 0;
}

int dirb200_stem_conv(const float* imgs_dev, int B, int H, int W, const void* w2_dev, const float* scale_dev,
                      const float* shift_dev, void* ws_dev, void* out_dev, void* stream) {
  DIRB_REQUIRE(imgs_dev && w2_dev && scale_dev && shift_dev && ws_dev && out_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(B > 0 && H >= 7 && W >= 7, DIRB200_EINVAL, "bad shape");
  return stem_tc(imgs_dev, B, H, W, CH16(w2_dev), scale_dev, shift_dev, H16(ws_dev), H16(out_dev), ST(stream));
}

int dirb200_stem_pool(const void* imgs_dev, int is_u8, int B, int H, int W, const float* mean_std_host, const void* w2_dev,
                      const float* scale_dev, const float* shift_dev, void* out_dev, void* stem_dev, void* stream) {
  DIRB_REQUIRE(imgs_dev && w2_dev && scale_dev && shift_dev && out_dev && (!is_u8 || mean_std_host), DIRB200_EINVAL,
               "null argument");
  DIRB_REQUIRE(B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad shape");
  return stem_pool(is_u8 ? nullptr : static_cast<const float*>(imgs_dev), is_u8 ? static_cast<const uint8_t*>(imgs_dev) : nullptr,
                   mean_std_host, B, H, W, CH16(w2_dev), scale_dev, shift_dev, H16(out_dev), H16(stem_dev), ST(stream));
}

int dirb200_maxpool_3x3s2(const void* in_dev, int B, int H, int W, int C, void* out_dev, void* stream) {
  DIRB_REQUIRE(in_dev && out_dev && B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad arguments");
  return maxpool_3x3s2(CH16(in_dev), B, H, W, C, H16(out_dev), ST(stream));
}

size_t dirb200_head_workspace_floats(int B, int HW, int C, int out_dim) { return head_workspace_floats(B, HW, C, out_dim); }

int dirb200_head_pool_fc_l2(const void* feat_dev, int B, int HW, int C, int pooling, float p, float eps,
                            int norm_features, const float* fc_w_dev, const float* fc_b_dev, int out_dim, float* ws_dev,
                            float* desc_dev, void* desc16_dev, void* stream) {
  DIRB_REQUIRE(feat_dev && ws_dev && desc_dev && B > 0 && HW > 0, DIRB200_EINVAL, "bad arguments");
  return head_pool_fc_l2(CH16(feat_dev), B, HW, C, pooling, p, eps, norm_features, fc_w_dev, fc_b_dev,
                         fc_w_dev ? out_dim : C, ws_dev, desc_dev, H16(desc16_dev), ST(stream));
}

int dirb200_center_bias(void* feat_dev, int B, int H, int W, int C, float b, void* stream) {
  DIRB_REQUIRE(feat_dev && B > 0 && H > 0 && W > 0, DIRB200_EINVAL, "bad arguments");
  return center_bias(H16(feat_dev), B, H, W, C, b, ST(stream));
}

int dirb200_pool_scales(const float* xs_dev, int S, int64_t N, int D, int mode, float gemp, int l2, float* out_dev,
                        void* stream) {
  DIRB_REQUIRE(xs_dev && out_dev, DIRB200_EINVAL, "null argument");
  return pool_scales(xs_dev, S, N, D, mode, gemp, l2, out_dev, ST(stream));
}

int dirb200_l2_normalize(const float* x_dev, int64_t N, int D, float eps, float* out_dev, void* out16_dev, void* stream) {
  DIRB_REQUIRE(x_dev && (out_dev || out16_dev), DIRB200_EINVAL, "null argument");
  return l2_normalize(x_dev, N, D, eps, out_dev, H16(out16_dev), ST(stream));
}

int dirb200_whiten(const float* x_dev, int64_t N, int D, const float* comp_dev, const float* mean_dev,
                   const float* colscale_dev, int Dout, int l2norm, float* y_dev, void* y16_dev, void* stream) {
  DIRB_REQUIRE(x_dev && comp_dev && y_dev && Dout > 0, DIRB200_EINVAL, "bad arguments");
  return whiten(x_dev, N, D, comp_dev, mean_dev, colscale_dev, Dout, l2norm, y_dev, H16(y16_dev), ST(stream));
}

int dirb200_f32_to_f16(const float* x_dev, int64_t n, void* out16_dev, void* stream) {
  DIRB_REQUIRE(x_dev && out16_dev, DIRB200_EINVAL, "null argument");
  return f32_to_f16(x_dev, n, H16(out16_dev), ST(stream));
}

}  // extern "C"
