// Internal C++ interface of the convolution kernels (conv.cu) and the small fused operators (ops.cu).
#pragma once
#include <mutex>

#include "common.h"

namespace dirb {

// Ragged batch (net.cu): the extents of the images of one tensor at one resolution.  hw = image 0's {h, w}, image n's
// at hw + n * ld; n = images.  Kernels write 0 outside an image's extent and pool over its own pixels only.
// kc_major (optional, same stride): per-image flag for 3x3 stride-1 convolutions - where set, the image's K loop runs
// in the order of the HALO mode (conv_pers.cuh), elsewhere tap by tap; such launches never use the HALO kernel.
struct ConvExt {
  const int* hw;
  int ld, n;
  const int* kc_major;
  int slot_w;          // row length of the tensor in pixels (the head and center_bias walk an image's own pixels)
};

struct ConvShape {
  int B, H, W, Cin, Cout, KH, KW, stride, pad;
  int Ho() const { return (H + 2 * pad - KH) / stride + 1; }
  int Wo() const { return (W + 2 * pad - KW) / stride + 1; }
  double flops() const { return 2.0 * B * Ho() * Wo() * (double)Cout * KH * KW * Cin; }
};

// w: [Cout][KH*KW*Cin] fp16 (K index = (kh*KW + kw)*Cin + c).
int conv_tc(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
            const __half* res, int relu, __half* out, cudaStream_t stream, const ConvExt* ext = nullptr);
// conv3 of a block fused with its 1x1 projection shortcut (see conv.cu).
int conv_fused_ds(int B, int Ho, int Wo, int Cmid, const __half* t2, int Hx, int Wx, int Cx, int xstride,
                  const __half* x, const __half* wcat, int Cout, const float* scale, const float* shift, __half* out,
                  cudaStream_t stream, const ConvExt* ext = nullptr);
// conv2 (3x3/s1) + BN + ReLU + conv3 (1x1, x4) + BN + residual + ReLU of a Bottleneck in one kernel (conv_c23.cuh).
bool conv_c23_supported(int H, int W, int Cm);
bool conv_c23_profitable(int B, int H, int W, int Cm);
int conv_c23(int B, int H, int W, int Cm, const __half* t1, const __half* w2, const float* scale2, const float* shift2,
             const __half* w3, const float* scale3, const float* shift3, const __half* res, __half* out,
             cudaStream_t stream, const ConvExt* ext = nullptr);
// conv3 (1x1, x4) + BN + residual + ReLU of an identity Bottleneck and conv1 (1x1) + BN + ReLU of the identity
// Bottleneck after it in one kernel (conv_c31.cuh): y = block output, t1 = the next block's conv1 output.
bool conv_c31_supported(int Cm);
bool conv_c31_profitable(int B, int H, int W, int Cm);
int conv_c31(int B, int H, int W, int Cm, const __half* t2, const __half* w3, const float* scale3, const float* shift3,
             const __half* x, __half* y, const __half* w1, const float* scale1, const float* shift1, __half* t1,
             cudaStream_t stream, const ConvExt* ext = nullptr);
// The same wgmma kernel with one tile per CTA (no persistence), kept as an A/B baseline (impl 2).
int conv_tc_np(const ConvShape& s, const __half* in, const __half* w, const float* scale, const float* shift,
               const __half* res, int relu, __half* out, cudaStream_t stream, const ConvExt* ext = nullptr);
// w: [Cout][Kpad] fp16, Kpad = KH*KW*Cin rounded up to 32, zero padded.
int conv_mma(const ConvShape& s, const __half* in, const __half* w, int Kpad, const float* scale, const float* shift,
             const __half* res, int relu, __half* out, cudaStream_t stream);

int num_sms();
// Process-wide switch: 3x3/s1 convolutions with the input patch loaded once per channel block (1, default) or tap by tap (0).
void set_conv_halo(int on);
int get_conv_halo();
int get_head_fused();
int nchw_to_nhwc8(const float* in, int B, int H, int W, __half* out, cudaStream_t stream);

// Stem 7x7/s2/p3 (3 -> 64) + BN + ReLU on tensor cores (space-to-depth + mma.sync, conv.cu).  imgs: NCHW fp32; w2: [64][256] fp16 in the
// space-to-depth tap order (pack_stem_w2); s2d_ws: scratch of stem_workspace_bytes(B,H,W); out NHWC fp16 (B,Ho,Wo,64).
size_t stem_workspace_bytes(int B, int H, int W);
// imgs_u8 != nullptr: the input is uint8 HWC (B,H,W,3) and is normalised on the fly with mean_std = {mean[3], std[3]}.
// Ragged batch: in_ext = the pictures' extents in the input (pixels outside read as 0 after normalisation), out_ext =
// their extents in the stem's output.
int stem_tc(const float* imgs, int B, int H, int W, const __half* w2, const float* scale, const float* shift,
            __half* s2d_ws, __half* out, cudaStream_t stream, const uint8_t* imgs_u8 = nullptr,
            const float* mean_std = nullptr, const ConvExt* in_ext = nullptr, const ConvExt* out_ext = nullptr);
// The stem and the 3x3/s2 max-pool after it in one kernel (conv_stem.cuh), bit-identical to stem_tc + maxpool_3x3s2:
// fp32 imgs, or uint8 imgs_u8 with mean_std, -> out NHWC fp16 (B,Hp,Wp,64).  stem_out (optional) receives the stem
// map (B,Ho,Wo,64) before pooling.  Ragged batch: the pictures' extents in the input, the stem map and the pooled map
// (rows of one table, one stride).
int stem_pool(const float* imgs, const uint8_t* imgs_u8, const float* mean_std, int B, int H, int W, const __half* w2,
              const float* scale, const float* shift, __half* out, __half* stem_out, cudaStream_t stream,
              const ConvExt* in_ext = nullptr, const ConvExt* stem_ext = nullptr, const ConvExt* pool_ext = nullptr);
// OIHW fp32 [64][3][7][7] -> [64][256] fp16 (host).
void pack_stem_w2(const float* w_oihw, __half* out);
int maxpool_3x3s2(const __half* in, int B, int H, int W, int C, __half* out, cudaStream_t stream,
                  const ConvExt* ext = nullptr);

size_t head_workspace_floats(int B, int HW, int C, int out_dim);
int head_pool_fc_l2(const __half* feat, int B, int HW, int C, int pooling, float p, float eps, int norm_features,
                    const float* fc_w, const float* fc_b, int out_dim, float* ws, float* desc, __half* desc16,
                    cudaStream_t stream, unsigned int* bar = nullptr, const ConvExt* ext = nullptr);
void set_head_fused(int on);   // 1 (default) = the plain head is ONE persistent kernel, 0 = one kernel per phase

// The pieces of head_pool_fc_l2, for heads that pool several maps side by side (FPN): see ops.cu.
int head_pool(const __half* feat, int B, int HW, int C, int pooling, float p, float eps, int norm_features, float* partial,
              float* g, int g_ld, int col_off, cudaStream_t stream, const ConvExt* ext = nullptr);
int head_fc_l2(const float* g, int B, int C, const float* fc_w, const float* fc_b, int out_dim, float* y, float* desc,
               __half* desc16, cudaStream_t stream);
size_t head_partial_floats(int B, int HW, int C);
// x4 += nearest-upsampled t (FPN lateral connection, rmac_resnet_fpn.py:56-60); NHWC fp16, out may alias x4.
int upsample_add(const __half* x4, const __half* t, __half* out, int B, int H, int W, int h, int w, int C,
                 cudaStream_t stream);

int pool_scales(const float* xs, int S, int64_t N, int D, int mode, float gemp, int l2, float* out,
                cudaStream_t stream);
int l2_normalize(const float* x, int64_t N, int D, float eps, float* out, __half* out16, cudaStream_t stream);
int center_bias(__half* x, int B, int H, int W, int C, float b, cudaStream_t stream, const ConvExt* ext = nullptr);
int f32_to_f16(const float* x, int64_t n, __half* out, cudaStream_t stream);
int whiten(const float* x, int64_t N, int D, const float* comp, const float* mean, const float* colscale, int Dout,
           int l2norm, float* y, __half* y16, cudaStream_t stream);

// Lease on the per-device scratch buffer kept for the life of the process (ops.cu).  acquire takes the device's
// scratch mutex, grows the buffer to `bytes` and orders `stream` after the previous lease's work; the mutex is held
// until the lease goes out of scope, whose destructor records the end of this stream's use on every return path
// (including errors after kernels were enqueued).  Enqueue all work on the buffer while the lease is alive.
class ScratchLease {
 public:
  ScratchLease() = default;
  ScratchLease(const ScratchLease&) = delete;
  ScratchLease& operator=(const ScratchLease&) = delete;
  ~ScratchLease();
  int acquire(size_t bytes, cudaStream_t stream, void** out);

 private:
  std::unique_lock<std::mutex> lock_;
  cudaEvent_t last_use_ = nullptr;
  cudaStream_t stream_ = nullptr;
};

}  // namespace dirb
