/* dirb200 - C ABI of the H100-native (sm_90a) descriptor-extraction + retrieval hot path.
 *
 * The reference (naver/deep-image-retrieval, "dirtorch") has no FFI: its boundary is a Python
 * duck-type (SURVEY.md 8b).  This header is the boundary a binding for that path would target:
 * plain C types, raw device/host pointers + sizes, a CUDA stream as void*, no torch types.
 * Each entry point names the reference call it replaces (file:line relative to the reference).
 *
 * Conventions
 *   - every function returns 0 on success, a negative DIRB200_E* code for library errors, or a
 *     positive cudaError_t; dirb200_last_error() returns a thread-local message;
 *   - "dev" pointers are device memory owned by the caller; the library allocates only inside
 *     opaque handles (packed weights, workspaces) freed by the matching *_destroy;
 *   - all launches are asynchronous on the given stream unless the name ends in _host;
 *   - create, finalize and set calls (no stream argument) have finished on the device when they
 *     return: their results may be used at once from any stream, blocking or not;
 *   - a handle is bound to one device and is not re-entrant (one handle per GPU / stream);
 *   - there is NO CPU fallback: on a machine without an sm_90 device every compute entry
 *     point fails with DIRB200_ENODEVICE.
 */
#ifndef DIRB200_H_
#define DIRB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DIRB200_OK 0
#define DIRB200_EINVAL (-1)    /* bad argument                                            */
#define DIRB200_ENOTSUP (-2)   /* shape / option outside what the kernels support          */
#define DIRB200_EDRIVER (-3)   /* driver entry point (cuTensorMapEncodeTiled) unavailable  */
#define DIRB200_EOVERFLOW (-4) /* candidate buffer overflow that could not be resolved     */
#define DIRB200_ESTATE (-5)    /* handle used in the wrong state                           */
#define DIRB200_ENODEVICE (-6) /* no sm_90 CUDA device                                     */
#define DIRB200_EKEY (-7)      /* unknown tensor / option name                             */

typedef struct dirb200_net dirb200_net;     /* one ResNet-GeM network on one GPU            */
typedef struct dirb200_index dirb200_index; /* one row-shard of a descriptor database       */
typedef struct dirb200_exchange dirb200_exchange; /* this rank's window of the peer-memory exchange of a sharded search */

int dirb200_version(void);
const char* dirb200_last_error(void);
/* 0 if `device` exists and is compute capability 10.x. */
int dirb200_device_check(int device);

/* ------------------------------------------------------------------ network (extraction)
 * Replaces nets.create_model(arch, **model_options) + net.load_state_dict(sd) + net(imgs):
 * dirtorch/nets/__init__.py:24-64, dirtorch/nets/rmac_resnet.py:12-69,
 * dirtorch/nets/backbones/resnet.py:46-87,102-174, dirtorch/nets/layers/pooling.py:38-54.   */

/* Process-wide kernel selectors (they pick which kernel a launcher uses; no reference counterpart - the reference
 * delegates kernel choice to torch.backends.cudnn, utils/common.py:74-75 cudnn.benchmark / cudnn.fastest).  Set them once,
 * not concurrently with a running call: "pdl" 1 (default) = programmatic dependent launch between consecutive
 * kernels; "head_fused" 1 (default) = pooling + FC + L2 of the plain head as ONE persistent kernel, 0 = one kernel per
 * phase (bit-identical results); "halo" 1 (default) / 0 = 3x3 stride-1 convolutions load their input patch once per
 * 64-channel block and read the nine taps as views of it, or load one box per tap.
 * dirb200_net_set_option forwards these keys here. */
int dirb200_set_global_option(const char* key, double value);
int dirb200_get_global_option(const char* key, double* value);
/* arch: "resnet50_rmac" | "resnet101_rmac" | "resnet152_rmac" (Bottleneck trunks, rmac_resnet.py:78-88). */
int dirb200_net_create(const char* arch, int device, dirb200_net** out);
/* Options.
 * Model options of rmac_resnet.py:15-37 (the three marked * must be set BEFORE dirb200_net_finalize, later
 * changes return DIRB200_ESTATE): "pooling"* 0=gem 1=max 2=avg; "without_fc"* 0/1; "out_dim"*; "norm_features" 0/1;
 * "center_bias" b >= 0 (rmac_resnet.py:52-56); "gem_eps" (pooling.py:39, default 1e-6);
 * "mean0".."mean2", "std0".."std2": Normalize constants of the uint8 entry points (default resnet.py:110-111).
 * Scheduling: "chunk" images per pass of the network (0 = auto); "host_chunk" images per pipeline stage of
 * dirb200_net_forward_host (default 16).
 * Implementation A/B switches: "conv_impl" 0 = persistent wgmma implicit GEMM (default), 1 = mma.sync implicit
 * GEMM (validation path), 2 = the same kernel with one tile per CTA (baseline); "fuse_ds" 1 (default) = projection
 * shortcut fused into conv3 as a K-concatenated GEMM; "fuse_c23" 0 (default) / 1 / 2 = conv2 + conv3 (+ residual) of the
 * identity blocks with 64 / 128 / 256 mid channels as one kernel (dirb200_conv_c23): never / where every SM gets at least
 * two tiles / wherever the kernel supports the shape; "fuse_stem" 1 (default) = stem convolution + maxpool as one kernel
 * (dirb200_stem_pool; conv_impl 0 and 2), 0 = space-to-depth, convolution and maxpool as three launches.  PROCESS-WIDE (they select kernels, not handle state; set them
 * once, not concurrently with a running forward): the global options above.
 * Diagnostics: "debug_taps" 1 = keep copies of the stage outputs for dirb200_net_debug_stage; "profile" 1 = time
 * every launch with CUDA events (dirb200_net_profile). */
int dirb200_net_set_option(dirb200_net* net, const char* key, double value);
/* One state_dict tensor by its reference key ("layer3.5.bn2.running_var", "adpool.p", "fc.weight" ...),
 * fp32 host memory, reference shape (conv OIHW).  "num_batches_tracked" keys are ignored. */
int dirb200_net_set_tensor(dirb200_net* net, const char* name, const float* host_data, const int64_t* shape,
                           int ndim);
/* Fold BN into per-channel scale/shift, repack conv weights to [Cout][KH][KW][Cin] fp16, upload. */
int dirb200_net_finalize(dirb200_net* net);
/* net(imgs): imgs_dev = NCHW fp32 normalised images (B,3,H,W); desc_dev = (B,out_dim) fp32 L2-normalised
 * descriptors; desc16_dev (optional, may be NULL) = the same in fp16.  test_dir.py:74. */
int dirb200_net_forward(dirb200_net* net, const float* imgs_dev, int B, int H, int W, float* desc_dev,
                        void* desc16_dev, void* stream);
/* Same through HOST buffers: H2D copy of the images, forward, D2H copy of the descriptors, stream sync
 * (the common.variables() -> net() -> tonumpy() sequence, common.py:205-218,23-27).  The batch is processed in
 * chunks of "host_chunk" images (option, default 16) with the H2D copy of the next chunk overlapping the compute
 * of the current one; pass pinned memory for the overlap to take effect. */
int dirb200_net_forward_host(dirb200_net* net, const float* imgs_host, int B, int H, int W, float* desc_host);
/* uint8 input (what an image decoder yields): imgs = HWC uint8 pixels (B,H,W,3); ToTensor + Normalize(mean,std)
 * (dirtorch/utils/transforms.py:27; options "mean0".."mean2", "std0".."std2", default = ImageNet values of
 * resnet.py:110-111) are applied on the fly in the stem's input stage, bit-identically to the fp32 entry points.
 * 4x fewer host->device bytes than the fp32 path (SURVEY.md 8f rank 1, first step). */
int dirb200_net_forward_u8(dirb200_net* net, const uint8_t* imgs_dev, int B, int H, int W, float* desc_dev,
                           void* desc16_dev, void* stream);
int dirb200_net_forward_host_u8(dirb200_net* net, const uint8_t* imgs_host, int B, int H, int W, float* desc_host);
/* Ragged batch: B images of different sizes in one network pass (test_dir.py:47-94 feeds them one per call,
 * test_dir.py:52-53).  Image i (hw_host[i] = {h_i, w_i}, host memory) sits in the top-left corner of slot i of one
 * (H, W) slot tensor: uint8 HWC (B,H,W,3) for the _u8 entry point, normalised NCHW fp32 (B,3,H,W) for the other.
 * Slot content outside the images is ignored, whatever it holds.  Every activation outside an image's extent is 0
 * and the head pools over the image's own pixels, so desc_dev row i (and desc16_dev, optional) equals, bit for bit,
 * the descriptor of a B = 1 forward of image i alone.  Needs 32 <= h_i <= H and 32 <= w_i <= W (else
 * DIRB200_EINVAL); FPN heads and conv_impl 1 return DIRB200_ENOTSUP. */
int dirb200_net_forward_ragged_u8(dirb200_net* net, const uint8_t* slots_dev, int B, int H, int W, const int* hw_host,
                                  float* desc_dev, void* desc16_dev, void* stream);
int dirb200_net_forward_ragged(dirb200_net* net, const float* slots_dev, int B, int H, int W, const int* hw_host,
                               float* desc_dev, void* desc16_dev, void* stream);
/* Bilinear resize of uint8 HWC RGB images (B,H,W,3) -> (B,Ho,Wo,3), byte-identical to PIL's
 * Image.resize((Wo,Ho), Image.BILINEAR) - the `Scale` transform of dirtorch/utils/transforms.py:133-185 - so that
 * multi-scale extraction (Scale(0.7), Scale(1.4)) can stay on the GPU in front of dirb200_net_forward_u8.
 * dirb200_resize_coeffs is the host-only coefficient table of one axis (bounds_out [2*out], kk_out [out*ksize];
 * call with kk_out == NULL to query ksize). */
int dirb200_resize_bilinear_u8(const uint8_t* in_dev, int B, int H, int W, int Ho, int Wo, uint8_t* out_dev, void* stream);
int dirb200_resize_coeffs(int in_size, int out_size, int* bounds_out, int* kk_out, int* ksize_out);
/* ------------------------------------------------------------------ baseline JPEG decoding
 * Replaces Image.open(f).convert("RGB") (dirtorch/datasets/dataset.py:52, dirtorch/datasets/generic.py:246) for
 * baseline JPEGs: the RGB pixels equal, byte for byte, what PIL (libjpeg-turbo, default ISLOW IDCT, fancy upsampling)
 * returns.  Supported: 8-bit baseline / extended-sequential Huffman, one interleaved scan of all components, 1 component
 * (grey, replicated to RGB) or 3 with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1, any restart interval.
 * dirb200_jpeg_probe (host only) parses the markers: info = {height, width, components, luma h-sampling, luma
 * v-sampling, restart interval, colour (0 YCbCr, 1 RGB, 2 grey), entropy-coded bytes}; returns 0 if the decoder takes
 * the file, DIRB200_ENOTSUP for a well-formed JPEG it does not (progressive, arithmetic, 12-bit, CMYK, multi-scan,
 * other sampling, DNL, Huffman tables with an all-ones code) and DIRB200_EINVAL for anything else (not a JPEG,
 * truncated, malformed).
 * The decoder handle owns pinned staging and device workspace, grown on demand.  dirb200_jpeg_decoder_decode decodes n images
 * (host buffers data_host[i] of sizes_host[i] bytes) in one upload: image i goes to out_dev + out_offsets_host[i] as
 * (h, w, 3) uint8 and status_dev[i] (device int32) is 0 when it was decoded; non-zero: the probe's code for files the
 * host parser refused, or a positive mask (1 marker in the scan, 2 restart markers, 4 block count of a restart segment, 8 invalid code)
 * when the entropy-coded data does not decode cleanly - the caller decodes such a file with PIL.  rounds_out (may be
 * NULL) = synchronisation rounds that changed a state.  Waits on the stream once per four synchronisation rounds.
 * Option "subseq_bits" (default 1024, multiple of 32 in [64, 2^20]): bits per subsequence of the parallel Huffman
 * decode.  dirb200_jpeg_debug_coefficients copies image `image` of the last decode's coefficients, int16 [nblocks][64]
 * in natural order, blocks in MCU order, DC prediction applied (dst_dev = NULL: *nblocks only). */
int dirb200_jpeg_probe(const uint8_t* data, size_t size, int info[8]);
typedef struct dirb200_jpeg_decoder dirb200_jpeg_decoder;
int dirb200_jpeg_decoder_create(int device, dirb200_jpeg_decoder** out);
int dirb200_jpeg_decoder_set_option(dirb200_jpeg_decoder* dec, const char* key, double value);
int dirb200_jpeg_decoder_decode(dirb200_jpeg_decoder* dec, int n, const uint8_t* const* data_host, const size_t* sizes_host,
                        uint8_t* out_dev, const int64_t* out_offsets_host, int* status_dev, int* rounds_out, void* stream);
int dirb200_jpeg_debug_coefficients(dirb200_jpeg_decoder* dec, int image, int16_t* dst_dev, size_t capacity, int* nblocks,
                                    void* stream);
int dirb200_jpeg_decoder_destroy(dirb200_jpeg_decoder* dec);
/* Debug tap (needs option "debug_taps"): copy the NHWC fp16 activation `what` of the LAST chunk of the last forward
 * into dst_dev (capacity in bytes); returns its dims as {n,h,w,c}.  Names: "stem_conv" (stem convolution, before the
 * maxpool), "stem" (after it), "layerL.B.conv1" / "layerL.B.conv2" / "layerL.B.down" (outputs of block B of layer L,
 * L = 1..4, as in the state-dict keys; conv2 only where it reaches memory, i.e. not inside conv_c23, and down only
 * where the projection shortcut is not fused into conv3), "layerL.B" (block output), "layer1".."layer4" (stage
 * outputs), and for FPN heads "fpn_lat" (conv1x5), "fpn_merge" (after the upsample-add) and "fpn_c4" (conv3c4). */
int dirb200_net_debug_stage(dirb200_net* net, const char* what, void* dst_dev, size_t capacity, int dims[4],
                            void* stream);
/* Per-class CUDA-event timing of the last forward run with option "profile" = 1: out16 = 4 rows of
 * {launches, milliseconds, algorithmic FLOPs, algorithmic bytes} for 0 wgmma convolutions, 1 stem convolution,
 * 2 layout + maxpool, 3 head.  Synchronises the device. */
int dirb200_net_profile(dirb200_net* net, double* out16);
/* Option "profile" = 1 (next forward) or 2 (accumulate over forwards until the option is set again): per launch TYPE
 * (e.g. "1x1 256->1024 +res @64x64") the launches, CUDA-event milliseconds, algorithmic FLOPs and bytes, as JSON text.
 * Two-call protocol: buf = NULL returns the size through *needed. */
int dirb200_net_profile_table(dirb200_net* net, char* buf, size_t cap, size_t* needed);
/* Number of kernels the last forward launched / algorithmic conv+fc FLOPs of the last forward. */
int dirb200_net_last_launches(dirb200_net* net, int64_t* launches, double* flops);
int dirb200_net_destroy(dirb200_net* net);

/* ------------------------------------------------------------------ single operators
 * (the building blocks of the network, exported for parity tests and reuse)                 */

/* NCHW fp32 (B,3,H,W) -> NHWC fp16 (B,H,W,8), channels 3..7 zero.  Input staging of resnet.py:158. */
int dirb200_nchw_to_nhwc8(const float* in_dev, int B, int H, int W, void* out_dev, void* stream);
/* Conv2d(bias=False) + folded BatchNorm (+ residual add) (+ ReLU), NHWC fp16 in/out.
 * w_dev: [Cout][KH][KW][Cin] fp16; scale/shift: [Cout] fp32; res_dev may be NULL.
 * impl: 0 persistent wgmma (needs Cin%64==0, Cout%64==0), 1 mma.sync (needs Cin%8==0, Cout%64==0), 2 one-tile-per-CTA wgmma.
 * resnet.py:56-63,70-85,115-118. */
int dirb200_conv_bn_act(const void* in_dev, int B, int H, int W, int Cin, const void* w_dev, int Cout, int KH,
                        int KW, int stride, int pad, const float* scale_dev, const float* shift_dev,
                        const void* res_dev, int relu, int impl, void* out_dev, void* stream);
/* conv2 + conv3 of a Bottleneck in one kernel (resnet.py:75-85): out = relu(bn3(conv1x1(relu(bn2(conv3x3(t1))))) + res).
 * t1 NHWC fp16 (B,H,W,Cm), w2 [Cm][3][3][Cm] fp16, w3 [4*Cm][Cm] fp16 (the layouts of dirb200_conv_bn_act), res / out
 * NHWC fp16 (B,H,W,4*Cm).  Cm in {64, 128, 256}, H >= 16, W >= 8, stride 1.  The conv2 output stays in shared memory as the
 * A operand of conv3 (fp16, the same rounding as the two-kernel path, whose result it equals bit for bit).  `variant`
 * selected CTA pairs in the sm_100a build; the sm_90a build has one variant and ignores it. */
int dirb200_conv_c23(const void* t1_dev, int B, int H, int W, int Cm, const void* w2_dev, const float* scale2_dev,
                     const float* shift2_dev, const void* w3_dev, const float* scale3_dev, const float* shift3_dev,
                     const void* res_dev, void* out_dev, int variant, void* stream);
/* conv3 of an identity Bottleneck and conv1 of the identity Bottleneck after it in one kernel (resnet.py:75-85):
 * y = relu(bn3(conv1x1(t2)) + x), t1 = relu(bn1(conv1x1(y))).  t2 NHWC fp16 (B,H,W,Cm), w3 [4*Cm][Cm] fp16, x / y NHWC
 * fp16 (B,H,W,4*Cm), w1 [Cm][4*Cm] fp16 (the layouts of dirb200_conv_bn_act), t1 NHWC fp16 (B,H,W,Cm).  Cm in
 * {64, 128, 256}.  conv1 reads y from shared memory; y and t1 equal the two dirb200_conv_bn_act launches bit for bit. */
int dirb200_conv_c31(const void* t2_dev, int B, int H, int W, int Cm, const void* w3_dev, const float* scale3_dev,
                     const float* shift3_dev, const void* x_dev, void* y_dev, const void* w1_dev, const float* scale1_dev,
                     const float* shift1_dev, void* t1_dev, void* stream);
/* The stem on tensor cores: Conv2d(3, 64, 7, stride 2, pad 3, bias=False) + folded BN + ReLU, resnet.py:115-118.
 * imgs_dev NCHW fp32 (B,3,H,W); w2_dev = the [64][256] fp16 weight layout produced (on the host) by
 * dirb200_stem_pack_weight from the OIHW fp32 [64][3][7][7] tensor; ws_dev scratch of
 * dirb200_stem_workspace_bytes(B,H,W) bytes; out_dev NHWC fp16 (B,Ho,Wo,64). */
size_t dirb200_stem_workspace_bytes(int B, int H, int W);
int dirb200_stem_pack_weight(const float* w_oihw_host, void* w2_host);
int dirb200_stem_conv(const float* imgs_dev, int B, int H, int W, const void* w2_dev, const float* scale_dev,
                      const float* shift_dev, void* ws_dev, void* out_dev, void* stream);
/* The stem and the max-pool after it (resnet.py:115-119) in one kernel that reads the images and writes the pooled map,
 * bit-identical to dirb200_stem_conv + dirb200_maxpool_3x3s2.  imgs_dev NCHW fp32 (B,3,H,W) (is_u8 0) or HWC uint8
 * (B,H,W,3) (is_u8 1, ToTensor + Normalize with mean_std_host = {mean[3], std[3]}); w2_dev as for dirb200_stem_conv;
 * out_dev NHWC fp16 (B,Hp,Wp,64); stem_dev (may be NULL) receives the stem map (B,Ho,Wo,64) before pooling. */
int dirb200_stem_pool(const void* imgs_dev, int is_u8, int B, int H, int W, const float* mean_std_host, const void* w2_dev,
                      const float* scale_dev, const float* shift_dev, void* out_dev, void* stem_dev, void* stream);
/* MaxPool2d(3, stride 2, pad 1) on NHWC fp16.  resnet.py:119,161. */
int dirb200_maxpool_3x3s2(const void* in_dev, int B, int H, int W, int C, void* out_dev, void* stream);
/* Global pooling + (L2 over C) + FC + L2: rmac_resnet.py:59-68, pooling.py:38-40.
 * feat_dev NHWC fp16 (B,h,w,C); pooling 0 gem(p, eps) / 1 max / 2 avg; fc_w_dev [out_dim][C] fp32 (NULL = without_fc);
 * ws_dev: fp32 scratch of dirb200_head_workspace_floats(B,h*w,C,out_dim) floats. */
size_t dirb200_head_workspace_floats(int B, int HW, int C, int out_dim);
int dirb200_head_pool_fc_l2(const void* feat_dev, int B, int HW, int C, int pooling, float p, float eps,
                            int norm_features, const float* fc_w_dev, const float* fc_b_dev, int out_dim,
                            float* ws_dev, float* desc_dev, void* desc16_dev, void* stream);

/* center_bias option, rmac_resnet.py:52-56: feat[n][h][w][:] *= 1 + bilinear(align_corners) resize to (H,W) of the
 * 4x4 map holding b on its central 2x2; in place on the NHWC fp16 map that feeds the global pooling. */
int dirb200_center_bias(void* feat_dev, int B, int H, int W, int C, float b, void* stream);

/* ------------------------------------------------------------------ descriptor post-processing */

/* common.pool + F.normalize: common.py:41-55, test_dir.py:121-122.  xs_dev: (S,N,D) fp32 stacked;
 * mode 0 mean, 1 gem (signed power gemp); l2 != 0 appends the row L2 normalisation. */
int dirb200_pool_scales(const float* xs_dev, int S, int64_t N, int D, int mode, float gemp, int l2, float* out_dev,
                        void* stream);
/* Row L2 normalisation, eps as F.normalize (1e-12). */
int dirb200_l2_normalize(const float* x_dev, int64_t N, int D, float eps, float* out_dev, void* out16_dev,
                         void* stream);
/* common.whiten_features: common.py:221-239.  Y = ((X - mean) . comp^T) * colscale, optional row L2.
 * comp_dev [Dout][D] fp32 (pca.components_[:whitenv]); mean_dev [D] or NULL; colscale_dev [Dout] =
 * 1 / (whitenm * explained_variance_^whitenp) or NULL; y16_dev optional fp16 copy. */
int dirb200_whiten(const float* x_dev, int64_t N, int D, const float* comp_dev, const float* mean_dev,
                   const float* colscale_dev, int Dout, int l2norm, float* y_dev, void* y16_dev, void* stream);
int dirb200_f32_to_f16(const float* x_dev, int64_t n, void* out16_dev, void* stream);

/* ------------------------------------------------------------------ similarity + top-k
 * Replaces scores = common.matmul(q, db) (common.py:30-38, test_dir.py:145) followed by the per-query
 * ranking (generic.py:207,221; dataset.py:100; test_dir.py:36) for the first k ranks.  Ordering: exact
 * (fp64-accumulated) dot product of the fp32 rows, descending; ties -> lower index first.               */

int dirb200_index_create(int device, int dim, dirb200_index** out);
/* Attach one row shard: db32_dev [N][dim] fp32 (exact re-scoring), db16_dev [N][dim] fp16 (tensor-core pass);
 * both caller-owned and must outlive the index.  index_offset is added to every returned index
 * (row-wise sharding across GPUs, SURVEY.md 8e). */
int dirb200_index_set_db(dirb200_index* idx, const float* db32_dev, const void* db16_dev, int64_t N,
                         int64_t index_offset);
/* "eps16": bound on |fp16-path score - exact score| used for the candidate band (default 1.2e-3, valid for
 * unit-norm rows); "sample_rows": rows scored densely to seed the threshold (0 = auto); "cand_cap": per-query
 * candidate-list capacity (0 = auto; a small value forces the overflow -> tightened re-run path); "retries": gated
 * retry passes enqueued after the filter pass (default 1; they return at once unless a list overflowed);
 * "deferred_check" = 1: search calls never synchronise the host, the caller collects the status with
 * dirb200_index_check (it is also collected at the start of the next search); "profile"; "count_eps" / "band_cap":
 * see dirb200_index_count_ge; "ws_budget": bytes of search workspace a call may use (default 4 GiB), which sets the
 * largest query block (dirb200_index_search_max_queries). */
int dirb200_index_set_option(dirb200_index* idx, const char* key, double value);
/* q32_dev [Q][dim] fp32, any Q >= 1, 1 <= k <= 2^27.  Outputs (device): scores_dev [Q][k] fp64 exact scores, idx_dev
 * [Q][k] int64.  If N < k the tail is filled with score -inf / index -1.  k <= 1024 re-scores and sorts the survivors
 * of each query in shared memory (at most 1024 survivors for k <= 256, 2048 above); k > 1024 keeps them in global
 * memory (at most min(2k, N) per query) and orders them with sorted runs and a rank-based merge.  Queries run in blocks
 * of dirb200_index_search_max_queries(k).  Everything is enqueued on `stream`; the call then waits once per block for
 * the status block (overflow that the device-side retries could not resolve, or more survivors than the limit above ->
 * DIRB200_EOVERFLOW) unless option "deferred_check" is set. */
int dirb200_index_search(dirb200_index* idx, const float* q32_dev, int Q, int k, double* scores_dev,
                         int64_t* idx_dev, void* stream);
/* Largest Q that one dirb200_index_search_begin of depth k accepts: its workspace (fp16 queries, seed scores, candidate
 * and survivor lists, all proportional to Q and growing with k) must fit option "ws_budget".  At least 1; at most 65535
 * when the search keeps one grid row per query (k > 1024, or N within the dense seed sample). */
int dirb200_index_search_max_queries(dirb200_index* idx, int k, int* q_max);
/* The same search in two phases, for a database sharded over several GPUs.  Phase 1 runs the tensor-core passes and
 * writes to sel_dev[Q] (caller-owned) the local min(k_shard, N_local)-th best fp16-path score per query (+inf for an
 * empty shard).  The caller MIN-reduces sel_dev over the shards (ncclAllReduce, 4*Q bytes): shard g holds
 * min(k_shard, N_g) rows at or above its own value, so the minimum is a valid lower bound on the global k-th best
 * PROVIDED  sum_g min(k_shard, N_g) >= min(k, sum_g N_g)  - the caller's obligation.  k_shard = ceil(k / shards)
 * satisfies it when every shard holds at least that many rows; with small shards use a larger value (k always
 * works; deep-image-retrieval_b200/dist.py: shard_quota picks the smallest valid one from the shard sizes).  The
 * tight bound lets each shard re-score only ~1.4 * k / shards rows instead of ~1.4 * k.  Phase 2 re-scores the rows
 * within the band of max(sel_dev[q], local k-th) exactly and returns the shard's ordered list.  Limits as for
 * dirb200_index_search, except that _begin refuses Q > dirb200_index_search_max_queries(k) with DIRB200_ENOTSUP. */
int dirb200_index_search_begin(dirb200_index* idx, const float* q32_dev, int Q, int k, int k_shard, float* sel_dev,
                               void* stream);
int dirb200_index_search_finish(dirb200_index* idx, const float* q32_dev, const float* sel_dev, double* scores_dev,
                                int64_t* idx_dev, void* stream);
/* Filtered search (DESIGN.md section 4.13, rules F1-F6).  Replaces building a new index over the allowed rows,
 * Index(X[subset]) (and the k + 1 over-fetch + host-side drop that pipeline._drop_self does for one excluded row): the
 * exact top-k of each query over the rows its allow set admits.  words_dev: caller-owned device bitmap of uint32 words
 * in global row numbering (row r = bit r & 31 of word r >> 5), one row of ld_words words per query, or ld_words = 0
 * for one row shared by every query; bit0 = the global number of this shard's row 0 (its index_offset).  Null detaches
 * it.  While it is attached, dirb200_index_search, _search_begin and _search_sharded(_phase) phase 1 apply it (later
 * phases use what their search began with; _search_finish does not read it), and every other entry point that ranks,
 * counts or selects rows (target_scores, rank_count, count_ge, range_search, self_join, nearest, search_lists) returns
 * DIRB200_ESTATE.  The result of each query is the exact top-k of its allowed rows, tail (-inf, -1); with every bit
 * set it equals the unfiltered search bit for bit.  The seed rows of a query block (the first S rows allowed for all of
 * its queries) are gathered into a buffer of S * dim * 2 bytes; a search whose buffer exceeds option "ws_budget" is
 * refused with DIRB200_ENOTSUP.  dirb200_index_set_db detaches the filter. */
int dirb200_index_set_allow(dirb200_index* idx, const uint32_t* words_dev, int64_t ld_words, int64_t bit0);
/* Builds per-query allow sets from lists of rows to leave out (replaces the over-fetch by one + host-side drop of
 * pipeline._drop_self, and per-query junk lists): clears bit rows_dev[i] of bitmap row q (ld_words words apart) for
 * every i in [off_dev[q], off_dev[q + 1]), q < Q.  Rows outside [0, 32 ld_words) are skipped.  Order-independent
 * (atomicAnd).  off_dev int64 [Q + 1], rows_dev int64, both on the device of words_dev; enqueued on `stream`. */
int dirb200_allow_exclude(uint32_t* words_dev, int Q, int64_t ld_words, const int64_t* off_dev, const int64_t* rows_dev,
                          void* stream);
/* Status of the last search, for option "deferred_check": waits for it to finish; DIRB200_EOVERFLOW if a candidate
 * list still overflowed after the retry passes or more than cap2 rows sat within the band of the k-th score. */
int dirb200_index_check(dirb200_index* idx);
/* Statistics of the last search: {dense_rows, candidates_total, survivors_total, retry passes run, launches}
 * (waits for a deferred search to finish). */
int dirb200_index_last_stats(dirb200_index* idx, int64_t stats[5]);
/* With option "profile" = 1: CUDA-event milliseconds of the phases of the last search (valid after its status was
 * collected), out9[0..6] = {query fp16 conversion + clears, seed GEMM, seed k-th select, filter GEMM, candidate k-th
 * select, gated retry passes (+ any cross-shard exchange between the phases), survivors + exact re-scoring + sort};
 * for k > 1024 out9[6..8] = {survivor compaction, exact re-scoring, run sort + merge}. */
int dirb200_index_last_profile(dirb200_index* idx, double out9[9]);
int dirb200_index_destroy(dirb200_index* idx);

/* Rank statistics for AP without the Q x N score matrix (replaces the per-query np.argsort of generic.py:207,221 +
 * junk removal :204-206,216-221 as far as the positions of the labelled rows are concerned).  Targets = the labelled
 * rows of each query, grouped by query: t_off[Q+1] (CSR), t_q[T] (query of target t), t_rows[T] GLOBAL database
 * indices, t_flags[T] (1 = count the rows ranking before this target - the positives; 0 = score only - junk rows).
 *   dirb200_index_target_scores: t_score_dev[t] = exact score <q, db[row]> for rows this shard owns, 0 otherwise
 *                                (several shards: SUM all-reduce of t_score_dev, 8*T bytes).
 *   dirb200_index_rank_count:    above_dev[t] = number of rows OF THIS SHARD that rank before target t under the
 *                                order of dirb200_index_search (exact score desc, ties -> lower global index), for
 *                                flagged targets (several shards: SUM all-reduce of above_dev).  t_score_dev must hold
 *                                the complete scores.  One tensor-core pass; queries whose candidate list overflows
 *                                ("count_cap", default 32768 rows scoring above their lowest positive) are counted
 *                                exactly from the fp32 rows instead (last_stats[3] = number of such queries).
 *                                Synchronises the stream.  Rows are assumed unit-norm (option "eps16"). */
int dirb200_index_target_scores(dirb200_index* idx, const float* q32_dev, int Q, const int* t_q_dev,
                                const int64_t* t_rows_dev, int T, double* t_score_dev, void* stream);
int dirb200_index_rank_count(dirb200_index* idx, const float* q32_dev, int Q, const int* t_off_host, const int* t_off_dev,
                             const int64_t* t_rows_dev, const unsigned char* t_flags_dev, const double* t_score_dev,
                             int T, int64_t* above_dev, void* stream);

/* Threshold counts for label-based AP without the Q x N score matrix (replaces sklearn's average_precision_score over
 * a full score row, dataset.py:83-92 / evaluation.py:41-43, and the full argsort of the top-k, dataset.py:94-101).
 * Thresholds of each query, grouped by query: thr_off_dev[Q+1] (CSR from 0 to T), thr_dev[T] fp32 in DESCENDING order
 * within each query (typically s_t = fp32 rounding of the exact scores of its positives, dirb200_index_target_scores).
 *   count_dev[t] = number of rows r OF THIS SHARD, global index r + offset != skip_row_dev[q] (-1 or a null pointer:
 *                  no row skipped), with fp32(exact score <q, row r>) >= thr[t].  Several shards: SUM all-reduce.
 * One fp64 tensor-core pass; pairs within eps of a rounding boundary are re-scored exactly (last_stats[1] = their
 * number), and a query whose pairs overflow the band list (option "band_cap", default 2^20 entries) is counted exactly
 * over all rows (last_stats[3] = number of such queries).  eps = 4 gamma_D |q| max|row| from the norms of the call,
 * or option "count_eps" (> 0) as an absolute override.  Synchronises the stream; DIRB200_EINVAL for malformed offsets
 * or thresholds that are not finite and descending. */
int dirb200_index_count_ge(dirb200_index* idx, const float* q32_dev, int Q, const int* thr_off_dev, const float* thr_dev,
                           int T, const int64_t* skip_row_dev, int64_t* count_dev, void* stream);

/* Merge G per-shard top-k lists (scores fp64 + global indices int64, as produced by an all-gather of
 * dirb200_index_search outputs: each list ordered best first, empty slots = index -1 at the tail, no row in two
 * lists) into the global top-k with the same ordering rule.  Shard g's [Q][k] block starts
 * shard_stride elements after shard g-1's (0 = dense [G][Q][k]); a packed all-gather buffer [G][2][Q][k] uses
 * shard_stride = 2*Q*k with idx_dev = scores_dev + Q*k.  Any G and k: up to G*k = 4096 the lists of a query are merged
 * in shared memory, beyond that straight from global memory (same rank-based merge, same result). */
int dirb200_topk_merge(const double* scores_dev, const int64_t* idx_dev, int G, int Q, int k, int64_t shard_stride,
                       double* out_scores_dev, int64_t* out_idx_dev, void* stream);
/* Sharded search over PEER MEMORY (one process per GPU of one NVLink / NVSwitch box; the reference's analogue of a
 * multi-GPU database is nn.DataParallel, utils/common.py:155, and scores = matmul(q, db) over the whole database,
 * common.py:30-38 + datasets/generic.py:207).  Every rank creates an exchange window (device buffer for up to max_q
 * queries x max_k results from `world` <= 8 ranks), hands its 64-byte CUDA IPC handle to the others (any transport:
 * torch.distributed, MPI, a file), and opens theirs.  dirb200_index_search_sharded then runs the whole two-phase
 * protocol on the caller's stream without any library collective: seed bounds, selection thresholds and the per-shard
 * lists are written by the producing kernels straight into every peer's window (stores over NVLink), the consuming
 * kernels wait on flags in their own window - two MIN all-reduces and the all-gather fused into the search kernels.  The
 * first MIN (every shard's k_shard-th seed bound) tightens the filter threshold of all shards before their filter pass:
 * ~k_shard / k of the candidates a stand-alone shard search captures.  It is a collective
 * call: every rank calls it the same number of times with the same Q, k, k_shard (k_shard: see _search_begin).
 * Results: global exact top-k on every rank.  Never synchronises; collect the status with dirb200_index_check
 * (DIRB200_EOVERFLOW also when a peer did not arrive within ~10 s).
 *   _open        handles = world x 64 bytes in rank order (entry `rank` is ignored)
 *   _open_local  same-process variant: all = the `world` exchange objects of this process (several shards driven by
 *                one process, tests); the four phases of the search (1 seed pass + seed bounds, 2 filter pass + selection
 *                thresholds, 3 exact re-scoring + lists, 4 merge) can then be issued shard by shard on one stream with
 *                dirb200_index_search_sharded_phase: phase p for every shard before phase p + 1 of any. */
int dirb200_exchange_create(int device, int world, int rank, int max_q, int max_k, dirb200_exchange** out);
int dirb200_exchange_ipc_handle(dirb200_exchange* x, void* handle64_out);
int dirb200_exchange_open(dirb200_exchange* x, const void* handles);
int dirb200_exchange_open_local(dirb200_exchange* x, dirb200_exchange* const* all);
int dirb200_exchange_close_peers(dirb200_exchange* x);   /* unmap the peers' windows; barrier among the ranks; then _destroy */
int dirb200_exchange_destroy(dirb200_exchange* x);
int dirb200_index_search_sharded(dirb200_index* idx, dirb200_exchange* x, const float* q32_dev, int Q, int k, int k_shard,
                                 double* scores_dev, int64_t* idx_dev, void* stream);
int dirb200_index_search_sharded_phase(dirb200_index* idx, dirb200_exchange* x, int phase, const float* q32_dev, int Q, int k,
                                       int k_shard, double* scores_dev, int64_t* idx_dev, void* stream);
/* Full exact score matrix (fp64 accumulate, fp32 out): the literal common.matmul for small evaluation sets. */
int dirb200_scores_exact(const float* q_dev, int Q, const float* db_dev, int64_t N, int D, float* out_dev,
                         void* stream);
/* Alpha query expansion, test_dir.py:24-44:  out_i = normalize(mean([q_i] + [db_j * s_ij^alpha, j in topk(i)])).
 * nn_idx_dev/nn_scores_dev: [Q][k] neighbour indices (-1 = none) and their scores.  Sharded mode (partial != 0, or
 * n_rows > 0): the indices are GLOBAL and db32_dev holds the rows [row_offset, row_offset+n_rows) of a sharded
 * database; neighbours owned by other shards are skipped (an EMPTY shard, n_rows == 0 with partial != 0, owns none and
 * may pass db32_dev = NULL).  Otherwise (partial == 0 and n_rows <= 0) the indices are plain rows of db32_dev.
 * partial != 0 writes the un-normalised SUM over the owned neighbours only, for a cross-GPU all-reduce.  Any k >= 1:
 * the weights are taken 2048 at a time, and every output element accumulates its neighbours in list order. */
int dirb200_aqe_expand(const float* q_dev, int Q, int D, const float* db32_dev, const int64_t* nn_idx_dev,
                       const double* nn_scores_dev, int k, double alpha, int partial, int64_t row_offset, int64_t n_rows,
                       float* out_dev, void* stream);

/* The statistics of a PCA fit, in fp64 (replaces the host work of sklearn's PCA.fit, _pca.py _fit_full).  x_dev
 * [N][D] fp32 row-major, any N >= 0.  Both ADD into the caller's buffers, so rows may be fed in chunks; both run in a
 * fixed summation order that depends on (N, D) only (no atomics): the same call gives bit-identical results on every
 * run and every device.  Scratch comes from the library's per-device cache.
 * dirb200_col_sums_f64: sum_dev[j] += sum_i x[i][j].
 * dirb200_gram_f64: gram_dev[i][j] += sum_r (x[r][i] - mean[i]) (x[r][j] - mean[j]), the full symmetric [D][D]
 * matrix, centred in fp64 (the covariance_eigh branch forms X^T X - n m m^T instead, which cancels when |mean| is
 * large against the spread).  D % 4 == 0 (else DIRB200_EINVAL) and D <= 8064 (else DIRB200_ENOTSUP: the split-K
 * partial tiles are bounded to 256 MiB). */
int dirb200_col_sums_f64(const float* x_dev, int64_t N, int D, double* sum_dev, void* stream);
int dirb200_gram_f64(const float* x_dev, int64_t N, int D, const double* mean_dev, double* gram_dev, void* stream);

/* The listwise AP loss of "Learning with Average Precision" (reference dirtorch/loss.py), without the N x 2nq x M
 * quantised tensor.  x_dev [N][M] fp32 scores, label_dev [N][M] uint8 (0 = negative, anything else = positive), any
 * N >= 1 and 1 <= M < 2^31 (else DIRB200_ENOTSUP), 2 <= nq <= 100.  table_dev: 4 nq fp32 on the device, the 2nq
 * quantiser weights then the 2nq biases, built as loss.py:29-41 builds the Conv1d (the kernels rely on that shape:
 * bin j peaks at fmaf(w_1, x, b_1) = j).  Bin j of a score is max(0, min(v_j, v_{j+nq})), v_i = fl32(fmaf(w_i, x, b_i)).
 * dirb200_aploss_forward: mode 0 = APLoss.forward (loss.py:43-55, eps 1e-16), 1 = TAPLoss (loss.py:90-119, eps 1e-8),
 * 2 = TAPLoss(simplified=True).  Writes hist_dev [N][2nq+1] int64 (c, cp and the positive count, each in units of
 * 2^-32; exact, independent of the launch shape), G_dev [N][2nq] fp64 (dAP/dc, dAP/dcp) and ap_dev [N] fp32 (the
 * per-row AP, computed in fp64 and rounded once; NaN for a row without positives, as the reference).
 * dirb200_aploss_backward: dx_dev [N][M] = grad_ap[n] * sum_j (G_c[n][j] + l G_cp[n][j]) dq_j/dx, with torch's
 * subgradients: clamp(min=0) passes where the min is >= 0, torch.min splits a tie 1/2 : 1/2.  Both run on `stream`
 * with no host synchronisation and no float atomics: the results are bit-identical on every run. */
int dirb200_aploss_forward(const float* x_dev, const uint8_t* label_dev, int64_t N, int64_t M, int nq,
                           const float* table_dev, int mode, int64_t* hist_dev, double* G_dev, float* ap_dev,
                           void* stream);
int dirb200_aploss_backward(const float* x_dev, const uint8_t* label_dev, int64_t N, int64_t M, int nq,
                            const float* table_dev, const double* G_dev, const float* grad_ap_dev, float* dx_dev,
                            void* stream);

/* Diffusion re-ranking: manifold ranking (Zhou et al., "Ranking on Data Manifolds", NIPS 2003) over the mutual-kNN
 * graph of the database, solved by conjugate gradient (Iscen et al., "Efficient Diffusion on Region Manifolds", CVPR
 * 2017).  The rules are restated in DESIGN.md section 4.7; all arithmetic is fp64 and no value is accumulated with
 * atomics, so a given input gives bit-identical output on every run.  Workspaces are caller-owned device buffers of
 * the *_workspace_bytes size.
 * dirb200_diffusion_graph: nn_idx_dev / nn_score_dev [N][width] are the exact top-width lists of the database against
 * itself (dirb200_index_search with width = k + 1, or fewer columns when N <= k; -1 entries are skipped).
 * nn(i) = the first k entries other than i itself (by index).  Writes the CSR of
 * S = D^-1/2 A D^-1/2 (step 2 of Zhou et al.'s algorithm, on the sparse mutual-kNN affinity of Iscen et al.): A_ij = max(s_ij, 0)^gamma for mutual neighbours (j in nn(i) and i in nn(j)), d_i = sum_j A_ij in
 * ascending j, S_ij = A_ij * (u_i * u_j) with u_i = 1/sqrt(d_i) (0 for d_i = 0): exactly symmetric.  row_ptr_dev
 * [N+1] int64, col_dev / val_dev capacity N * k (nnz = row_ptr[N] <= N k), columns ascending within a row.  1 <= k <=
 * 2047 (else DIRB200_ENOTSUP), width <= k + 1, gamma > 0.
 * dirb200_diffusion_seeds: y_dev [N][Q] (zeroed by the call) gets y[j][q] = max(s, 0)^gamma for each (j, s) of query
 * q's top-kq list idx_dev / score_dev [Q][kq] (the query vector y of Iscen et al.; entries -1 are skipped).
 * dirb200_diffusion_solve: (I - alpha S) f = y for the Q columns of y_dev [N][Q] (the closed form
 * f* = (I - alpha S)^-1 y of Zhou et al.'s iteration, up to its (1 - alpha) scale) by conjugate gradient from f = 0: at most `iters` iterations, query q stops
 * (f, r, p frozen) at the first iteration whose recurrence residual has ||r|| <= tol ||y_q||; y_q = 0 gives f = 0.
 * Writes f_dev [N][Q], iters_dev [Q] (iterations done) and resid_dev [Q] (final recurrence ||r||).  A query's f is
 * bit-identical whatever Q and whatever its column.  0 <= alpha < 1, iters >= 1, tol >= 0.
 * dirb200_diffusion_rank_count: for the flagged targets t of each query (CSR offsets t_off [Q+1] on host and device,
 * t_rows int64 in [0, N), t_flags uint8), above_dev[t] = the number of rows ranking before t_rows[t] when the column
 * q of f_dev [N][Q] is ranked by f descending, ties -> lower index, -0 == +0 (0 for unflagged targets), and
 * t_score_dev[t] = f[t_rows[t]][q] for every target.  At most 12000 targets per query and 65535 queries (else
 * DIRB200_ENOTSUP).
 * dirb200_diffusion_topk: the exact top-k rows of each column q of f_dev [N][Q] under the same order (Zhou et al.'s
 * step 4, "rank each point according to its score f*"): scores_dev [Q][k] fp64 = f, idx_dev [Q][k] int64.  1 <= k <=
 * N, Q <= 65535 (else DIRB200_ENOTSUP). */
size_t dirb200_diffusion_graph_workspace_bytes(int64_t N, int k);
int dirb200_diffusion_graph(const int64_t* nn_idx_dev, const double* nn_score_dev, int64_t N, int width, int k,
                            double gamma, void* ws_dev, int64_t* row_ptr_dev, int* col_dev, double* val_dev, void* stream);
int dirb200_diffusion_seeds(const int64_t* idx_dev, const double* score_dev, int Q, int kq, double gamma, int64_t N,
                            double* y_dev, void* stream);
size_t dirb200_diffusion_solve_workspace_bytes(int64_t N, int Q);
int dirb200_diffusion_solve(const int64_t* row_ptr_dev, const int* col_dev, const double* val_dev, int64_t N,
                            const double* y_dev, int Q, double alpha, int iters, double tol, void* ws_dev, double* f_dev,
                            int* iters_dev, double* resid_dev, void* stream);
size_t dirb200_diffusion_rank_count_workspace_bytes(int Q, int T);
int dirb200_diffusion_rank_count(const double* f_dev, int64_t N, int Q, const int* t_off_host, const int* t_off_dev,
                                 const int64_t* t_rows_dev, const uint8_t* t_flags_dev, int T, void* ws_dev,
                                 double* t_score_dev, int64_t* above_dev, void* stream);
size_t dirb200_diffusion_topk_workspace_bytes(int Q, int k);
int dirb200_diffusion_topk(const double* f_dev, int64_t N, int Q, int k, void* ws_dev, double* scores_dev,
                           int64_t* idx_dev, void* stream);

/* Truncated diffusion (Iscen et al. 2017): each query solved on the subgraph of its own top-m rows R_q (DESIGN.md
 * section 4.7, rules T1-T6).  Every query of a call has the same m (= min(m, N) rows); local row l of query q is the
 * l-th row of R_q in ascending global index.  Per-query local matrices are stored ELL, column-major per query: entry e
 * of local row l at [q][e][l], kw entries per row (kw >= the longest row of the global graph).
 * dirb200_diffusion_graph_weights: dirb200_diffusion_graph (the same workspace, the same row_ptr / col / val bits),
 * and also a_dev (capacity N * k) = A_ij, the values before normalisation, and u_dev [N] = u_i.
 * dirb200_diffusion_trunc_build: from the exact lists list_idx_dev / list_score_dev [Q][m] (Index.search at depth m)
 * and the global CSR of A: rows_dev [Q][m] int64 (R_q ascending), lcnt_dev [Q][m] (entries per local row),
 * lcol_dev [Q][kw][m] int32 (local columns, ascending) and lval_dev [Q][kw][m] fp64 = S'_ij = A_ij * (u'_i * u'_j),
 * d_dev / u_dev [Q][m] = d'_i (the row of A within R_q summed in ascending j) and u'_i = 1/sqrt(d'_i) (0 if d'_i = 0),
 * y_dev [Q][m] = max(s, 0)^gamma at the first kq list entries, 0 elsewhere.  1 <= kq <= m <= N, gamma > 0.
 * dirb200_diffusion_trunc_solve: (I - alpha S') f' = y' per query by conjugate gradient, all iterations in one launch,
 * with the arithmetic and the reduction order of dirb200_diffusion_solve (with m = N it returns that call's f, iteration
 * count and residual bit for bit).  Writes f_dev [Q][m], iters_dev [Q], resid_dev [Q]; the same arguments as
 * dirb200_diffusion_solve otherwise.
 * dirb200_diffusion_trunc_topk: the first k rows under rule T6: the m local rows by f' descending, ties -> lower row,
 * -0 == +0, then (k > m) entries m .. k-1 of the exact lists list_idx_dev / list_score_dev [Q][list_width] (list_width
 * >= k; unused when k <= m).  scores_dev [Q][k] = f' for the local rows, the exact score after them; idx_dev [Q][k].
 * Q <= 65535 (else DIRB200_ENOTSUP).
 * dirb200_diffusion_trunc_rank_count: for each target (device CSR offsets t_off_dev [Q+1], t_rows_dev, t_flags_dev):
 * inside_dev = 1 when the row lies in R_q, value_dev = its f' (0 outside), above_dev = the rows of R_q ranking before
 * it under rule T6 (flagged targets inside R_q; 0 otherwise).  A target outside R_q ranks after all of R_q, in exact
 * score order: its rank count is dirb200_index_rank_count's. */
int dirb200_diffusion_graph_weights(const int64_t* nn_idx_dev, const double* nn_score_dev, int64_t N, int width, int k,
                                    double gamma, void* ws_dev, int64_t* row_ptr_dev, int* col_dev, double* val_dev,
                                    double* a_dev, double* u_dev, void* stream);
size_t dirb200_diffusion_trunc_build_workspace_bytes(int Q, int m);
int dirb200_diffusion_trunc_build(const int64_t* row_ptr_dev, const int* col_dev, const double* a_dev, int64_t N,
                                  int kw, const int64_t* list_idx_dev, const double* list_score_dev, int Q, int m,
                                  int kq, double gamma, void* ws_dev, int64_t* rows_dev, int* lcnt_dev, int* lcol_dev,
                                  double* lval_dev, double* d_dev, double* u_dev, double* y_dev, void* stream);
size_t dirb200_diffusion_trunc_solve_workspace_bytes(int Q, int m);
int dirb200_diffusion_trunc_solve(const int* lcnt_dev, const int* lcol_dev, const double* lval_dev, int kw,
                                  const double* y_dev, int Q, int m, double alpha, int iters, double tol, void* ws_dev,
                                  double* f_dev, int* iters_dev, double* resid_dev, void* stream);
size_t dirb200_diffusion_trunc_topk_workspace_bytes(int Q, int m, int k);
int dirb200_diffusion_trunc_topk(const int64_t* rows_dev, const double* f_dev, int Q, int m,
                                 const int64_t* list_idx_dev, const double* list_score_dev, int list_width, int k,
                                 void* ws_dev, double* scores_dev, int64_t* idx_dev, void* stream);
int dirb200_diffusion_trunc_rank_count(const int64_t* rows_dev, const double* f_dev, int Q, int m,
                                       const int* t_off_dev, const int64_t* t_rows_dev, const uint8_t* t_flags_dev,
                                       int T, uint8_t* inside_dev, double* value_dev, int64_t* above_dev, void* stream);

/* Range search and self-join (DESIGN.md section 4.8, rules J1-J6).  e(a, b) is the exact score of the search
 * (fp64 accumulation of the fp32 products, the same bits as dirb200_index_search; e(a, b) == e(b, a)).  A row is a
 * candidate when its fp16-path score reaches tau - eps16 (option "eps16", computed in fp64 and rounded down to fp32);
 * candidates are re-scored exactly and kept when e >= tau.  The result (a CSR: offsets int64, rows int64 + the index
 * offset, scores fp64, each list ordered by (e desc, row asc)) stays in the handle until the next call; its size goes to
 * *total_out and dirb200_index_join_fetch copies it out.  A candidate list that overflows its capacity is detected from
 * the exact match counts and re-run with enough capacity, or its block of rows is halved to fit option "ws_budget";
 * the result does not depend on either.  What cannot fit the budget fails with DIRB200_EOVERFLOW, naming the count.
 * Both calls synchronise the stream once per block of rows for the candidate counts and once per sort sub-block.
 * Option "join_cap": candidate capacity per row of the first pass (0 = min(columns, 4096)).
 * dirb200_index_range_search: for each query q32_dev[q] (Q >= 1) the rows with e(q, r) >= tau, no self-exclusion.
 * dirb200_index_self_join: for the rows i of [row0, row1) (row0 a multiple of 128, row1 <= N) the rows j > i with
 * e(x_i, x_j) >= tau; CSR by i - row0.  Only the 128 x 128 tiles on or above the diagonal run on the tensor cores.
 * tau must be finite (DIRB200_EINVAL). */
int dirb200_index_range_search(dirb200_index* idx, const float* q32_dev, int Q, double tau, int64_t* total_out,
                               void* stream);
int dirb200_index_self_join(dirb200_index* idx, int64_t row0, int64_t row1, double tau, int64_t* total_out,
                            void* stream);
/* Copies the last result: off_dev [rows + 1], idx_dev / scores_dev [total] (may be null when total is 0).
 * Synchronises the stream. */
int dirb200_index_join_fetch(dirb200_index* idx, int64_t* off_dev, int64_t* idx_dev, double* scores_dev, void* stream);
/* Counters of the last range search / self-join: stats = {candidates, pairs, filter re-runs, filter launches, tensor-core
 * tiles}; with option "profile" = 1, ms = CUDA-event milliseconds of {filter passes, exact re-scoring, sort +
 * compaction}. */
int dirb200_index_join_stats(dirb200_index* idx, int64_t stats[5], double ms[3]);
/* Connected components of the undirected graph of n rows given as a CSR (row_ptr_dev [n+1], col_dev [nnz], both int64;
 * each pair may appear once or in both directions): labels_dev [n] = the smallest row of each row's component (rule
 * J4), the same on every run.  Synchronises the stream once per hooking round. */
size_t dirb200_join_components_workspace_bytes(int64_t n);
int dirb200_join_components(const int64_t* row_ptr_dev, const int64_t* col_dev, int64_t n, int64_t nnz, void* ws_dev,
                            int64_t* labels_dev, void* stream);
/* Groups = components of >= 2 rows, by ascending label, members ascending: group g holds
 * members_dev[group_off_dev[g] .. group_off_dev[g+1]).  Capacities: group_off_dev n / 2 + 1, members_dev n.
 * counts_out = {groups, members} (host).  Synchronises the stream. */
size_t dirb200_join_groups_workspace_bytes(int64_t n);
int dirb200_join_groups(const int64_t* labels_dev, int64_t n, void* ws_dev, int64_t* group_off_dev, int64_t* members_dev,
                        int64_t counts_out[2], void* stream);

/* Exact nearest row for many queries (extension; DESIGN.md section 4.9, rules K2 / K3): for each query q32_dev[q]
 * (Q >= 0) labels_dev[q] = the smallest row (+ the index offset) maximising the exact score, scores_dev[q] that score:
 * the top-1 of dirb200_index_search bit for bit.  One PERS_EPI_SIM_GMAX pass gives the fp16-path maximum of each group
 * of 32 rows; the groups within 2 eps16 (rounded down to fp32) of the largest are re-scored exactly, or every row when
 * more than option "nearest_cap" (default 16, at most 256) groups qualify.  Query blocks fit option "ws_budget".
 * Synchronises the stream.  dirb200_index_nearest_stats: {queries with more than one candidate group, queries
 * re-scored over all rows, rows re-scored} of the last call. */
int dirb200_index_nearest(dirb200_index* idx, const float* q32_dev, int Q, int64_t* labels_dev, double* scores_dev,
                          void* stream);
int dirb200_index_nearest_stats(dirb200_index* idx, int64_t stats[3]);
/* Inverted-file search (extension; DESIGN.md section 4.10, rules I2-I6).  dirb200_index_set_lists attaches caller-owned
 * list buffers to an index whose database is set: db16_lists_dev [N][dim] fp16 rows in list order (list ascending, then
 * row ascending), perm_dev [N] int64 (list position -> row of the index), cell_off_dev [K + 1] int64 (list c holds
 * positions cell_off[c] .. cell_off[c + 1] - 1; empty lists allowed).  The original-order db32 / db16 stay, so
 * exact search and rank counts still work on the handle.  K = 0, or a later dirb200_index_set_db, detaches the lists.
 * Synchronises the stream (the offsets are checked on the host).
 * dirb200_index_search_lists: probes_dev [Q][nprobe] int64 (distinct lists in [0, K) per query, 1 <= nprobe <= K) ->
 * the exact top-k of the union of each query's probed lists, scores_dev / idx_dev [Q][k] ordered by (score desc, row
 * asc) with the scores and tail padding (-inf, -1) of dirb200_index_search (rule I4); with every list probed, that
 * search bit for bit.  Grouped tensor-core passes over a device-built table of (list, query tile, row tile) tiles
 * (rule I5), exact re-scoring and the search's finish; a query block whose candidate lists overflow runs again at the
 * exact count or in halves within option "ws_budget", else DIRB200_EOVERFLOW (rule I6).  Options eps16, cand_cap,
 * ws_budget and profile apply.  Synchronises the stream three times per query block (table sizes, candidate counts,
 * status).
 * dirb200_index_lists_stats: {pairs, query rows issued (padding included), tiles, probed rows (sum over queries of the
 * union's size), candidates, re-runs} of the last call; with option "profile", ms = CUDA-event milliseconds of {table
 * build, GMAX pass + seed, FILTER pass + selection, finish}. */
int dirb200_index_set_lists(dirb200_index* idx, const void* db16_lists_dev, const int64_t* perm_dev,
                            const int64_t* cell_off_dev, int K, void* stream);
int dirb200_index_search_lists(dirb200_index* idx, const float* q32_dev, int Q, int k, const int64_t* probes_dev,
                               int nprobe, double* scores_dev, int64_t* idx_dev, void* stream);
int dirb200_index_lists_stats(dirb200_index* idx, int64_t stats[6], double ms[4]);
/* Spherical k-means (extension; DESIGN.md section 4.9, rules K4-K7) on unit fp32 rows x32_dev [n][d] (d a multiple of
 * 64, n < 2^29).  The assignment (rule K2) is dirb200_index_nearest of the rows against the centres.
 * dirb200_kmeans_stats: counts_dev [k] = cluster sizes of labels_dev [n]; out = {labels that differ from prev_dev (n
 * when prev_dev is null), sum of rint(scores_dev[i] * 2^32) (the objective in units of 2^-32, exact in any order),
 * empty clusters}.  Synchronises the stream. */
size_t dirb200_kmeans_stats_workspace_bytes(int64_t n, int k);
int dirb200_kmeans_stats(const int64_t* labels_dev, const double* scores_dev, const int64_t* prev_dev, int64_t n, int k,
                         void* ws_dev, int* counts_dev, int64_t out[3], void* stream);
/* Rule K4, in place on labels_dev / counts_dev (the sizes dirb200_kmeans_stats returned): each empty cluster, in
 * ascending order, takes the row of lowest (score, row) among the rows whose cluster still has >= 2 rows.  k <= n.
 * *moves_out = rows moved.  Synchronises the stream. */
size_t dirb200_kmeans_relocate_workspace_bytes(int64_t n);
int dirb200_kmeans_relocate(int64_t* labels_dev, const double* scores_dev, int64_t n, int k, int* counts_dev,
                            void* ws_dev, int64_t* moves_out, void* stream);
/* Rule K5: centres_dev [k][d] = fl32(s_c / sqrt(||s_c||^2)), s_c the fp64 sum of cluster c's rows in ascending row
 * order (counts_dev [k]: the cluster sizes of labels_dev, as dirb200_kmeans_stats / _relocate leave them), in chunks of 256 rows (each chunk summed sequentially, the chunk sums added in chunk order); ||s_c||^2 as
 * DESIGN.md section 4.9 states.  A cluster with s_c = 0 (or no rows) keeps its centre; *zero_sums_out counts them.
 * Synchronises the stream. */
size_t dirb200_kmeans_update_workspace_bytes(int64_t n, int k, int d);
int dirb200_kmeans_update(const float* x32_dev, int64_t n, int d, const int64_t* labels_dev, const int* counts_dev, int k,
                          float* centres_dev, void* ws_dev, int64_t* zero_sums_out, void* stream);
/* Rule K7, k-means++ by D^2 sampling: chosen_dev [k] = the rows drawn, chosen_dev[0] = first; draw j >= 1 uses
 * u_host[j - 1] in [0, 1) (host, k - 1 values).  Weights w_i = max(0, 2 - 2 e(x_i, nearest chosen row)) in int64 units
 * of 2^-32, 0 for chosen rows; with T their total, the drawn row is the first whose inclusive prefix exceeds
 * min(floor(u * double(T)), T - 1).  When T = 0 (fewer than k distinct rows) that draw and all later ones are -1.
 * Synchronises the stream once, at the end. */
size_t dirb200_kmeans_pp_workspace_bytes(int64_t n, int k);
int dirb200_kmeans_pp(const float* x32_dev, int64_t n, int d, int64_t first, const double* u_host, int k, void* ws_dev,
                      int64_t* chosen_dev, void* stream);

/* Product quantisation of the inverted lists (DESIGN.md section 4.11, rules P1-P8).  D % 64 == 0, M in {8, 16, 32, 64,
 * 128} dividing D with D / M <= 256 (else DIRB200_ENOTSUP).  Codebooks are [M][256][D / M] fp32; a row's residual is
 * fl32(x - centres_dev[labels_dev[row]]).  None of these synchronises the stream.
 * Rule P4: codes_dev = the nearest codeword of each (row, sub-space), row-major [n][M] (m_major = 0) or [M][n]. */
int dirb200_pq_assign(const float* x_dev, int64_t n, int D, const int64_t* labels_dev, const float* centres_dev,
                      const float* codebooks_dev, int M, uint8_t* codes_dev, int m_major, void* stream);
/* Rule P3's update from the m-major codes of dirb200_pq_assign: codeword j of sub-space m = fl32(s / count), s the
 * sequential fp64 sum of its members' residuals in row order; a codeword without members keeps its value.
 * *empty_dev (device int64) = codewords without members. */
int dirb200_pq_update(const float* x_dev, int64_t n, int D, const int64_t* labels_dev, const float* centres_dev,
                      const uint8_t* codes_dev, int M, float* codebooks_dev, int64_t* empty_dev, void* stream);
/* Rule P5's tables: tables_dev [Q][M][256] = fl32(sum over t ascending of q_{m,t} C_m[j][t]) in fp64, no FMA. */
int dirb200_pq_tables(const float* q_dev, int Q, int D, const float* codebooks_dev, int M, float* tables_dev,
                      void* stream);
/* Rules P5-P7 for one block of Q <= 65535 queries: the ADC scores of the rows of each query's probes (probes_dev /
 * probe_scores_dev [Q][nprobe], the exact centre scores), the first min(R, |R(q)|) in (a desc, row asc) order, and
 * their first k (k <= R) in (e desc, row asc) order -> out_scores fp64 / out_rows int64 [Q][k], padded (-inf, -1).
 * codes_dev [N][M] and perm_dev [N] are in list order, list_off_dev [K + 1] the lists' offsets, qoff_dev [Q + 1] the
 * offsets of the queries' probed rows in the block (qoff_dev[Q] = total).  rows: the [N][D] fp32 rows, device memory
 * or pinned host memory (read in place; pageable memory is DIRB200_EINVAL).  ms: null, or 3 doubles receiving the
 * milliseconds of the scan, the selection and the refinement (then the stream is synchronised). */
size_t dirb200_pq_search_ws_bytes(int Q, int64_t total, int R);
int dirb200_pq_search(const float* q_dev, int Q, int D, const float* tables_dev, int M, const int64_t* probes_dev,
                      const double* probe_scores_dev, int nprobe, const uint8_t* codes_dev, const int64_t* perm_dev,
                      const int64_t* list_off_dev, const int64_t* qoff_dev, int64_t total, const float* rows, int R,
                      int k, void* ws_dev, double* out_scores, int64_t* out_rows, double* ms, void* stream);

/* Graph search over a pruned kNN graph of the database (DESIGN.md section 4.12, rules G1-G8).  Rows are int32; none of
 * these synchronises the stream or needs a workspace.
 * Rules G3 / G4: knn_dev [n][K] (row r's kNN list without r, -1 entries allowed, the non-negative entries of a row
 * distinct), K <= 128 -> fwd_dev [n][degree] = F(r), -1 padded; degree <= 128 (else DIRB200_ENOTSUP). */
int dirb200_graph_prune(const int* knn_dev, int64_t n, int K, int degree, int* fwd_dev, void* stream);
/* Rule G5: fwd_dev [n][degree] of dirb200_graph_prune and Rev as a CSR (rev_off_dev [n + 1] int64, rev_src_dev the
 * sources s of each target r ordered by (r's position in F(s), s)) -> graph_dev [n][degree], -1 padded. */
int dirb200_graph_merge(const int* fwd_dev, int64_t n, int degree, const int64_t* rev_off_dev, const int* rev_src_dev,
                        int* graph_dev, void* stream);
/* The shared memory one query of dirb200_graph_search takes (0 for bad arguments, SIZE_MAX beyond any device). */
size_t dirb200_graph_search_smem_bytes(int n_seeds, int itopk, int width, int degree, int max_iter);
/* Rule G7 for Q queries (q_dev [Q][D] fp32, D % 4 == 0) over x_dev [n][D] fp32 and graph_dev [n][degree], from the
 * seeds_dev [Q][n_seeds] (distinct rows, rule G6) -> out_scores fp64 / out_rows int64 [Q][k] (k <= itopk), padded
 * (-inf, -1); n_visited [Q] = |V|, n_iter [Q] = the iterations run.  vis_rows int64 / vis_scores fp64 [Q][n_seeds +
 * max_iter * width * degree], or both null: V in arrival order with its exact scores (entries past |V| unwritten).
 * Parameters whose shared memory exceeds the device's per-block opt-in limit are DIRB200_EINVAL. */
int dirb200_graph_search(const float* q_dev, int Q, int D, const float* x_dev, int64_t n, const int* graph_dev,
                         int degree, const int* seeds_dev, int n_seeds, int itopk, int width, int max_iter, int k,
                         double* out_scores, int64_t* out_rows, int64_t* vis_rows, double* vis_scores, int* n_visited,
                         int* n_iter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIRB200_H_ */
