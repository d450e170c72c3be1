// C-ABI entry points of the encoder path (include/hairfast_b200.h, "Encoder backbones" section).
#include <string.h>

#include "hf_kernels.cuh"

using namespace hf;

static inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

static int check_conv2d(const hf_conv2d_desc* d) {
  HF_REQUIRE(d, "conv2d: null descriptor");
  HF_REQUIRE(d->dtype == HF_BF16 || d->dtype == HF_F16, "conv2d: bad dtype %d", d->dtype);
  HF_REQUIRE(d->ksize == 1 || d->ksize == 3, "conv2d: kernel size %d unsupported (1 or 3)", d->ksize);
  HF_REQUIRE(d->stride == 1 || d->stride == 2, "conv2d: stride %d unsupported (1 or 2)", d->stride);
  HF_REQUIRE(d->groups >= 1 && d->cin > 0 && d->cout > 0 && d->cin % d->groups == 0 && d->cout % d->groups == 0,
             "conv2d: bad channels / groups (%d -> %d, groups %d)", d->cin, d->cout, d->groups);
  HF_REQUIRE(d->cin_pad >= d->cin && d->cin_pad % (32 * d->groups) == 0,
             "conv2d: cin_pad=%d must be >= cin and a multiple of 32 per group", d->cin_pad);
  HF_REQUIRE(d->groups == 1 || d->cin_pad == d->cin, "conv2d: channel padding is not supported with groups > 1");
  HF_REQUIRE(d->cout % 32 == 0, "conv2d: cout=%d must be a multiple of 32", d->cout);
  HF_REQUIRE((d->prepadded == 0 || d->prepadded == 1) && (d->transposed == 0 || d->transposed == 1),
             "conv2d: prepadded / transposed must be 0 or 1");
  HF_REQUIRE(!d->prepadded || (d->ksize == 3 && d->stride == 1 && !d->transposed),
             "conv2d: a prepadded input needs a stride-1 3x3 conv");
  HF_REQUIRE(!d->transposed || (d->ksize == 3 && d->stride == 2 && d->groups == 1),
             "conv2d: the transposed form is ConvTranspose2d(3, stride 2, padding 1, output_padding 1), no groups");
  return HF_OK;
}

// the shape half of the launch: what conv_plan reads
static ConvLaunch conv2d_launch_shape(const hf_conv2d_desc* d, int batch, int height, int width) {
  ConvLaunch cl;
  memset(&cl, 0, sizeof(cl));
  cl.B = batch; cl.H = height; cl.W = width;
  cl.Cin = d->cin_pad; cl.Cout = d->cout;
  cl.taps = d->ksize * d->ksize; cl.dtype = d->dtype;
  cl.stride = d->transposed ? 1 : d->stride; cl.groups = d->groups;   // transposed: the four-parity 3x3 form
  cl.up = d->transposed; cl.prepadded = d->prepadded;
  cl.epi = 1;
  return cl;
}

extern "C" {

size_t hf_conv2d_packed_bytes(const hf_conv2d_desc* d) {
  if (check_conv2d(d)) return 0;
  return align256((size_t)(d->transposed ? 4 : 1) * d->cout * d->ksize * d->ksize * (d->cin_pad / d->groups) * 2);
}

int hf_conv2d_pack(const hf_conv2d_desc* d, const float* weight, const float* out_scale, void* packed, void* stream) {
  int rc = check_conv2d(d);
  if (rc) return rc;
  if ((rc = ensure_device_current())) return rc;
  HF_REQUIRE(weight && packed && ((uintptr_t)packed & 255) == 0, "hf_conv2d_pack: null / unaligned pointer");
  if (d->transposed)
    return launch_pack_conv2d_transposed(weight, out_scale, packed, d->cout, d->cin, d->cin_pad, d->dtype,
                                         (cudaStream_t)stream);
  return launch_pack_conv2d(weight, out_scale, packed, d->cout, d->cin / d->groups, d->cin_pad / d->groups, d->ksize,
                            d->dtype, (cudaStream_t)stream);
}

int hf_conv2d_forward(const hf_conv2d_desc* d, const void* packed, const hf_conv2d_io* io, void* stream) {
  int rc = check_conv2d(d);
  if (rc) return rc;
  if ((rc = ensure_device_current())) return rc;
  reset_launch_count();
  HF_REQUIRE(packed && io && io->x16, "hf_conv2d_forward: null pointer");
  HF_REQUIRE(io->y16 || io->y16b || io->y32_nchw, "hf_conv2d_forward: no output requested");
  HF_REQUIRE(io->batch > 0 && io->height > 0 && io->width > 0, "hf_conv2d_forward: bad shape");
  HF_REQUIRE(io->act != 1 || io->slope, "hf_conv2d_forward: PReLU needs a slope vector");
  ConvLaunch cl = conv2d_launch_shape(d, io->batch, io->height, io->width);
  cl.xhat_in = io->x16; cl.wpk = packed;
  cl.enc_shift = io->shift; cl.enc_act = io->act; cl.enc_slope = io->act == 1 ? io->slope : nullptr;
  cl.enc_slope0 = io->slope0;
  cl.enc_residual = io->residual16;
  cl.enc_post = io->act_after_residual ? 1 : 0;
  cl.xhat_out = io->y16;
  cl.enc_s2 = io->y16b_scale; cl.enc_b2 = io->y16b_shift; cl.enc_y16b = io->y16b;
  cl.out_nchw = io->y32_nchw;
  return launch_conv(cl, (cudaStream_t)stream, nullptr);
}

int hf_conv2d_plan_query(const hf_conv2d_desc* d, int batch, int height, int width, int* out) {
  int rc = check_conv2d(d);
  if (rc) return rc;
  HF_REQUIRE(out, "hf_conv2d_plan_query: null output");
  ConvPlan pl;
  if ((rc = conv_plan(conv2d_launch_shape(d, batch, height, width), &pl))) return rc;
  conv_plan_export(pl, out);
  return HF_OK;
}

int hf_nchw_to_nhwc16(const float* x, const float* scale, const float* shift, void* y16, int batch, int channels,
                      int c_pad, int height, int width, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_nchw_to_nhwc16(x, scale, shift, y16, batch, channels, c_pad, height * width, dtype,
                               (cudaStream_t)stream);
}

int hf_nhwc16_to_nchw(const void* x16, float* y, int batch, int channels, int height, int width, int dtype,
                      void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_nhwc16_to_nchw(x16, y, batch, channels, height * width, dtype, (cudaStream_t)stream);
}

size_t hf_channel_reduce_workspace_bytes(int batch, int hw, int channels) {
  if (batch <= 0 || hw <= 0 || channels <= 0) return 0;
  return (size_t)batch * channel_reduce_splits(batch, hw, channels) * channels * sizeof(float);
}

size_t hf_instance_norm_workspace_bytes(int batch, int hw, int channels) {
  if (batch <= 0 || hw <= 0 || channels <= 0) return 0;
  return hf_channel_reduce_workspace_bytes(batch, hw, channels) + 2 * (size_t)batch * channels * sizeof(float);
}

int hf_instance_norm_lrelu_nhwc16(const void* x16, void* y16, void* workspace, int batch, int hw, int channels,
                                  float slope, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_instance_norm_act(x16, y16, (float*)workspace, batch, hw, channels, 1e-5f, slope, dtype,
                                  (cudaStream_t)stream);
}

int hf_reflect_pad1_nhwc16(const void* x16, void* y16, int batch, int height, int width, int channels, int dtype,
                           void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_reflect_pad1(x16, y16, batch, height, width, channels, dtype, (cudaStream_t)stream);
}

int hf_channel_mean_nhwc16(const void* x16, float* mean, void* workspace, int batch, int hw, int channels, int dtype,
                           void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_se_gate(x16, nullptr, nullptr, mean, (float*)workspace, batch, hw, channels, 0, dtype,
                        (cudaStream_t)stream);
}

int hf_se_gate_nhwc16(const void* x16, const float* fc1_weight, const float* fc2_weight, float* gate, void* workspace,
                      int batch, int hw, int channels, int reduced, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  HF_REQUIRE(fc1_weight && fc2_weight, "hf_se_gate_nhwc16: null fc weights");
  return launch_se_gate(x16, fc1_weight, fc2_weight, gate, (float*)workspace, batch, hw, channels, reduced, dtype,
                        (cudaStream_t)stream);
}

int hf_scale_add_nhwc16(const void* res16, const float* se, const void* shortcut16, int shortcut_stride,
                        const float* s2, const float* b2, void* y16, void* y16b, int batch, int height, int width,
                        int channels, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_scale_add(res16, se, shortcut16, shortcut_stride, s2, b2, y16, y16b, batch, height, width, channels,
                          dtype, (cudaStream_t)stream);
}

int hf_upsample_add_nhwc16(const void* x16, const void* y16, void* out16, int batch, int h, int w, int height,
                           int width, int channels, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_upsample_add(x16, y16, out16, batch, h, w, height, width, channels, dtype, (cudaStream_t)stream);
}

int hf_adaptive_avgpool_nhwc16(const void* x16, float* y, int batch, int height, int width, int channels, int oh,
                               int ow, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_adaptive_avgpool(x16, y, batch, height, width, channels, oh, ow, dtype, (cudaStream_t)stream);
}

/* ---- BiSeNet glue (SURVEY 8f-3) ---- */
int hf_stem7x7s2_nhwc16(const float* x, const void* wpacked, const float* shift, void* y16, int batch, int height,
                        int width, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_stem7x7s2_fused(x, wpacked, shift, y16, batch, height, width, dtype, (cudaStream_t)stream);
}

int hf_stem3x3_nhwc16(const float* x, const void* wpacked, const float* shift, const float* slope, const float* s2,
                      const float* b2, void* y16, void* y16b, int batch, int height, int width, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_stem3x3_fused(x, wpacked, shift, slope, s2, b2, y16, y16b, batch, height, width, dtype,
                              (cudaStream_t)stream);
}

int hf_maxpool3x3s2_nhwc16(const void* x16, void* y16, int batch, int height, int width, int channels, int dtype,
                           void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_maxpool3x3s2(x16, y16, batch, height, width, channels, dtype, (cudaStream_t)stream);
}

int hf_pooled_fc_nhwc16(const void* x16, const float* weight, const float* scale, const float* shift, int act,
                        float* out, void* workspace, int batch, int hw, int channels, int cout, int dtype,
                        void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_pooled_fc(x16, weight, scale, shift, act, out, (float*)workspace, batch, hw, channels, cout, dtype,
                          (cudaStream_t)stream);
}

int hf_gate_add_up_nhwc16(const void* x16, const float* gate, const float* addvec, const void* addt16, void* y16,
                          int batch, int height, int width, int channels, int up, int dtype, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_gate_add_up(x16, gate, addvec, addt16, y16, batch, height, width, channels, up, dtype,
                            (cudaStream_t)stream);
}

int hf_bicubic_downsample_f32(const float* x, const float* kernel, float* y, int planes, int height, int width,
                              int factor, int clip_round, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_bicubic_down(x, kernel, y, planes, height, width, factor, clip_round, (cudaStream_t)stream);
}

int hf_dilate_erode_f32(const float* mask, float* dilate, float* erode, void* workspace, int planes, int height,
                        int width, int iterations, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_dilate_erode(mask, dilate, erode, (float*)workspace, planes, height, width, iterations,
                             (cudaStream_t)stream);
}

int hf_bilinear_argmax_nchw_f32(const float* x, long long* labels, int batch, int channels, int in_channels, int h,
                                int w, int height, int width, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_bilinear_argmax(x, labels, batch, channels, in_channels, h, w, height, width, (cudaStream_t)stream);
}

int hf_align_masks_f32(const float* hair_mask1, const float* hair_mask2, const float* hair_mask_target, float* masks,
                       int n, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_align_masks(hair_mask1, hair_mask2, hair_mask_target, masks, n, (cudaStream_t)stream);
}

int hf_fspace_blend_f32(const float* first, const float* const* src, const float* const* mask, const float* scale_a,
                        const float* scale_b, float* out, int n_stage, int channels, int height, int width,
                        int mask_height, int mask_width, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_fspace_blend(first, src, mask, scale_a, scale_b, out, n_stage, channels, height, width, mask_height,
                             mask_width, (cudaStream_t)stream);
}

int hf_bilinear_upsample_nchw_f32(const float* x, float* y, int batch, int channels, int in_channels, int h, int w,
                                  int height, int width, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  return launch_bilinear_up_nchw(x, y, batch, channels, in_channels, h, w, height, width, (cudaStream_t)stream);
}

}  // extern "C"
