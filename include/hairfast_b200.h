/* hairfast_b200.h -- C ABI of libhairfast_sm90.so
 *
 * H100 (sm_90a) implementation of the HairFastGAN hot path: the StyleGAN2 generator forward
 * (ModulatedConv2d / StyledConv / ToRGB / upfirdn2d / fused bias+LeakyReLU).  Plain pointers and
 * sizes only -- no torch types.  All pointers are DEVICE pointers unless stated otherwise; every
 * output buffer is caller-allocated (the library never allocates device memory); every call
 * enqueues on the given cudaStream_t (passed as void*) and returns without synchronising, so the
 * calls are CUDA-graph capturable.  Return value: HF_OK (0) or a negative error code;
 * hf_last_error() gives the message (thread-local).
 *
 * Each entry point cites the reference interface (AIRI-Institute/HairFastGAN @ 49e98019) it
 * replaces.  INTEGRATION.md shows the reference-side binding.
 */
#ifndef HAIRFAST_B200_H_
#define HAIRFAST_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HF_OK 0
#define HF_ERR_INVALID (-1)     /* bad argument / unsupported shape */
#define HF_ERR_CUDA (-2)        /* CUDA runtime / driver error */
#define HF_ERR_UNSUPPORTED (-3) /* device is not sm_90 */

/* 16-bit storage/operand type of the tensor-core path (accumulation is always fp32) */
#define HF_BF16 0
#define HF_F16 1

#define HF_MAX_STYLED 17 /* conv1 + convs.0..15 for size 1024 */
#define HF_MAX_TORGB 9   /* to_rgb1 + to_rgbs.0..7 */

int hf_version(void);
const char* hf_last_error(void);
/* Select the CUDA device for subsequent calls of this thread (the reference uses the current
 * device of the calling thread, op/fused_bias_act_kernel.cu:54-56). */
int hf_set_device(int device);
int hf_sm_count(void);

/* ------------------------------------------------------------------------------------------
 * Operator boundary (models/stylegan2/op)
 * ------------------------------------------------------------------------------------------ */

/* Replaces upfirdn2d_op.upfirdn2d(input[major,H,W,1], kernel[kh,kw], up_x, up_y, down_x, down_y,
 * pad_x0, pad_x1, pad_y0, pad_y1) (op/upfirdn2d.cpp:12-22, op/upfirdn2d_kernel.cu:209-369).
 * x: [planes, in_h, in_w] fp32, y: [planes, out_h, out_w] fp32 with
 * out = (in*up + pad0 + pad1 - k) / down + 1.  planes = N*C (minor dim is 1 on every reference
 * call path, op/upfirdn2d.py:99). */
int hf_upfirdn2d_f32(const float* x, float* y, const float* kernel, int planes, int in_h, int in_w,
                     int kernel_h, int kernel_w, int up_x, int up_y, int down_x, int down_y,
                     int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream);

/* Replaces fused.fused_bias_act(input, bias, refer, act, grad=0, alpha, scale)
 * (op/fused_bias_act.cpp:11-21, op/fused_bias_act_kernel.cu:19-99), forward only:
 * y[i] = act(x[i] + bias[(i / step_b) % size_b]) * scale; act: 1 = linear, 3 = leaky relu(alpha).
 * bias may be NULL (size_b = 0). */
int hf_bias_act_f32(const float* x, const float* bias, float* y, int64_t n, int size_b, int64_t step_b,
                    int act, float alpha, float scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * Module level: one StyledConv / ModulatedConv2d (models/stylegan2/model.py:183-343)
 * ------------------------------------------------------------------------------------------ */

typedef struct {
  int cin, cout;
  int ksize;    /* 3 (StyledConv) or 1 */
  int upsample; /* 0 plain, 1 = conv_transpose(stride 2) + blur (model.py:252-263) */
  int dtype;    /* HF_BF16 / HF_F16 */
} hf_conv_desc;

/* Bytes of the packed-weight blob for one conv: 16-bit GEMM operand [N,K] (+ the four polyphase
 * kernels for upsample) followed by the fp32 demod table Wsq[cout,cin]. */
size_t hf_conv_packed_bytes(const hf_conv_desc* d);

/* Pack ModulatedConv2d.weight[1,cout,cin,k,k] (fp32; scaled by 1/sqrt(cin*k*k) here, model.py:220)
 * and, for upsample, compose it with blur_kernel[4,4] (model.py:204-210) into the polyphase form.
 * Once per weight load. */
int hf_conv_pack(const hf_conv_desc* d, const float* weight, const float* blur_kernel, void* packed,
                 void* stream);

typedef struct {
  int batch, height, width;  /* input spatial size */
  const float* x;            /* [B,cin,H,W] fp32 NCHW; batch_stride_x = 0 broadcasts one sample */
  int x_batch_broadcast;
  const float* style;        /* [B, style_dim] latent rows for this layer (row stride style_stride) */
  int style_dim;
  int64_t style_stride;
  const float* mod_weight;   /* conv.modulation.weight [cin, style_dim] */
  const float* mod_bias;     /* conv.modulation.bias [cin] */
  int demodulate;
  /* StyledConv tail (NoiseInjection model.py:288-293 + FusedLeakyReLU op/fused_act.py:73-82);
   * noise == NULL and act == 0 gives the bare ModulatedConv2d.forward */
  const float* noise;        /* [noise_batch,1,Ho,Wo] or NULL */
  int noise_batch;           /* 1 or B */
  const float* noise_weight; /* device scalar, or NULL */
  const float* act_bias;     /* [cout] or NULL */
  int act;                   /* 0 none, 1 = leaky_relu(0.2) * sqrt(2) */
  float* y;                  /* [B,cout,Ho,Wo] fp32 NCHW */
  void* workspace;           /* hf_conv_workspace_bytes() */
} hf_conv_io;

size_t hf_conv_workspace_bytes(const hf_conv_desc* d, int batch, int height, int width);

/* Introspection (tests / DESIGN tables; needs no device): the tiling the library will use for this
 * conv.  out[12] = {halo kernel?, n_tile, num_n_tiles, tiles per round G, halo ring slots, halo pitch,
 * weights resident?, pipeline stages, dynamic smem bytes, work items, grid, channels per K chunk}. */
int hf_conv_plan_query(const hf_conv_desc* d, int batch, int height, int width, int* out /* host[12] */);

/* Replaces ModulatedConv2d.forward (model.py:238-279) / StyledConv.forward (model.py:337-343). */
int hf_conv_forward(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, void* stream);

/* Measurement helper (no reference counterpart): runs hf_conv_forward's prologue once, then the
 * wgmma convolution kernel alone `iters` times between two CUDA events recorded on `stream`, and
 * returns the average kernel duration in milliseconds (host pointer).  Synchronises the stream. */
int hf_conv_time_kernel(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, int iters,
                        float* avg_ms /* host */, void* stream);

/* Replaces ToRGB.forward (model.py:356-365): modulated 1x1 conv without demodulation + bias +
 * Upsample(skip) (model.py:35-53).  x [B,cin,H,W], skip [B,3,H/2,W/2] or NULL, y [B,3,H,W]; fp32. */
int hf_torgb_forward(const float* x, const float* style, int64_t style_stride, int style_dim,
                     const float* conv_weight /* [1,3,cin,1,1] */, const float* mod_weight,
                     const float* mod_bias, const float* bias /* [1,3,1,1] */,
                     const float* up_kernel /* [4,4] or NULL */, const float* skip, float* y, int batch,
                     int cin, int height, int width, void* workspace /* batch*cin*4 bytes */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Generator level (models/stylegan2/model.py:368-565)
 * ------------------------------------------------------------------------------------------ */

typedef struct {
  int size;               /* 256 / 512 / 1024 */
  int style_dim;          /* 512 */
  int channel_multiplier; /* 2 */
  int dtype;              /* HF_BF16 / HF_F16 */
} hf_gen_config;

/* Device pointers to the fp32 parameters, in Generator.state_dict() naming.  Styled convs:
 * index 0 = conv1, index i+1 = convs.{i}; ToRGB: index 0 = to_rgb1, index i+1 = to_rgbs.{i}. */
typedef struct {
  const float* const_input;                  /* input.input [1,C,4,4] */
  const float* conv_weight[HF_MAX_STYLED];       /* *.conv.weight [1,cout,cin,3,3] */
  const float* conv_mod_weight[HF_MAX_STYLED];   /* *.conv.modulation.weight [cin,style_dim] */
  const float* conv_mod_bias[HF_MAX_STYLED];     /* *.conv.modulation.bias [cin] */
  const float* conv_blur_kernel[HF_MAX_STYLED];  /* *.conv.blur.kernel [4,4] (upsampling convs) */
  const float* conv_noise_weight[HF_MAX_STYLED]; /* *.noise.weight [1] */
  const float* conv_act_bias[HF_MAX_STYLED];     /* *.activate.bias [cout] */
  const float* rgb_weight[HF_MAX_TORGB];         /* *.conv.weight [1,3,cin,1,1] */
  const float* rgb_mod_weight[HF_MAX_TORGB];
  const float* rgb_mod_bias[HF_MAX_TORGB];
  const float* rgb_bias[HF_MAX_TORGB];           /* *.bias [1,3,1,1] */
  const float* rgb_up_kernel[HF_MAX_TORGB];      /* *.upsample.kernel [4,4] (NULL for to_rgb1) */
} hf_gen_weights;

size_t hf_generator_packed_bytes(const hf_gen_config* cfg);
size_t hf_generator_workspace_bytes(const hf_gen_config* cfg, int batch);

/* One-time repack of the generator parameters (what Net.load_weights feeds, models/Net.py:37-42). */
int hf_generator_pack(const hf_gen_config* cfg, const hf_gen_weights* w, void* packed, void* stream);

typedef struct {
  int batch;
  const float* latent;   /* [B, n_latent, style_dim] fp32 (input_is_latent=True, model.py:521-522) */
  const float* noise[HF_MAX_STYLED]; /* per styled conv: [noise_batch,1,R,R] fp32 (explicit; the host
                                        draws random noise in reference order, model.py:288-291) */
  int noise_batch[HF_MAX_STYLED];    /* 1 = shared across the batch (registered buffers), or B */
  int start_layer, end_layer;        /* model.py:488-489 */
  const float* layer_in; /* [B,C,R,R] fp32 NCHW input of layer start_layer (>0), model.py:546 */
  const float* skip_in;  /* [B,3,R,R] running RGB handed in (forward's `skip`), or NULL */
  float* out_feature;    /* early exit: `out` [B,C,R,R] fp32 NCHW (model.py:537-538,550-551) */
  float* out_rgb;        /* image [B,3,size,size], or the early-exit `skip` [B,3,R,R] */
  /* FeatureStyleEncoder generator variant (pixel2style2pixel/models/stylegan2/model.py:527-560):
   * insert_feature: x = (1-alpha)*x + alpha*feature_in[i] before the styled conv that consumes latent
   * index i (i >= 1; [B,Cin_i,R,R] fp32 NCHW or NULL).  Only alpha == 1 (what HairFast runs:
   * min(1, 1e-4 * n_iter) with n_iter = 1e5, trainer.py:358-359) is implemented.
   * return_features: features_out[0] = ConstantInput output, features_out[i+1] = output of styled conv i
   * ([B,Cout_i,R,R] fp32 NCHW each; NULL entries are skipped). */
  const float* feature_in[HF_MAX_STYLED];
  float feature_alpha;
  float* features_out[HF_MAX_STYLED + 1];
} hf_gen_io;

/* Replaces Generator.forward(styles=[latent], input_is_latent=True, noise=..., layer_in, skip,
 * start_layer, end_layer) (model.py:477-565).  Writes out_rgb (and out_feature on the early exit;
 * *early_exit tells which return form applies: 0 = (image, None), 1 = (out, skip)). */
int hf_generator_forward(const hf_gen_config* cfg, const void* packed, const hf_gen_io* io,
                         void* workspace, int* early_exit /* host */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Encoder backbones on the same convolution kernels (SURVEY 8 rows a13 / a14):
 * e4e Encoder4Editing (models/encoder4editing/models/encoders/psp_encoders.py:124-200, helpers.py:57-140)
 * and FeatureStyleEncoder fs_encoder_v2 (models/FeatureStyleEncoder/nets/feature_style_encoder.py:12-65,
 * arcface/iresnet.py:28-163).  Activations travel as NHWC 16-bit tensors between the calls.
 * ------------------------------------------------------------------------------------------ */

typedef struct {
  int cin, cout;   /* logical channels of the nn.Conv2d */
  int cin_pad;     /* channels of the stored NHWC input (>= cin, multiple of 32 per group; 3 -> 32 for the stem) */
  int ksize;       /* 1 or 3 (padding = ksize / 2) */
  int stride;      /* 1 or 2 */
  int groups;      /* >= 1; used to run the 18 GradualStyleBlock heads as one grouped conv */
  int dtype;
} hf_conv2d_desc;

size_t hf_conv2d_packed_bytes(const hf_conv2d_desc* d);

/* Replaces nn.Conv2d weight handling: weight [cout, cin/groups, k, k] fp32; out_scale [cout] (NULL = 1) is
 * folded into the weights -- the BatchNorm2d that FOLLOWS the conv in bottleneck_IR_SE / IBasicBlock
 * (eval mode: gamma / sqrt(running_var + eps)); its shift goes to hf_conv2d_io.shift. */
int hf_conv2d_pack(const hf_conv2d_desc* d, const float* weight, const float* out_scale, void* packed, void* stream);

typedef struct {
  int batch, height, width; /* input spatial size */
  const void* x16;          /* [B,H,W,cin_pad*] 16-bit NHWC (for groups > 1: cin_pad * groups channels) */
  const float* shift;       /* [cout] conv bias and/or BatchNorm shift, or NULL */
  int act;                  /* 0 none, 1 PReLU(slope[cout]), 2 LeakyReLU(slope0), 3 ReLU */
  const float* slope;       /* [cout] for PReLU */
  float slope0;             /* nn.LeakyReLU() default 0.01 in GradualStyleBlock (psp_encoders.py:42,46) */
  const void* residual16;   /* [B,Ho,Wo,cout] 16-bit NHWC added after the activation, or NULL */
  void* y16;                /* [B,Ho,Wo,cout] 16-bit NHWC or NULL */
  const float* y16b_scale;  /* second output y16b = v * scale[c] + shift[c]: the BatchNorm that PRECEDES the next */
  const float* y16b_shift;  /*   conv (cannot be folded into its weights because of the zero padding)          */
  void* y16b;
  float* y32_nchw;          /* [B,cout,Ho,Wo] fp32 NCHW or NULL */
  int act_after_residual;   /* 0: v = act(conv) + residual (IR blocks); 1: v = act(conv + residual) (ResNet BasicBlock,
                               face_parsing/resnet.py:44-46) */
} hf_conv2d_io;

/* Replaces nn.Conv2d.forward (+ the folded BatchNorm2d / PReLU / LeakyReLU / residual add around it). */
int hf_conv2d_forward(const hf_conv2d_desc* d, const void* packed, const hf_conv2d_io* io, void* stream);

/* x [B,C,H,W] fp32 NCHW -> y16 [B,H,W,c_pad] 16-bit NHWC, y = x*scale[c] + shift[c] (NULL = identity), zero padded */
int hf_nchw_to_nhwc16(const float* x, const float* scale, const float* shift, void* y16, int batch, int channels,
                      int c_pad, int height, int width, int dtype, void* stream);
/* x16 [B,H,W,C] 16-bit NHWC -> y [B,C,H,W] fp32 NCHW */
int hf_nhwc16_to_nchw(const void* x16, float* y, int batch, int channels, int height, int width, int dtype,
                      void* stream);
/* Scratch (bytes) for the two-stage deterministic channel reduction below. */
size_t hf_channel_reduce_workspace_bytes(int batch, int hw, int channels);
/* SEModule.avg_pool (helpers.py:60): mean over H*W -> [B,C] fp32.  channels % 8 == 0. */
int hf_channel_mean_nhwc16(const void* x16, float* mean, void* workspace, int batch, int hw, int channels, int dtype,
                           void* stream);
/* Whole SEModule gate (helpers.py:57-75): gate[b,c] = sigmoid(fc2 . relu(fc1 . mean_hw(x)));
 * fc1_weight [reduced, channels], fc2_weight [channels, reduced] fp32 (the bias-free 1x1 convs). */
int hf_se_gate_nhwc16(const void* x16, const float* fc1_weight, const float* fc2_weight, float* gate, void* workspace,
                      int batch, int hw, int channels, int reduced, int dtype, void* stream);
/* bottleneck_IR_SE tail (helpers.py:117-120): out = res * se[b,c] + shortcut[b, y*s, x*s, c];
 * se / shortcut16 / y16 / y16b may be NULL; y16b = out * s2[c] + b2[c] */
int hf_scale_add_nhwc16(const void* res16, const float* se, const void* shortcut16, int shortcut_stride,
                        const float* s2, const float* b2, void* y16, void* y16b, int batch, int height, int width,
                        int channels, int dtype, void* stream);
/* _upsample_add (helpers.py:123-140): bilinear(align_corners=True) upsample of x16 [B,h,w,C] to HxW, plus y16 */
int hf_upsample_add_nhwc16(const void* x16, const void* y16, void* out16, int batch, int h, int w, int height,
                           int width, int channels, int dtype, void* stream);
/* nn.AdaptiveAvgPool2d((oh,ow)) -> fp32 NCHW [B,C,oh,ow] */
int hf_adaptive_avgpool_nhwc16(const void* x16, float* y, int batch, int height, int width, int channels, int oh,
                               int ow, int dtype, void* stream);

/* ---- BiSeNet face parsing (models/CtrlHair/external_code/face_parsing/{model,resnet}.py) ---- */
/* 3x3 RGB stem of the IR-SE / iresnet encoders fused: Conv2d(3,64,3,1,1) + eval BatchNorm + PReLU
 * (psp_encoders.py:176-178 input_layer; arcface/iresnet.py:92-95 conv1/bn1/prelu).  x [B,3,H,W] fp32 NCHW ->
 * y16 [B,H,W,64] = prelu(conv*bn_scale + shift) and, when y16b != NULL, y16b = y16 * s2[c] + b2[c] (the first block's
 * leading BatchNorm), both 16-bit NHWC.  wpacked: 16-bit [64][56], row n = weight[n,c,ky,kx] * bn_scale[n] at
 * k = ky*16 + kx*4 + c (c < 3, kx < 3), zero elsewhere; shift / slope / s2 / b2: [64] fp32. */
int hf_stem3x3_nhwc16(const float* x, const void* wpacked, const float* shift, const float* slope, const float* s2,
                      const float* b2, void* y16, void* y16b, int batch, int height, int width, int dtype, void* stream);

/* Resnet18.conv1 7x7/s2/p3 + bn1 + ReLU fused (face_parsing/resnet.py:60-61,69-70): x [B,3,H,W] fp32 NCHW ->
 * y16 [B,(H+1)/2,(W+1)/2,64] 16-bit NHWC.  wpacked: 16-bit [64][184], row n = weight[n,c,ky,kx] * bn_scale[n] at
 * k = ky*24 + kx*3 + c (k < 168, kx*3+c < 21), zero elsewhere; shift [64] fp32 = the BatchNorm shift. */
int hf_stem7x7s2_nhwc16(const float* x, const void* wpacked, const float* shift, void* y16, int batch, int height,
                        int width, int dtype, void* stream);

/* im2col for Resnet18.conv1 (resnet.py:60,69; 7x7 / stride 2 / pad 3 on 3 channels): x [B,3,H,W] fp32 NCHW ->
 * y16 [B,Ho,Wo,160] 16-bit NHWC, channel k = (c*7 + ky)*7 + kx (= the flattening of the conv weight [64,3,7,7]),
 * zero for k >= 147 and outside the image; Ho = (H-1)/2+1.  The stem is then hf_conv2d_forward with
 * {cin 147, cin_pad 160, ksize 1} and the folded bn1 + ReLU epilogue. */
int hf_im2col7x7s2_nhwc16(const float* x, void* y16, int batch, int height, int width, int dtype, void* stream);
/* nn.MaxPool2d(3, 2, 1) (resnet.py:62,71) on 16-bit NHWC; output (H-1)/2+1 x (W-1)/2+1 */
int hf_maxpool3x3s2_nhwc16(const void* x16, void* y16, int batch, int height, int width, int channels, int dtype,
                           void* stream);
/* 1x1 conv of the globally pooled feature + folded BatchNorm + activation (act: 0 none, 1 ReLU, 2 sigmoid):
 * out[b,o] = act((sum_c weight[o,c] * mean_hw(x)[b,c]) * scale[o] + shift[o]); scale / shift may be NULL.
 * AttentionRefinementModule attention (model.py:82-86), ContextPath.conv_avg (model.py:114-115).
 * workspace: hf_channel_reduce_workspace_bytes(batch, hw, channels). */
int hf_pooled_fc_nhwc16(const void* x16, const float* weight, const float* scale, const float* shift, int act,
                        float* out, void* workspace, int batch, int hw, int channels, int cout, int dtype,
                        void* stream);
/* ContextPath merge (model.py:116-128): y[b,Y,X,c] = x[b,Y/up,X/up,c]*gate[b,c] + addvec[b,c] + addt[b,Y/up,X/up,c];
 * up = 1 or 2 (F.interpolate nearest); gate / addvec / addt16 may be NULL; height, width = input size. */
int hf_gate_add_up_nhwc16(const void* x16, const float* gate, const float* addvec, const void* addt16, void* y16,
                          int batch, int height, int width, int channels, int up, int dtype, void* stream);
/* F.interpolate(bilinear, align_corners=True) (model.py:239-241) of the first `channels` of `in_channels` planes:
 * x [B,in_channels,h,w] -> y [B,channels,height,width], fp32 NCHW */
int hf_bilinear_upsample_nchw_f32(const float* x, float* y, int batch, int channels, int in_channels, int h, int w,
                                  int height, int width, void* stream);

/* Fused upsample + arg-max for face parsing: labels[b,Y,X] = argmax_c of the bilinear (align_corners=True)
 * interpolation of x[b,c] to (height, width) -- BiSeNet.forward's F.interpolate (face_parsing/model.py:239) followed
 * by `out.squeeze(0).argmax(0)` (face_parsing/my_parsing_util.py:87-88).  Same arithmetic as
 * hf_bilinear_upsample_nchw_f32, first maximum wins (torch.argmax).  labels: int64 [B,height,width]. */
int hf_bilinear_argmax_nchw_f32(const float* x, long long* labels, int batch, int channels, int in_channels, int h,
                                int w, int height, int width, void* stream);

/* ---- stage glue ---- */
/* BicubicDownSample.forward (utils/bicubic.py:36-78): reflect-pad + separable `4*factor`-tap FIR + decimation by
 * `factor`, vertical pass first.  x [planes,H,W] -> y [planes,H/factor,W/factor] fp32; kernel [4*factor] = the
 * normalised taps of BicubicDownSample.__init__ (:20-33); clip_round != 0 applies clamp(round(v), 0, 255) after each
 * pass (:63-64,68-69).  factor 1..8. */
int hf_bicubic_downsample_f32(const float* x, const float* kernel, float* y, int planes, int height, int width,
                              int factor, int clip_round, void* stream);

/* DilateErosion.mask (utils/image_utils.py:42-55): `iterations` rounds of {3x3 cross sum with zero padding; dilation
 * keeps sum > 0, erosion keeps sum == 5}, both started from `mask` [planes,H,W] fp32 (values 0 / 1).
 * workspace: 4 * planes * H * W floats (unused when iterations <= 1). */
int hf_dilate_erode_f32(const float* mask, float* dilate, float* erode, void* workspace, int planes, int height,
                        int width, int iterations, void* stream);

/* Mask algebra of the F-space alignment (models/Alignment.py:139-143): from the three 0/1 hair masks [n] each,
 * masks = [1 - (1 - hm1)(1 - hmx), hmx, hm2 * hmx] -> `masks` [3, n] fp32 (the input of DilateErosion.mask, :145). */
int hf_align_masks_f32(const float* hair_mask1, const float* hair_mask2, const float* hair_mask_target, float* masks,
                       int n, void* stream);

/* F-space blend chain (models/Alignment.py:153-159; with one stage: the Embedding mixing, models/Embedding.py:86-92):
 *   w_s = scale_a[s] + scale_b[s] * F.interpolate(mask[s] [mask_height, mask_width], size=(height, width), 'bicubic')
 *   F   = src[s] + w_s * (F - src[s])   for s = 0 .. n_stage-1, F starting from `first`
 * first, src[s], out: [channels, height, width] fp32; w_s broadcasts over channels; src / mask are HOST arrays of
 * n_stage device pointers, scale_a / scale_b HOST arrays of n_stage floats (1 <= n_stage <= 4).  Alignment uses
 * (scale_a, scale_b) = (1, -1) (`interpolation_low = 1 - free_mask_down_32`), Embedding (0, opts.mixing). */
int hf_fspace_blend_f32(const float* first, const float* const* src, const float* const* mask, const float* scale_a,
                        const float* scale_b, float* out, int n_stage, int channels, int height, int width,
                        int mask_height, int mask_width, void* stream);

/* Number of kernels the last hf_generator_forward / hf_conv_forward of this thread launched. */
int hf_last_launch_count(void);
/* Number of kernels every hf_* call of this thread has launched since the library was loaded. */
long long hf_total_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* HAIRFAST_B200_H_ */
