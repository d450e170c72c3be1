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

/* 16-bit storage/operand type of the tensor-core path (accumulation is always fp32).  A call that takes an
 * `int dtype` returns HF_ERR_INVALID for any other value, before it checks its other arguments. */
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
 * bias may be NULL (size_b = 0): then nothing is added, so y keeps the sign of a zero x like the reference. */
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
  const float* style;        /* [B, style_dim] latent rows for this layer (row stride style_stride); style and
                                mod_weight 16-byte aligned (else HF_ERR_INVALID, nothing launched) */
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
 * conv.  out[12] = {0, n_tile, num_n_tiles, 1, activation ring slots, 0, 0, pipeline stages, dynamic smem bytes,
 * work items (M tiles x N tiles), grid, channels per K chunk}.  out[4] tells the two mainloops apart: the slot count
 * of the activation ring on the column-shift path (stride-1 3x3 on 16 x 8 tiles of one sample), 0 on the per-tap
 * path, whose activation boxes share the ring slots of the weight boxes.  out[0], out[3], out[5] and out[6] are
 * constants kept for callers of the earlier layout. */
int hf_conv_plan_query(const hf_conv_desc* d, int batch, int height, int width, int* out /* host[12] */);

/* Replaces ModulatedConv2d.forward (model.py:238-279) / StyledConv.forward (model.py:337-343). */
int hf_conv_forward(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, void* stream);

/* Measurement helper (no reference counterpart): runs hf_conv_forward's prologue once, then the
 * wgmma convolution kernel alone `iters` times between two CUDA events recorded on `stream`, and
 * returns the average kernel duration in milliseconds (host pointer).  Synchronises the stream. */
int hf_conv_time_kernel(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, int iters,
                        float* avg_ms /* host */, void* stream);

/* Replaces ToRGB.forward (model.py:356-365): modulated 1x1 conv without demodulation + bias +
 * Upsample(skip) (model.py:35-53).  x [B,cin,H,W], skip [B,3,H/2,W/2] or NULL, y [B,3,H,W]; fp32.
 * style and mod_weight must be 16-byte aligned (else HF_ERR_INVALID, nothing launched). */
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
  const float* latent;   /* [B, n_latent, style_dim] fp32 (input_is_latent=True, model.py:521-522), 16-byte aligned
                            (else HF_ERR_INVALID, nothing launched) */
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
   * ([B,Cout_i,R,R] fp32 NCHW each; NULL entries are skipped; an early exit still fills out_feature as well). */
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
  /* 1: the stored input already carries the 1-pixel border (e.g. nn.ReflectionPad2d(1), which the TMA zero fill cannot
   * produce): no padding is added and the output is (H-2) x (W-2) of the stored H x W.  ksize 3, stride 1. */
  int prepadded;
  /* 1: nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1): weight [cin, cout, 3, 3], output
   * 2H x 2W.  Runs as four 3x3 correlations, one per output parity (4x the algorithmic FLOPs); stride must be 2,
   * groups 1. */
  int transposed;
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

/* hf_conv_plan_query for the launch hf_conv2d_forward makes at this input size (needs no device): same out[12]. */
int hf_conv2d_plan_query(const hf_conv2d_desc* d, int batch, int height, int width, int* out /* host[12] */);

/* x [B,C,H,W] fp32 NCHW -> y16 [B,H,W,c_pad] 16-bit NHWC, y = x*scale[c] + shift[c] (NULL = identity), zero padded */
int hf_nchw_to_nhwc16(const float* x, const float* scale, const float* shift, void* y16, int batch, int channels,
                      int c_pad, int height, int width, int dtype, void* stream);
/* x16 [B,H,W,C] 16-bit NHWC -> y [B,C,H,W] fp32 NCHW */
int hf_nhwc16_to_nchw(const void* x16, float* y, int batch, int channels, int height, int width, int dtype,
                      void* stream);
/* SEAN's Zencoder (models/sean_codes/models/networks/architecture.py:154-207) around hf_conv2d_forward. */
/* Scratch (bytes) of hf_instance_norm_lrelu_nhwc16. */
size_t hf_instance_norm_workspace_bytes(int batch, int hw, int channels);
/* nn.InstanceNorm2d(affine=False, track_running_stats=False) + nn.LeakyReLU(slope) on x16 [B,HW,C] 16-bit NHWC -> y16
 * (may alias x16): per-(b, c) mean, then the biased variance of the centred values (two passes, eps 1e-5), fp32
 * statistics in a fixed summation order (the reduction of hf_channel_mean_nhwc16).  channels % 8 == 0; x16 and y16
 * 16-byte aligned. */
int hf_instance_norm_lrelu_nhwc16(const void* x16, void* y16, void* workspace, int batch, int hw, int channels,
                                  float slope, int dtype, void* stream);
/* nn.ReflectionPad2d(1): x16 [B,H,W,C] -> y16 [B,H+2,W+2,C] 16-bit NHWC.  H, W >= 2, channels % 8 == 0. */
int hf_reflect_pad1_nhwc16(const void* x16, void* y16, int batch, int height, int width, int channels, int dtype,
                           void* stream);

/* The five calls below move 16 bytes at a time: their 16-bit tensors, and se, must be 16-byte aligned (else
 * HF_ERR_INVALID, nothing launched).  Scratch (bytes) for the two-stage deterministic channel reduction below. */
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

/* nn.MaxPool2d(3, 2, 1) (resnet.py:62,71) on 16-bit NHWC; output (H-1)/2+1 x (W-1)/2+1; both 16-byte aligned */
int hf_maxpool3x3s2_nhwc16(const void* x16, void* y16, int batch, int height, int width, int channels, int dtype,
                           void* stream);
/* 1x1 conv of the globally pooled feature + folded BatchNorm + activation (act: 0 none, 1 ReLU, 2 sigmoid):
 * out[b,o] = act((sum_c weight[o,c] * mean_hw(x)[b,c]) * scale[o] + shift[o]); scale / shift may be NULL.
 * AttentionRefinementModule attention (model.py:82-86), ContextPath.conv_avg (model.py:114-115).
 * workspace: hf_channel_reduce_workspace_bytes(batch, hw, channels); x16 16-byte aligned. */
int hf_pooled_fc_nhwc16(const void* x16, const float* weight, const float* scale, const float* shift, int act,
                        float* out, void* workspace, int batch, int hw, int channels, int cout, int dtype,
                        void* stream);
/* ContextPath merge (model.py:116-128): y[b,Y,X,c] = x[b,Y/up,X/up,c]*gate[b,c] + addvec[b,c] + addt[b,Y/up,X/up,c];
 * up = 1 or 2 (F.interpolate nearest); gate / addvec / addt16 may be NULL; height, width = input size; the 16-bit
 * tensors 16-byte aligned. */
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
 * (scale_a, scale_b) = (1, -1) (`interpolation_low = 1 - free_mask_down_32`), Embedding (0, opts.mixing).
 * No pointer needs more than 4-byte alignment: when first, a src[s] or out is not 16-byte aligned the kernel reads and
 * writes 4 bytes at a time instead of 16.  NULL first, src, mask, scale_a, scale_b, out or a NULL src[s] / mask[s] is
 * an error. */
int hf_fspace_blend_f32(const float* first, const float* const* src, const float* const* mask, const float* scale_a,
                        const float* scale_b, float* out, int n_stage, int channels, int height, int width,
                        int mask_height, int mask_width, void* stream);

/* ---- SEAN decode_sean (models/sean_codes/models/pix2pix_model.py:309-325, UI_mode, batch 1) ----
 * The SPADE generator's block convolutions run on hf_conv2d_forward; these calls supply the rest. */

/* labels: int64 [size,size] (the `target_mask` label values) -> maps: int8 label maps at R = size/32, size/16, ..., size
 * concatenated in that order (R = 8..256 for size 256), L_R[y,x] = label[y*size/R, x*size/R] (F.interpolate nearest,
 * generator.py:75, normalization.py:115).  *bad (device int) = number of labels outside 0..18. */
int hf_sean_labels(const long long* labels, int8_t* maps, int* bad, int size, void* stream);

/* 3x3 zero-padded convolution of the one-hot map of `labels` [res,res] (19 classes) as a table lookup:
 * y16[p,c] = act(bias[c] + sum_{tap, p+tap inside} table[tap][L(p+tap)][c]); table [9][19][channels] fp32 =
 * weight[c, j, ky, kx] at tap = ky*3 + kx; bias [channels] or NULL; act 0 none / 3 ReLU; y16 [res,res,channels]
 * 16-bit NHWC.  SPADEGenerator.fc (generator.py:33,75-76) and every SPADE.mlp_shared (normalization.py:241-253). */
int hf_sean_onehot_conv(const int8_t* labels, const float* table, const float* bias, int act, void* y16, int res,
                        int channels, int dtype, void* stream);

/* One ACE layer's style-table operands (all fp32, device). */
typedef struct {
  const float* fc_w;   /* [19][512][512]: fc_mu{j}.weight */
  const float* fc_b;   /* [19][512]: fc_mu{j}.bias */
  const float* tw;     /* [9*n2][512]: row tap*n2 + n = [a_g conv_gamma.weight; a_b conv_beta.weight][n, :, tap] */
  float* table;        /* out: [19][9][n2] */
  int n2;              /* 2 * norm_nc */
} hf_sean_ace_tables;

/* Per-call style tables of n_ace (<= 16) ACE layers in two launches:
 * code_j = image_code[j] ([19][512]) unless that row is all zero, then mean_code[j] (pix2pix_model.py:312-315);
 * mu_j = relu(fc_w[j] . code_j + fc_b[j]) (normalization.py:133-135); table[j][tap][n] = tw[tap*n2 + n] . mu_j.
 * aces: HOST array; mu_workspace: n_ace * 19 * 512 floats.  image_code, mean_code, mu_workspace and every ACE's fc_w
 * and tw are read with 16-byte loads: each must be 16-byte aligned. */
int hf_sean_style_tables(const float* image_code, const float* mean_code, const hf_sean_ace_tables* aces, int n_ace,
                         float* mu_workspace, void* stream);

/* ACE.forward (normalization.py:108-189) + optional leaky_relu(0.2) (architecture.py:95-96), batch 1:
 * v = (x + noise[w*res + h] * noise_var[c]) * bn_scale[c] + bn_shift[c]; g / b = gamma_beta[c] / gamma_beta[C + c]
 * (+ sum over valid taps of table[L(p+tap)][tap][c] / [C + c] when table != NULL); out = v * (1 + g) + b.
 * x16 / y16 [res,res,channels] 16-bit NHWC; noise [res*res] (torch.randn(1, W, H, 1)); gamma_beta [2C,res,res] fp32
 * NCHW; table [19][9][2C] fp32 (hf_sean_style_tables) or NULL; labels [res,res].  res^2 % 32 == 0, channels % 64 == 0. */
int hf_sean_ace_apply(const void* x16, const float* noise, const float* noise_var, const float* bn_scale,
                      const float* bn_shift, const float* gamma_beta, const float* table, const int8_t* labels,
                      int lrelu, void* y16, int res, int channels, int dtype, void* stream);

/* tanh(conv_img(leaky_relu(x, 0.2))) (generator.py:107-108): x16 [res,res,channels] 16-bit NHWC, weight [3][channels]
 * [3][3], bias [3] -> y [3,res,res] fp32 NCHW.  channels % 8 == 0, <= 256; x16 16-byte aligned. */
int hf_sean_conv_img(const void* x16, const float* weight, const float* bias, float* y, int res, int channels,
                     int dtype, void* stream);

/* Zencoder.forward's tail (architecture.py:177-207) for one batch: codes[b][j][c] = mean over the pixels p with
 * labels[b * label_stride + p] == j of tanh(y[b][c][p]), exactly 0 where class j has no pixel.  y [B,channels,hw]
 * fp32 NCHW (the last conv's output, bias included); labels int8 (hf_sean_labels' 128^2 level per sample); codes
 * [B,19,channels] fp32.  Fixed summation order, no atomics. */
int hf_sean_class_means(const float* y, const int8_t* labels, long long label_stride, float* codes, int batch,
                        int channels, int hw, void* stream);

/* ---- CtrlHair shape adaptor (models/CtrlHair/shape_branch/model.py:146-199) ---- */
/* mask_label_to_one_hot's label side (shape_util.py:6-14): mask [n] int64 is rewritten 255 -> 19 in place; labels
 * [n] int8 gets 0..19 (19 = the all-zero one-hot); *bad = the count of values outside {0..19, 255}. */
int hf_shape_labels(long long* mask, int8_t* labels, int* bad, int n, void* stream);

/* MaskEncoder layer 0 (ZeroPad 1 + Conv 4x4 stride 2) as a lookup: y16[p][c] = cmap[p][c] + sum over the taps inside
 * the (2 res)^2 label map of table[tap][label][c].  labels [2res][2res] int8 (hf_shape_labels); table [16][20][channels]
 * fp32 (tap = ky*4 + kx); cmap [res*res][channels] fp32 (positional channels' conv + bias); y16 [res,res,channels]
 * 16-bit NHWC.  channels % 8 == 0. */
int hf_shape_onehot_s2(const int8_t* labels, const float* table, const float* cmap, void* y16, int res, int channels,
                       int dtype, void* stream);

/* Split-K GEMM with compact 16-bit weights w16 [cout][K] (k = tap*cin + c) and the im2col gathered from x16
 * [hin,win,cin] 16-bit NHWC.  mode 0: 1x1 / Linear (P = hin*win, K = cin); mode 1: ZeroPad 1 + Conv 4x4 stride 2
 * (P = hin/2 * win/2, K = 16 cin); mode 2: nearest 2x upsample + Conv 3x3 pad 1 (P = 4 hin win, K = 9 cin).
 * y[p][co] = bias[co] + sum_k (fp32 partials per split, added in split order) -> y32 fp32 and / or y16 16-bit, both
 * [P][cout].  cin % 8 == 0; workspace hf_shape_gemm_workspace_bytes. */
int hf_shape_gemm(int mode, const void* w16, const void* x16, const float* bias, float* y32, void* y16, float* workspace,
                  int cin, int cout, int hin, int win, int dtype, void* stream);
size_t hf_shape_gemm_workspace_bytes(int mode, int cin, int cout, int hin, int win);
/* The plan hf_shape_gemm picks on a device with `sms` SMs (needs no device): out[5] = {pixel tile, K splits, 64-wide
 * K tiles, cout tiles, pixel tiles}. */
int hf_shape_gemm_plan(int mode, int cin, int cout, int hin, int win, int sms, int* out);

/* CtrlHair LayerNorm (my_torchlib/module.py:183-205) over the whole [pixels, channels] 16-bit NHWC sample, then
 * LeakyReLU(slope): (x - mean) / (unbiased std + 1e-5) * gamma[c] + beta[c].  Fixed-order fp32 statistics.
 * workspace hf_shape_layer_norm_workspace_bytes(pixels * channels). */
int hf_shape_layer_norm_lrelu(const void* x16, const float* gamma, const float* beta, void* y16, float* workspace,
                              int pixels, int channels, float slope, int dtype, void* stream);
size_t hf_shape_layer_norm_workspace_bytes(long long n);

/* Both decoders' out_layer (Conv 3x3 pad 1 over the 32-channel maps hair16 / face16 [res,res,32] 16-bit NHWC) and the
 * argmax over cat[face[:13], hair, face[13:]]: table [19][9][32] fp32 in that channel order, bias [19];
 * labels [res*res] int64, ties to the first index. */
int hf_shape_logits_argmax(const void* hair16, const void* face16, const float* table, const float* bias,
                           long long* labels, int res, int dtype, void* stream);

/* ---- HairFast's latent modulation stacks (models/Encoders.py:13-137) ---- */
/* One call covers `stacks` stacks of 5 ModulationModule(layers, inp, middle) for `batch` samples: rows = batch *
 * layers.  Branch j of a stack (0..9) is module j / 2's gamma_function (j even) or beta_function (j odd).  Every call
 * taking a descriptor returns HF_ERR_INVALID ("<call>: bad dtype N") for a dtype other than HF_BF16 / HF_F16 before
 * it checks its other arguments.  Supported: 1 <= layers <= 24, inp = 512 * n with n * stacks <= 3, middle a multiple
 * of 256 up to 1024, stacks 1 or 2. */
typedef struct {
  int layers; /* L, rows per sample */
  int inp;    /* embedding width */
  int middle; /* gamma / beta hidden width */
  int stacks; /* 1, or 2 for PostProcessModel's to_latent_1 / to_latent_2 */
  int dtype;  /* HF_BF16 / HF_F16: operands, hidden rows */
} hf_mod_desc;
/* fp32 rows [batch][layers][512] with unit column stride; strides in elements (0 broadcasts). */
typedef struct {
  const float* ptr;
  long long batch_stride;
  long long row_stride;
} hf_mod_rows;

/* Scratch of hf_mod_gemm, hf_mod_hidden and hf_mod_chain for one call's descriptor and batch (needs a device). */
size_t hf_mod_workspace_bytes(const hf_mod_desc* d, int batch);
/* The split-K plan of style layer 1 or 2 on a device with `sms` SMs (needs no device): out[5] = {row tile, K splits,
 * 64-wide K tiles, output tiles, row tiles}. */
int hf_mod_gemm_plan(const hf_mod_desc* d, int batch, int layer, int sms, int* out);
/* The 16-bit embedding e16 [stacks][rows][inp]: stack s's columns 512 j .. 512 j + 511 are src[s * inp / 512 + j].
 * e16 must be 16-byte aligned. */
int hf_mod_embed16(const hf_mod_desc* d, int batch, const hf_mod_rows* src, void* e16, void* stream);
/* Grouped split-K GEMM of style layer 1 or 2, y32 = x16 w16^T + bias, partials added in split order:
 *   layer 1: stacks groups, w16 [stacks][10 middle][inp], x16 = e16 [stacks][rows][inp], bias [stacks][10 middle],
 *            y32 [stacks][rows][10 middle];
 *   layer 2: 10 stacks groups, w16 [10 stacks][512][middle], x16 = h16 [rows][10 stacks middle] (group g reads
 *            columns g middle ..), bias [10 stacks][512], y32 = gamma / beta [10 stacks][rows][512].
 * bias may be NULL.  w16 and x16 must be 16-byte aligned. */
int hf_mod_gemm(const hf_mod_desc* d, int batch, int layer, const void* w16, const void* x16, const float* bias,
                float* y32, float* workspace, void* stream);
/* Style layer 1 with the rest of Linear -> LayerNorm([middle]) -> LeakyReLU(0.01) fused into its reduction:
 * h16[p][(s 10 + j) middle + n] for branch j of stack s; bias [stacks][10 middle], ln_w / ln_b [stacks][10][middle]
 * (biased variance, eps 1e-5).  w16 and e16 must be 16-byte aligned, h16 2-byte aligned. */
int hf_mod_hidden(const hf_mod_desc* d, int batch, const void* w16, const void* e16, const float* bias,
                  const float* ln_w, const float* ln_b, void* h16, float* workspace, void* stream);
/* The fc chain on thread-block clusters of 8 CTAs per (stack, sample): PixelNorm over the layers of x0[s], then per
 * module fc (fc_w16 [stacks][5][512][512], fc_b [stacks][5][512]), LayerNorm over the whole [layers, 512] sample,
 * x (1 + gamma) + beta (gb from hf_mod_gemm layer 2) and LeakyReLU(0.01) except after the last module.
 * out [batch][layers][512] = base + 0.1 dt for one stack, base + 0.1 (dt_0 + dt_1) for two.  One kernel launch; with
 * two stacks it is preceded by a cudaMemsetAsync of the completion counters in the workspace.  fc_w16 must be 16-byte
 * aligned. */
int hf_mod_chain(const hf_mod_desc* d, int batch, const void* fc_w16, const float* fc_b, const float* gb,
                 const hf_mod_rows* x0, const hf_mod_rows* base, float* out, float* workspace, void* stream);

/* ---- FFHQ face alignment after the landmarks (utils/shape_predictor.py:145-185) ---- */
/* Images are uint8 RGB, [rows][pitch][3] with `pitch` >= width pixels per row.  Every stage computes what the library
 * call it replaces computes (DESIGN.md, "Face alignment"). */
/* Pillow's LANCZOS resampling of one axis from in_size to out_size: taps per output, and the coefficient table
 * [out_size][taps + 2] int32 (first input, input count, 22-bit fixed-point weights), computed on the host with libm
 * (needs no device).  taps returns -1 for a size <= 0. */
int hf_align_lanczos_taps(int in_size, int out_size);
int hf_align_lanczos_coeffs(int in_size, int out_size, int* table);
/* Image.resize((Wo, Ho), LANCZOS): horizontal pass (coeff_x = table(W, Wo)) into the workspace, then vertical pass
 * (coeff_y = table(H, Ho)) into dst [Ho][Wo][3]; a pass whose size does not change is skipped.  Device tables.
 * workspace hf_align_resample_workspace_bytes(H, W, Ho, Wo) bytes (0: none needed). */
size_t hf_align_resample_workspace_bytes(int H, int W, int Ho, int Wo);
int hf_align_resample_u8(const uint8_t* src, int H, int W, int src_pitch, uint8_t* dst, int Ho, int Wo,
                         const int* coeff_x, const int* coeff_y, uint8_t* workspace, void* stream);
/* The padding branch (:170-178) on src [H][W]: pad = {left, top, right, bottom} (host, each > 0), weights = the
 * scipy Gaussian of sigma qsize * 0.02 from its centre outwards, [radius + 1] float64 on the device; dst [H + top +
 * bottom][W + left + right][3].  workspace hf_align_pad_blend_workspace_bytes(Hp, Wp) of the padded size.
 * 13 launches: pad, two blur axes, median init and 4 x (histogram, select), blend. */
size_t hf_align_pad_blend_workspace_bytes(int Hp, int Wp);
int hf_align_pad_blend_u8(const uint8_t* src, int H, int W, int src_pitch, const int* pad, const double* weights,
                          int radius, uint8_t* dst, void* workspace, void* stream);
/* Its stages on their own: gaussian_filter(x, [s, s, 0]) of x, y [Hp][Wp][3] float32 (workspace Hp Wp 3 floats), and
 * np.median(x, axis=(0, 1)) of x [pixels][3] float32 into med[3] (workspace hf_align_median_workspace_bytes()). */
int hf_align_gaussian_f32(const float* x, float* y, int Hp, int Wp, const double* weights, int radius,
                          float* workspace, void* stream);
size_t hf_align_median_workspace_bytes(void);
int hf_align_median_f32(const float* x, long long pixels, float* med, void* workspace, void* stream);
/* Image.transform((out_w, out_h), QUAD, data, BILINEAR) of src [H][W]: coeffs (host) = the 8 bilinear coefficients
 * Pillow derives from the 8 corner values (x0, (ne_x - x0) / w, ..., see face_align.quad_coefficients). */
int hf_align_quad_u8(const uint8_t* src, int H, int W, int src_pitch, const double* coeffs, uint8_t* dst, int out_w,
                     int out_h, void* stream);

/* Number of kernels the last hf_generator_forward / hf_conv_forward of this thread launched. */
int hf_last_launch_count(void);
/* Number of kernels every hf_* call of this thread has launched since the library was loaded. */
long long hf_total_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* HAIRFAST_B200_H_ */
