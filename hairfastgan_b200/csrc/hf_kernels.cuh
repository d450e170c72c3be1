// Internal launcher declarations shared by the translation units of libhairfast_sm90.so.
#pragma once
#include "hf_common.cuh"

namespace hf {

void count_launch(int n = 1);
void reset_launch_count();

// ---- hf_ops.cu : HBM-bound SIMT kernels ------------------------------------------------------
int launch_upfirdn2d(const float* x, float* y, const float* k, int planes, int in_h, int in_w, int kh, int kw,
                     int up_x, int up_y, int down_x, int down_y, int px0, int px1, int py0, int py1,
                     cudaStream_t st);
int launch_bias_act(const float* x, const float* b, float* y, int64_t n, int size_b, int64_t step_b, int act,
                    float alpha, float scale, cudaStream_t st);

struct AffineJob {      // s[b,i] = wscale * sum_j style[b, j] * mw[i,j] + mb[i]   (EqualLinear, lr_mul=1)
  const float* mw;      // [C, D]
  const float* mb;      // [C]
  const float* style;   // row b at style + b*style_stride
  float* s;             // [B, C]
  int C;
  float wscale;         // 1/sqrt(D)
  int block_begin;      // first block of this job (prefix sum; filled by the launcher)
};
struct DemodJob {       // d[b,o] = rsqrt(sum_i s[b,i]^2 * wsq[o,i] + 1e-8)
  const float* wsq;     // [Cout, Cin]
  const float* s;       // [B, Cin]
  float* d;             // [B, Cout]
  int Cout, Cin;
  int block_begin;
};
constexpr int kMaxJobs = 32;
int launch_affine(AffineJob* jobs, int njobs, int B, int D, int64_t style_stride, cudaStream_t st);
int launch_demod(DemodJob* jobs, int njobs, int B, cudaStream_t st);

// x [B or 1, C, HW] fp32 NCHW  ->  xh [B, HW, C] 16-bit, xh = (blend(x, feat)) * s[b,c]
int launch_modulate_to_nhwc(const float* x, int x_broadcast, const float* s, const float* feat, float alpha,
                            void* xh, int B, int C, int HW, int dtype, cudaStream_t st);

// rgb[b,j,Y,X] = bias[j] + sum_t partial[t][b,j,Y,X] + up2(skip)[b,j,Y,X]
int launch_rgb_combine(const float* partial, int num_partials, const float* bias, const float* skip,
                       const float* up_kernel, float* rgb, int B, int H, int W, cudaStream_t st);

// ToRGB on fp32 NCHW input: y = sum_i w1s[j,i]*s[b,i]*x[b,i,p] + bias[j] + up2(skip)
int launch_torgb_nchw(const float* x, const float* w1, float w_scale, const float* s, const float* bias,
                      const float* skip, const float* up_kernel, float* y, int B, int C, int H, int W,
                      cudaStream_t st);

// weight packing
int launch_pack_conv(const float* w, const float* blur, void* wpk, float* wsq, int Cout, int Cin, int ksize,
                     int up, int nc, int dtype, cudaStream_t st);
int launch_scale_copy(const float* src, float* dst, int64_t n, float scale, cudaStream_t st);

// ---- hf_enc_ops.cu : encoder-side glue kernels -------------------------------------------------
int launch_pack_conv2d(const float* w, const float* out_scale, void* wpk, int cout, int cin_g, int cin_pad, int ksize,
                       int dtype, cudaStream_t st);
int launch_nchw_to_nhwc16(const float* x, const float* scale, const float* shift, void* y16, int B, int C, int Cpad,
                          int HW, int dtype, cudaStream_t st);
int launch_nhwc16_to_nchw(const void* x16, float* y, int B, int C, int HW, int dtype, cudaStream_t st);
int channel_reduce_splits(int B, int HW, int C);
int launch_channel_partial(const void* x16, float* ws, int B, int HW, int C, int dtype, cudaStream_t st, int* splits);
// BiSeNet glue (hf_seg_ops.cu)
int launch_im2col7x7s2(const float* x, void* y16, int B, int H, int W, int dtype, cudaStream_t st);
int launch_stem7x7s2_fused(const float* x, const void* wpacked, const float* shift, void* y16, int B, int H, int W,
                           int dtype, cudaStream_t st);
int launch_stem3x3_fused(const float* x, const void* wpacked, const float* shift, const float* slope, const float* s2,
                         const float* b2, void* y16, void* y16b, int B, int H, int W, int dtype, cudaStream_t st);
int launch_maxpool3x3s2(const void* x16, void* y16, int B, int H, int W, int C, int dtype, cudaStream_t st);
int launch_pooled_fc(const void* x16, const float* w, const float* scale, const float* shift, int act, float* out,
                     float* ws, int B, int HW, int C, int Cout, int dtype, cudaStream_t st);
int launch_gate_add_up(const void* x16, const float* gate, const float* addvec, const void* addt16, void* y16, int B,
                       int h, int w, int C, int up, int dtype, cudaStream_t st);
int launch_bicubic_down(const float* x, const float* k, float* y, int planes, int H, int W, int factor, int clip_round,
                        cudaStream_t st);
int launch_dilate_erode(const float* mask, float* dilate, float* erode, float* ws, int planes, int H, int W,
                        int iterations, cudaStream_t st);
int launch_bilinear_argmax(const float* x, long long* labels, int B, int C, int Cin, int h, int w, int H, int W,
                           cudaStream_t st);
int launch_align_masks(const float* hm1, const float* hm2, const float* hmx, float* out, int n, cudaStream_t st);
int launch_fspace_blend(const float* first, const float* const* src, const float* const* mask, const float* scale_a,
                        const float* scale_b, float* out, int n_stage, int C, int Ho, int Wo, int Hm, int Wm,
                        cudaStream_t st);
int launch_bilinear_up_nchw(const float* x, float* y, int B, int C, int Cin, int h, int w, int H, int W,
                            cudaStream_t st);
int launch_se_gate(const void* x16, const float* fc1, const float* fc2, float* out, float* ws, int B, int HW, int C,
                   int Cr, int dtype, cudaStream_t st);
int launch_scale_add(const void* res16, const float* se, const void* shortcut16, int sc_stride, const float* s2,
                     const float* b2, void* y16, void* y16b, int B, int H, int W, int C, int dtype, cudaStream_t st);
int launch_upsample_add(const void* x16, const void* y16, void* out16, int B, int h, int w, int H, int W, int C,
                        int dtype, cudaStream_t st);
int launch_adaptive_avgpool(const void* x16, float* y, int B, int H, int W, int C, int oh, int ow, int dtype,
                            cudaStream_t st);
int ensure_device_current();

// ---- hf_conv_tc.cu : wgmma implicit-GEMM convolution ----------------------------------------
struct ConvLaunch {
  int B, H, W;            // input spatial size
  int Cin, Cout;
  int taps;               // 9 (3x3, pad 1) or 1 (1x1)
  int up;                 // 1: polyphase stride-2 transposed conv + blur -> output 2H x 2W
  int dtype;
  const void* xhat_in;    // [B,H,W,Cin] 16-bit NHWC (already multiplied by this conv's s[b,cin])
  const void* wpk;        // packed weights [Ntot, taps*Cin] 16-bit
  int nc;                 // couts per N tile the weights were packed for (up only); 0 for plain
  const float* d;         // [B,Cout] demod or NULL
  const float* noise;     // [nb,1,Ho,Wo] or NULL
  int noise_batch;        // 1 or B
  const float* noise_w;   // device scalar or NULL
  const float* bias;      // [Cout] or NULL
  int act;                // 1: lrelu(0.2)*sqrt(2)
  const float* s_next;    // [B,Cout] scale applied to the 16-bit output, or NULL (=1)
  void* xhat_out;         // [B,Ho,Wo,Cout] 16-bit NHWC or NULL
  float* out_nchw;        // [B,Cout,Ho,Wo] fp32 (unscaled) or NULL
  const float* rgb_w;     // [3,Cout] (pre-scaled 1/sqrt(Cout)) or NULL
  const float* rgb_s;     // [B,Cout] ToRGB modulation
  float* rgb_partial;     // [num_n_tiles][B,3,Ho,Wo]
  int force_n_tile;       // 0 = auto
  // ---- plain (encoder) convolution: epi = 1 selects the affine / PReLU / residual epilogue
  int epi;                // 0 generator epilogue, 1 encoder epilogue
  int stride;             // 1 or 2 (0 = 1)
  int groups;             // grouped weights: N tile g reads input channels [g*Cin/groups, ...)
  const float* enc_scale; // [Cout] accumulator scale (NULL = 1)
  const float* enc_shift; // [Cout] bias / BN shift (NULL = 0)
  int enc_act;            // 0 none, 1 PReLU(enc_slope[Cout]), 2 LeakyReLU(enc_slope0), 3 ReLU
  int enc_post;           // 1: the activation follows the residual add
  const float* enc_slope;
  float enc_slope0;
  const void* enc_residual;   // [B,Ho,Wo,Cout] 16-bit NHWC added after the activation, or NULL
  const float* enc_s2;    // second 16-bit output: y16b = v*s2[o] + b2[o] (the consumer's pre-conv BatchNorm)
  const float* enc_b2;
  void* enc_y16b;
};
struct ConvPlan {
  // halo, G, na_slots, pitch, b_resident, a_slot_bytes: halo-tile scheduling fields of the plan query ABI
  // (hf_conv_plan_query); conv_wgmma_kernel loads one box per (tap, channel chunk) and reports 0 / 1 / 0 / 0 / 0 / 0.
  int halo;
  int G;
  int ng;                 // consumer warpgroups (MMA + epilogue), 64 GEMM rows each
  int na_slots, pitch;
  int b_resident;
  uint32_t a_slot_bytes;
  int TW, TH, TB;         // pixel tile: TW*TH*TB = 128 GEMM rows
  int tiles_x, tiles_y, tiles_b, num_m_tiles;
  int n_tile, num_n_tiles, nc;
  int kchunk;             // channels per pipeline stage (64 -> SWIZZLE_128B, 32 -> SWIZZLE_64B)
  int stages;
  size_t smem_bytes;
  int num_tiles, grid;
};
int conv_plan(const ConvLaunch& a, ConvPlan* p);
int conv_up_nc(int Cout);            // couts per N tile used when packing an upsampling conv
int launch_conv(const ConvLaunch& a, cudaStream_t st, ConvPlan* plan_out);

}  // namespace hf
