// Internal launcher declarations shared by the translation units of libhairfast_sm90.so.
#pragma once
#include "hf_common.cuh"

namespace hf {

void count_launch(int n = 1);
void reset_launch_count();
// makes the device of hf_set_device current on this thread (no-op before the first hf_set_device)
int ensure_device_current();

// ---- hf_ops.cu : HBM-bound SIMT kernels ------------------------------------------------------
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
// ConvTranspose2d(3, stride 2, padding 1, output_padding 1) weight [cin, cout, 3, 3] -> the four-parity 3x3 operand
// [4 * cout][9 * cin_pad] of the upsampling conv (row (o / 32) * 128 + parity * 32 + o % 32)
int launch_pack_conv2d_transposed(const float* w, const float* out_scale, void* wpk, int cout, int cin, int cin_pad,
                                  int dtype, cudaStream_t st);
// stage 1 of the deterministic channel reduction of x16 [B,HW,C]: ws[(b*S + s)*C + c] = partial sums, *splits = S
int launch_channel_partial(const void* x16, float* ws, int B, int HW, int C, int dtype, cudaStream_t st, int* splits);

// ---- hf_conv_tc.cu : wgmma implicit-GEMM convolution ----------------------------------------
struct ConvLaunch {
  int B, H, W;            // input spatial size
  int Cin, Cout;
  int taps;               // 9 (3x3, pad 1) or 1 (1x1)
  int prepadded;          // 1: the stored input already carries the 1-pixel border (3x3, stride 1): output (H-2)x(W-2)
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
  // halo, G, pitch, b_resident: fields of the plan query ABI (hf_conv_plan_query) that described the resident-halo
  // scheduler of the B200 kernel this one replaced; conv_wgmma_kernel has no such scheduler and always reports
  // 0 / 1 / 0 / 0.
  int halo;
  int G;
  int ng;                 // consumer warpgroups (MMA + epilogue), 64 GEMM rows each
  int na_slots;           // activation ring slots: kShiftASlots with shift_boxes, 0 on the per-tap path
  int pitch;
  int b_resident;
  // 1: one (TH + 2)-row activation box per (channel chunk, column shift) serves the three row shifts; activation
  // boxes and weight boxes then have separate rings (kShiftASlots slots of a_slot_bytes; `stages` weight slots)
  int shift_boxes;
  uint32_t a_slot_bytes;
  int TW, TH, TB;         // pixel tile: TW*TH*TB = 128 GEMM rows
  int tiles_x, tiles_y, tiles_b, num_m_tiles;
  int n_tile, num_n_tiles, nc;
  int kchunk;             // channels per pipeline stage (64 -> SWIZZLE_128B, 32 -> SWIZZLE_64B)
  int stages;             // ring slots: (activation + weight) boxes, or weight boxes only with shift_boxes
  size_t smem_bytes;
  int num_tiles, grid;
};
int conv_plan(const ConvLaunch& a, ConvPlan* p);
void conv_plan_export(const ConvPlan& pl, int* out /* host[12], the layout of hf_conv_plan_query */);
int conv_up_nc(int Cout);            // couts per N tile used when packing an upsampling conv
int launch_conv(const ConvLaunch& a, cudaStream_t st, ConvPlan* plan_out);

}  // namespace hf
