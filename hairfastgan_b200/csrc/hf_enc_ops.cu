// Encoder-side kernels around the wgmma convolution (SURVEY 8 rows a13 / a14): plain-conv weight packing
// (BatchNorm scale folded per output channel), NCHW fp32 <-> NHWC 16-bit conversion, squeeze-excite pooling
// and combine, FPN bilinear upsample-add, adaptive average pooling.  All HBM-bound SIMT, fp32 math.
#include <algorithm>

#include "hf_kernels.cuh"

namespace hf {

static inline int cdiv_i(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

template <int DT>
__device__ __forceinline__ float ld16(const uint16_t* p) { return Half2T<DT>::to_float(*p); }

// wpk[o][tap*cin_pad + c] = w[o, c, tap] * out_scale[o]   (c >= cin -> 0: channel padding of the input)
template <int DT>
__global__ void __launch_bounds__(256) pack_conv2d_kernel(const float* __restrict__ w, const float* __restrict__ osc,
                                                          uint16_t* __restrict__ wpk, int cout, int cin_g,
                                                          int cin_pad, int taps) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= (int64_t)cout * cin_pad) return;
  const int c = (int)(idx % cin_pad), o = (int)(idx / cin_pad);
  const float sc = osc ? osc[o] : 1.f;
  const size_t K = (size_t)taps * cin_pad;
  for (int t = 0; t < taps; ++t) {
    const float v = c < cin_g ? w[((size_t)o * cin_g + c) * taps + t] * sc : 0.f;
    wpk[(size_t)o * K + (size_t)t * cin_pad + c] = Half2T<DT>::one(v);
  }
}

int launch_pack_conv2d(const float* w, const float* out_scale, void* wpk, int cout, int cin_g, int cin_pad, int ksize,
                       int dtype, cudaStream_t st) {
  HF_REQUIRE(w && wpk, "pack_conv2d: null pointer");
  HF_REQUIRE(cin_pad >= cin_g && cin_pad % 32 == 0, "pack_conv2d: cin_pad=%d must be >= cin and a multiple of 32", cin_pad);
  const int taps = ksize * ksize;
  const int grid = cdiv_i((int64_t)cout * cin_pad, 256);
  if (dtype == HF_BF16)
    pack_conv2d_kernel<HF_BF16><<<grid, 256, 0, st>>>(w, out_scale, (uint16_t*)wpk, cout, cin_g, cin_pad, taps);
  else
    pack_conv2d_kernel<HF_F16><<<grid, 256, 0, st>>>(w, out_scale, (uint16_t*)wpk, cout, cin_g, cin_pad, taps);
  HF_LAUNCH_OK("pack_conv2d");
  count_launch();
  return HF_OK;
}

// x [B,C,HW] fp32 -> y16 [B,HW,Cpad]; y = x*scale[c] + shift[c]; channels >= C are zero
template <int DT>
__global__ void __launch_bounds__(256) nchw_to_nhwc16_kernel(const float* __restrict__ x, const float* __restrict__ sc,
                                                             const float* __restrict__ sh, uint16_t* __restrict__ y,
                                                             int C, int Cpad, int HW) {
  __shared__ float tile[64][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 64, p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = c0 + ty + 8 * k, p = p0 + tx;
    float v = 0.f;
    if (c < C && p < HW) {
      v = __ldg(x + ((size_t)b * C + c) * HW + p);
      if (sc) v *= __ldg(sc + c);
      if (sh) v += __ldg(sh + c);
    }
    tile[ty + 8 * k][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int p = p0 + ty + 8 * k, c = c0 + 2 * tx;
    if (p < HW && c < Cpad)
      *reinterpret_cast<uint32_t*>(y + ((size_t)b * HW + p) * Cpad + c) =
          Half2T<DT>::pack(tile[2 * tx][ty + 8 * k], tile[2 * tx + 1][ty + 8 * k]);
  }
}

int launch_nchw_to_nhwc16(const float* x, const float* scale, const float* shift, void* y16, int B, int C, int Cpad,
                          int HW, int dtype, cudaStream_t st) {
  HF_REQUIRE(x && y16, "nchw_to_nhwc16: null pointer");
  HF_REQUIRE(Cpad >= C && Cpad % 2 == 0, "nchw_to_nhwc16: bad channel padding %d for %d", Cpad, C);
  dim3 grid(cdiv_i(HW, 32), cdiv_i(Cpad, 64), B);
  if (dtype == HF_BF16)
    nchw_to_nhwc16_kernel<HF_BF16><<<grid, 256, 0, st>>>(x, scale, shift, (uint16_t*)y16, C, Cpad, HW);
  else
    nchw_to_nhwc16_kernel<HF_F16><<<grid, 256, 0, st>>>(x, scale, shift, (uint16_t*)y16, C, Cpad, HW);
  HF_LAUNCH_OK("nchw_to_nhwc16");
  count_launch();
  return HF_OK;
}

// x16 [B,HW,C] -> y fp32 [B,C,HW]
template <int DT>
__global__ void __launch_bounds__(256) nhwc16_to_nchw_kernel(const uint16_t* __restrict__ x, float* __restrict__ y,
                                                             int C, int HW) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int p = p0 + ty + 8 * k, c = c0 + tx;
    tile[ty + 8 * k][tx] = (p < HW && c < C) ? ld16<DT>(x + ((size_t)b * HW + p) * C + c) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c0 + ty + 8 * k, p = p0 + tx;
    if (c < C && p < HW) y[((size_t)b * C + c) * HW + p] = tile[tx][ty + 8 * k];
  }
}

int launch_nhwc16_to_nchw(const void* x16, float* y, int B, int C, int HW, int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && y, "nhwc16_to_nchw: null pointer");
  dim3 grid(cdiv_i(HW, 32), cdiv_i(C, 32), B);
  if (dtype == HF_BF16)
    nhwc16_to_nchw_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, C, HW);
  else
    nhwc16_to_nchw_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, C, HW);
  HF_LAUNCH_OK("nhwc16_to_nchw");
  count_launch();
  return HF_OK;
}

// Squeeze-excite pooling (SEModule, helpers.py:57-75) in two deterministic stages.
// Stage 1: per-(b, pixel split, 64-channel slab) partial sums of an NHWC 16-bit tensor.  256 threads = 8 lanes of
// 8 channels (16-byte loads) x 32 pixel rows; fixed summation order.  part[(b*S + s)*C + c].
template <int DT>
__global__ void __launch_bounds__(256) channel_sum_partial_kernel(const uint16_t* __restrict__ x,
                                                                  float* __restrict__ part, int HW, int C, int chunk) {
  __shared__ float red[32][65];
  const int b = blockIdx.y, s = blockIdx.z, S = gridDim.z, c0 = blockIdx.x * 64;
  const int lane8 = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int c = c0 + lane8 * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int p0 = s * chunk, p1 = min(HW, p0 + chunk);
  if (c < C) {
    for (int p = p0 + row; p < p1; p += 32) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((size_t)b * HW + p) * C + c));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        acc[2 * k] += Half2T<DT>::to_float((uint16_t)(w[k] & 0xFFFF));
        acc[2 * k + 1] += Half2T<DT>::to_float((uint16_t)(w[k] >> 16));
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[row][lane8 * 8 + k] = acc[k];
  __syncthreads();
  if (threadIdx.x < 64 && c0 + threadIdx.x < C) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += red[r][threadIdx.x];
    part[((size_t)b * S + s) * C + c0 + threadIdx.x] = t;
  }
}

// Stage 2, one CTA per sample: mean[c] = sum_s part / HW; with fc weights, gate = sigmoid(W2 . relu(W1 . mean))
// (fc1 [Cr,C], fc2 [C,Cr], both bias-free 1x1 convs); without, out = mean.
__global__ void __launch_bounds__(256) se_gate_kernel(const float* __restrict__ part, int S, float inv_hw,
                                                      const float* __restrict__ w1, const float* __restrict__ w2,
                                                      float* __restrict__ out, int C, int Cr) {
  extern __shared__ float sm[];
  float* mean = sm;
  float* hid = sm + C;
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int c = tid; c < C; c += 256) {
    float t = 0.f;
    for (int s = 0; s < S; ++s) t += part[((size_t)b * S + s) * C + c];
    mean[c] = t * inv_hw;
    if (!w1) out[(size_t)b * C + c] = mean[c];
  }
  if (!w1) return;
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int j = warp; j < Cr; j += 8) {
    float t = 0.f;
    for (int c = lane; c < C; c += 32) t = fmaf(__ldg(w1 + (size_t)j * C + c), mean[c], t);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xFFFFFFFFu, t, o);
    if (lane == 0) hid[j] = fmaxf(t, 0.f);
  }
  __syncthreads();
  for (int c = tid; c < C; c += 256) {
    float t = 0.f;
    for (int j = 0; j < Cr; ++j) t = fmaf(__ldg(w2 + (size_t)c * Cr + j), hid[j], t);
    out[(size_t)b * C + c] = 1.f / (1.f + __expf(-t));
  }
}

int channel_reduce_splits(int B, int HW, int C) {
  const int64_t ctas = (int64_t)B * cdiv_i(C, 64);
  int s = cdiv_i((int64_t)4 * num_sms(), ctas);
  s = std::min(s, std::max(1, HW / 64));
  return std::max(1, std::min(s, 64));
}

// gate/mean [B,C] <- x16 [B,HW,C]; workspace: B * splits * C floats
int launch_se_gate(const void* x16, const float* fc1, const float* fc2, float* out, float* ws, int B, int HW, int C,
                   int Cr, int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && out && ws, "se_gate: null pointer");
  HF_REQUIRE(C % 8 == 0 && B > 0 && HW > 0, "se_gate: channels must be a multiple of 8");
  HF_REQUIRE((fc1 == nullptr) == (fc2 == nullptr) && (!fc1 || (Cr > 0 && Cr <= 4096)), "se_gate: bad fc weights");
  int S = 1;
  const int rc = launch_channel_partial(x16, ws, B, HW, C, dtype, st, &S);
  if (rc) return rc;
  se_gate_kernel<<<B, 256, (size_t)(C + (fc1 ? Cr : 0)) * sizeof(float), st>>>(ws, S, 1.f / (float)HW, fc1, fc2, out, C,
                                                                                 Cr);
  HF_LAUNCH_OK("se_gate");
  count_launch();
  return HF_OK;
}

// stage 1 alone: ws[(b*S + s)*C + c] = partial channel sums; *splits = S
int launch_channel_partial(const void* x16, float* ws, int B, int HW, int C, int dtype, cudaStream_t st, int* splits) {
  HF_REQUIRE(x16 && ws && C % 8 == 0 && B > 0 && HW > 0, "channel_partial: bad arguments");
  const int S = channel_reduce_splits(B, HW, C), chunk = cdiv_i(HW, S);
  dim3 grid(cdiv_i(C, 64), B, S);
  if (dtype == HF_BF16)
    channel_sum_partial_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, ws, HW, C, chunk);
  else
    channel_sum_partial_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, ws, HW, C, chunk);
  HF_LAUNCH_OK("channel_sum_partial");
  count_launch();
  if (splits) *splits = S;
  return HF_OK;
}

// out = res * se[b,c] + shortcut[b, y*sc_stride, x*sc_stride, c]   (bottleneck_IR_SE.forward, helpers.py:117-120;
// MaxPool2d(1, stride) shortcut = strided subsample).  y16 = out ; y16b = out*s2[c] + b2[c] (next block's BN).
template <int DT>
__global__ void __launch_bounds__(256) scale_add_kernel(const uint16_t* __restrict__ res, const float* __restrict__ se,
                                                        const uint16_t* __restrict__ sc, int sc_stride,
                                                        const float* __restrict__ s2, const float* __restrict__ b2,
                                                        uint16_t* __restrict__ y, uint16_t* __restrict__ yb, int H,
                                                        int W, int C, int64_t total2) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total2; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int64_t e = (int64_t)i * 2;
    const int c = (int)(e % C);
    int64_t t = e / C;
    const int x = (int)(t % W); t /= W;
    const int yy = (int)(t % H);
    const int b = (int)(t / H);
    const uint32_t r2 = *reinterpret_cast<const uint32_t*>(res + e);
    float v0 = Half2T<DT>::to_float((uint16_t)(r2 & 0xFFFF)), v1 = Half2T<DT>::to_float((uint16_t)(r2 >> 16));
    if (se) { v0 *= __ldg(se + (size_t)b * C + c); v1 *= __ldg(se + (size_t)b * C + c + 1); }
    if (sc) {
      const size_t si = (((size_t)b * H * sc_stride + (size_t)yy * sc_stride) * W * sc_stride + (size_t)x * sc_stride) * C + c;
      const uint32_t q2 = *reinterpret_cast<const uint32_t*>(sc + si);
      v0 += Half2T<DT>::to_float((uint16_t)(q2 & 0xFFFF));
      v1 += Half2T<DT>::to_float((uint16_t)(q2 >> 16));
    }
    if (y) *reinterpret_cast<uint32_t*>(y + e) = Half2T<DT>::pack(v0, v1);
    if (yb) {
      const float a0 = s2 ? __ldg(s2 + c) : 1.f, a1 = s2 ? __ldg(s2 + c + 1) : 1.f;
      const float c0 = b2 ? __ldg(b2 + c) : 0.f, c1 = b2 ? __ldg(b2 + c + 1) : 0.f;
      *reinterpret_cast<uint32_t*>(yb + e) = Half2T<DT>::pack(fmaf(v0, a0, c0), fmaf(v1, a1, c1));
    }
  }
}

// same, 8 channels (16 bytes) per thread; C % 8 == 0
template <int DT>
__global__ void __launch_bounds__(256) scale_add_vec8_kernel(const uint16_t* __restrict__ res,
                                                             const float* __restrict__ se,
                                                             const uint16_t* __restrict__ sc, int sc_stride,
                                                             const float* __restrict__ s2, const float* __restrict__ b2,
                                                             uint16_t* __restrict__ y, uint16_t* __restrict__ yb, int H,
                                                             int W, int C8, int64_t total8) {
  const int C = C8 * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total8; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int c = (int)(i % C8) * 8;
    int t = i / C8;
    const int x = (int)(t % W); t /= W;
    const int yy = (int)(t % H);
    const int b = (int)(t / H);
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(res + (size_t)i * 8));
    const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
    float v[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[2 * k] = Half2T<DT>::to_float((uint16_t)(rw[k] & 0xFFFF));
      v[2 * k + 1] = Half2T<DT>::to_float((uint16_t)(rw[k] >> 16));
    }
    if (se) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(se + (size_t)b * C + c));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(se + (size_t)b * C + c + 4));
      v[0] *= g0.x; v[1] *= g0.y; v[2] *= g0.z; v[3] *= g0.w;
      v[4] *= g1.x; v[5] *= g1.y; v[6] *= g1.z; v[7] *= g1.w;
    }
    if (sc) {
      const size_t si = (((size_t)b * H * sc_stride + (size_t)yy * sc_stride) * W * sc_stride + (size_t)x * sc_stride) * C + c;
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(sc + si));
      const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        v[2 * k] += Half2T<DT>::to_float((uint16_t)(qw[k] & 0xFFFF));
        v[2 * k + 1] += Half2T<DT>::to_float((uint16_t)(qw[k] >> 16));
      }
    }
    if (y) {
      uint4 o;
      o.x = Half2T<DT>::pack(v[0], v[1]); o.y = Half2T<DT>::pack(v[2], v[3]);
      o.z = Half2T<DT>::pack(v[4], v[5]); o.w = Half2T<DT>::pack(v[6], v[7]);
      *reinterpret_cast<uint4*>(y + (size_t)i * 8) = o;
    }
    if (yb) {
      float a[8], d[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) { a[k] = s2 ? __ldg(s2 + c + k) : 1.f; d[k] = b2 ? __ldg(b2 + c + k) : 0.f; }
      uint4 o;
      o.x = Half2T<DT>::pack(fmaf(v[0], a[0], d[0]), fmaf(v[1], a[1], d[1]));
      o.y = Half2T<DT>::pack(fmaf(v[2], a[2], d[2]), fmaf(v[3], a[3], d[3]));
      o.z = Half2T<DT>::pack(fmaf(v[4], a[4], d[4]), fmaf(v[5], a[5], d[5]));
      o.w = Half2T<DT>::pack(fmaf(v[6], a[6], d[6]), fmaf(v[7], a[7], d[7]));
      *reinterpret_cast<uint4*>(yb + (size_t)i * 8) = o;
    }
  }
}

int launch_scale_add(const void* res16, const float* se, const void* shortcut16, int sc_stride, const float* s2,
                     const float* b2, void* y16, void* y16b, int B, int H, int W, int C, int dtype, cudaStream_t st) {
  HF_REQUIRE(res16 && (y16 || y16b), "scale_add: null pointer");
  HF_REQUIRE(C % 2 == 0 && (sc_stride == 1 || sc_stride == 2), "scale_add: bad C / stride");
  if (C % 8 == 0) {
    const int64_t total8 = (int64_t)B * H * W * C / 8;
    HF_REQUIRE(total8 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total8);
    const int grid8 = (int)std::min<int64_t>((total8 + 255) / 256, (int64_t)num_sms() * 16);
    if (dtype == HF_BF16)
      scale_add_vec8_kernel<HF_BF16><<<grid8, 256, 0, st>>>((const uint16_t*)res16, se, (const uint16_t*)shortcut16,
                                                            sc_stride, s2, b2, (uint16_t*)y16, (uint16_t*)y16b, H, W,
                                                            C / 8, total8);
    else
      scale_add_vec8_kernel<HF_F16><<<grid8, 256, 0, st>>>((const uint16_t*)res16, se, (const uint16_t*)shortcut16,
                                                           sc_stride, s2, b2, (uint16_t*)y16, (uint16_t*)y16b, H, W,
                                                           C / 8, total8);
    HF_LAUNCH_OK("scale_add");
    count_launch();
    return HF_OK;
  }
  const int64_t total2 = (int64_t)B * H * W * C / 2;
  HF_REQUIRE(total2 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total2);
  const int grid = (int)std::min<int64_t>((total2 + 255) / 256, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    scale_add_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)res16, se, (const uint16_t*)shortcut16, sc_stride,
                                                     s2, b2, (uint16_t*)y16, (uint16_t*)y16b, H, W, C, total2);
  else
    scale_add_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)res16, se, (const uint16_t*)shortcut16, sc_stride,
                                                    s2, b2, (uint16_t*)y16, (uint16_t*)y16b, H, W, C, total2);
  HF_LAUNCH_OK("scale_add");
  count_launch();
  return HF_OK;
}

// out = bilinear_upsample(x, size=(H,W), align_corners=True) + y   (_upsample_add, helpers.py:123-140)
template <int DT>
__global__ void __launch_bounds__(256) upsample_add_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ y,
                                                           uint16_t* __restrict__ out, int h, int w, int H, int W, int C,
                                                           int64_t total2) {
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total2; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int64_t e = (int64_t)i * 2;
    const int c = (int)(e % C);
    int64_t t = e / C;
    const int X = (int)(t % W); t /= W;
    const int Y = (int)(t % H);
    const int b = (int)(t / H);
    const float fy = Y * ry, fx = X * rx;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + 1 < h ? y0 + 1 : y0, x1 = x0 + 1 < w ? x0 + 1 : x0;
    const float ly = fy - y0, lx = fx - x0;
    float v[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t base = (size_t)b * h * w * C + c + u;
      const float a00 = ld16<DT>(x + base + ((size_t)y0 * w + x0) * C), a01 = ld16<DT>(x + base + ((size_t)y0 * w + x1) * C);
      const float a10 = ld16<DT>(x + base + ((size_t)y1 * w + x0) * C), a11 = ld16<DT>(x + base + ((size_t)y1 * w + x1) * C);
      v[u] = (1.f - ly) * ((1.f - lx) * a00 + lx * a01) + ly * ((1.f - lx) * a10 + lx * a11) + ld16<DT>(y + e + u);
    }
    *reinterpret_cast<uint32_t*>(out + e) = Half2T<DT>::pack(v[0], v[1]);
  }
}

template <int DT>
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[2 * k] = Half2T<DT>::to_float((uint16_t)(w[k] & 0xFFFF));
    f[2 * k + 1] = Half2T<DT>::to_float((uint16_t)(w[k] >> 16));
  }
}

// same arithmetic (same operation order per element), 8 channels per thread; C % 8 == 0
template <int DT>
__global__ void __launch_bounds__(256) upsample_add_vec8_kernel(const uint16_t* __restrict__ x,
                                                                const uint16_t* __restrict__ y,
                                                                uint16_t* __restrict__ out, int h, int w, int H, int W,
                                                                int C8, int64_t total8) {
  const int C = C8 * 8;
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total8; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int c = (int)(i % C8) * 8;
    int t = i / C8;
    const int X = (int)(t % W); t /= W;
    const int Y = (int)(t % H);
    const int b = (int)(t / H);
    const float fy = Y * ry, fx = X * rx;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + 1 < h ? y0 + 1 : y0, x1 = x0 + 1 < w ? x0 + 1 : x0;
    const float ly = fy - y0, lx = fx - x0;
    const size_t base = (size_t)b * h * w * C + c;
    float a00[8], a01[8], a10[8], a11[8], yy[8], v[8];
    unpack8<DT>(__ldg(reinterpret_cast<const uint4*>(x + base + ((size_t)y0 * w + x0) * C)), a00);
    unpack8<DT>(__ldg(reinterpret_cast<const uint4*>(x + base + ((size_t)y0 * w + x1) * C)), a01);
    unpack8<DT>(__ldg(reinterpret_cast<const uint4*>(x + base + ((size_t)y1 * w + x0) * C)), a10);
    unpack8<DT>(__ldg(reinterpret_cast<const uint4*>(x + base + ((size_t)y1 * w + x1) * C)), a11);
    unpack8<DT>(__ldg(reinterpret_cast<const uint4*>(y + (size_t)i * 8)), yy);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      v[k] = (1.f - ly) * ((1.f - lx) * a00[k] + lx * a01[k]) + ly * ((1.f - lx) * a10[k] + lx * a11[k]) + yy[k];
    uint4 o;
    o.x = Half2T<DT>::pack(v[0], v[1]); o.y = Half2T<DT>::pack(v[2], v[3]);
    o.z = Half2T<DT>::pack(v[4], v[5]); o.w = Half2T<DT>::pack(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + (size_t)i * 8) = o;
  }
}

int launch_upsample_add(const void* x16, const void* y16, void* out16, int B, int h, int w, int H, int W, int C,
                        int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && y16 && out16 && C % 2 == 0, "upsample_add: bad arguments");
  if (C % 8 == 0) {
    const int64_t total8 = (int64_t)B * H * W * C / 8;
    HF_REQUIRE(total8 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total8);
    const int grid8 = (int)std::min<int64_t>((total8 + 255) / 256, (int64_t)num_sms() * 16);
    if (dtype == HF_BF16)
      upsample_add_vec8_kernel<HF_BF16><<<grid8, 256, 0, st>>>((const uint16_t*)x16, (const uint16_t*)y16,
                                                               (uint16_t*)out16, h, w, H, W, C / 8, total8);
    else
      upsample_add_vec8_kernel<HF_F16><<<grid8, 256, 0, st>>>((const uint16_t*)x16, (const uint16_t*)y16,
                                                              (uint16_t*)out16, h, w, H, W, C / 8, total8);
    HF_LAUNCH_OK("upsample_add");
    count_launch();
    return HF_OK;
  }
  const int64_t total2 = (int64_t)B * H * W * C / 2;
  HF_REQUIRE(total2 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total2);
  const int grid = (int)std::min<int64_t>((total2 + 255) / 256, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    upsample_add_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, (const uint16_t*)y16, (uint16_t*)out16, h,
                                                        w, H, W, C, total2);
  else
    upsample_add_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, (const uint16_t*)y16, (uint16_t*)out16, h, w,
                                                       H, W, C, total2);
  HF_LAUNCH_OK("upsample_add");
  count_launch();
  return HF_OK;
}

// AdaptiveAvgPool2d((oh,ow)) of an NHWC 16-bit tensor -> fp32 NCHW [B,C,oh,ow] (fs_encoder_v2, feature_style_encoder.py)
template <int DT>
__global__ void __launch_bounds__(256) adaptive_avgpool_kernel(const uint16_t* __restrict__ x, float* __restrict__ y,
                                                               int H, int W, int C, int oh, int ow, int64_t total) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int ox = (int)(t % ow); t /= ow;
    const int oy = (int)(t % oh);
    const int b = (int)(t / oh);
    const int ys = (oy * H) / oh, ye = ((oy + 1) * H + oh - 1) / oh;      // PyTorch adaptive pooling windows
    const int xs = (ox * W) / ow, xe = ((ox + 1) * W + ow - 1) / ow;
    float acc = 0.f;
    for (int yy = ys; yy < ye; ++yy)
      for (int xx = xs; xx < xe; ++xx) acc += ld16<DT>(x + (((size_t)b * H + yy) * W + xx) * C + c);
    y[(((size_t)b * C + c) * oh + oy) * ow + ox] = acc / (float)((ye - ys) * (xe - xs));
  }
}

// same, one CTA per (64-channel slab, output bin, sample): 8 lanes of 8 channels (16-byte loads) x 32 window pixels
// in flight, fixed-order shared-memory reduction.  C % 8 == 0.
template <int DT>
__global__ void __launch_bounds__(256) adaptive_avgpool_vec8_kernel(const uint16_t* __restrict__ x,
                                                                    float* __restrict__ y, int H, int W, int C, int oh,
                                                                    int ow) {
  __shared__ float red[32][65];
  const int b = blockIdx.z, oy = blockIdx.y / ow, ox = blockIdx.y % ow, c0 = blockIdx.x * 64;
  const int lane8 = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int c = c0 + lane8 * 8;
  const int ys = (oy * H) / oh, ye = ((oy + 1) * H + oh - 1) / oh;
  const int xs = (ox * W) / ow, xe = ((ox + 1) * W + ow - 1) / ow;
  const int ww = xe - xs, n = (ye - ys) * ww;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    for (int p = row; p < n; p += 32) {
      const int yy = ys + p / ww, xx = xs + p % ww;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((size_t)b * H + yy) * W + xx) * C + c));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        acc[2 * k] += Half2T<DT>::to_float((uint16_t)(w[k] & 0xFFFF));
        acc[2 * k + 1] += Half2T<DT>::to_float((uint16_t)(w[k] >> 16));
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[row][lane8 * 8 + k] = acc[k];
  __syncthreads();
  if (threadIdx.x < 64 && c0 + threadIdx.x < C) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += red[r][threadIdx.x];
    y[(((size_t)b * C + c0 + threadIdx.x) * oh + oy) * ow + ox] = t / (float)n;
  }
}

int launch_adaptive_avgpool(const void* x16, float* y, int B, int H, int W, int C, int oh, int ow, int dtype,
                            cudaStream_t st) {
  HF_REQUIRE(x16 && y && oh > 0 && ow > 0, "adaptive_avgpool: bad arguments");
  if (C % 8 == 0 && (int64_t)oh * ow <= 65535 && B <= 65535) {
    dim3 grid(cdiv_i(C, 64), oh * ow, B);
    if (dtype == HF_BF16)
      adaptive_avgpool_vec8_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, H, W, C, oh, ow);
    else
      adaptive_avgpool_vec8_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, H, W, C, oh, ow);
    HF_LAUNCH_OK("adaptive_avgpool");
    count_launch();
    return HF_OK;
  }
  const int64_t total = (int64_t)B * oh * ow * C;
  HF_REQUIRE(total < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total);
  const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    adaptive_avgpool_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, H, W, C, oh, ow, total);
  else
    adaptive_avgpool_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, y, H, W, C, oh, ow, total);
  HF_LAUNCH_OK("adaptive_avgpool");
  count_launch();
  return HF_OK;
}

}  // namespace hf
