// Kernels around the wgmma convolution for the BiSeNet face-parsing network (SURVEY 8f-3; reference
// models/CtrlHair/external_code/face_parsing/{model,resnet}.py): the 7x7 stride-2 RGB stem, 3x3 stride-2 max pooling,
// pooled 1x1 "attention" convolutions, gated add with nearest 2x upsampling, and the final bilinear logit upsampling.
// All SIMT, fp32 math, deterministic.
#include <algorithm>

#include "hf_kernels.cuh"

namespace hf {

static inline int cdiv_s(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

template <int DT>
__device__ __forceinline__ void unpack8s(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[2 * k] = Half2T<DT>::to_float((uint16_t)(w[k] & 0xFFFF));
    f[2 * k + 1] = Half2T<DT>::to_float((uint16_t)(w[k] >> 16));
  }
}
template <int DT>
__device__ __forceinline__ uint4 pack8s(const float* v) {
  uint4 o;
  o.x = Half2T<DT>::pack(v[0], v[1]); o.y = Half2T<DT>::pack(v[2], v[3]);
  o.z = Half2T<DT>::pack(v[4], v[5]); o.w = Half2T<DT>::pack(v[6], v[7]);
  return o;
}

// ------------------------------------------------------------------------------------------------
// Resnet18.conv1 (resnet.py:60,69): 7x7, stride 2, pad 3 on 3 channels.  K = 147 per output pixel is too thin for an
// implicit-GEMM tap loop (Cin = 3 would be padded to 32 per tap: 11x wasted MMA work) and the first, direct SIMT
// version ran at 30 TFLOP/s fp32 = 26 % of a BiSeNet forward.  So the stem is an explicit im2col into a 16-bit NHWC
// tensor [B,Ho,Wo,160] (channel k = (c*7 + ky)*7 + kx, zero above 147 and outside the image) followed by the
// ordinary 1x1 tensor-core convolution with the folded BatchNorm + ReLU epilogue.  One thread = 8 channels of one pixel.
// ------------------------------------------------------------------------------------------------
constexpr int kStemK = 147, kStemKPad = 160, kI2cTile = 128;

template <int DT>
__global__ void __launch_bounds__(256) im2col7x7s2_kernel(const float* __restrict__ x, uint16_t* __restrict__ y, int H,
                                                          int W, int Ho, int Wo, int64_t total) {
  // one CTA per output row (b, oy) (grid-stride): the only runtime-divisor divisions are per row; inside the row
  // the (ox, 8-channel chunk) split divides by the constant 20
  // The 21 input row segments (3 channels x 7 rows, zero filled outside the image) of a 128-pixel tile are staged in
  // shared memory with coalesced loads; every thread then gathers 8 consecutive k from there.
  __shared__ float sx[21][kI2cTile * 2 + 6];
  const int plane = H * W;
  const int rows = (int)total;                 // = B * Ho
  constexpr int CH = kStemKPad / 8, SW = kI2cTile * 2 + 6;
  const int xtiles = (Wo + kI2cTile - 1) / kI2cTile;
  for (int work = blockIdx.x; work < rows * xtiles; work += gridDim.x) {
    const int row = work / xtiles, ox0 = (work - row * xtiles) * kI2cTile;
    const int b = row / Ho, oy = row - b * Ho;
    const float* xb = x + (size_t)b * 3 * plane;
    const int ybase = 2 * oy - 3, xbase = 2 * ox0 - 3;
    __syncthreads();
    // two unrolled phases: every global load of a thread is in flight before its first shared store
    constexpr int N_STAGE = (21 * SW + 255) / 256;
    float stage[N_STAGE];
#pragma unroll
    for (int it = 0; it < N_STAGE; ++it) {
      const int i = threadIdx.x + it * 256;
      const int rr = i / SW, q = i - rr * SW;
      const int c = rr / 7, yy = ybase + (rr - c * 7), xx = xbase + q;
      stage[it] = (i < 21 * SW && (unsigned)yy < (unsigned)H && (unsigned)xx < (unsigned)W)
                      ? __ldg(xb + c * plane + yy * W + xx) : 0.f;
    }
#pragma unroll
    for (int it = 0; it < N_STAGE; ++it) {
      const int i = threadIdx.x + it * 256;
      if (i < 21 * SW) sx[i / SW][i - (i / SW) * SW] = stage[it];
    }
    __syncthreads();
    const int npix = min(kI2cTile, Wo - ox0);
    uint16_t* ytile = y + ((size_t)row * Wo + ox0) * kStemKPad;
    for (int idx = threadIdx.x; idx < npix * CH; idx += blockDim.x) {
      const int oxl = idx / CH, k0 = (idx - oxl * CH) * 8;
      int rr = k0 / 7, kx = k0 - rr * 7;             // rr = c*7 + ky; walk kx fastest
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[j] = rr < 21 ? sx[rr][2 * oxl + kx] : 0.f;
        if (++kx == 7) { kx = 0; ++rr; }
      }
      *reinterpret_cast<uint4*>(ytile + (size_t)idx * 8) = pack8s<DT>(v);
    }
  }
}

int launch_im2col7x7s2(const float* x, void* y16, int B, int H, int W, int dtype, cudaStream_t st) {
  HF_REQUIRE(x && y16, "im2col7x7s2: null pointer");
  HF_REQUIRE(B > 0 && H > 0 && W > 0, "im2col7x7s2: bad shape");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t total = (int64_t)B * Ho;         // output rows
  HF_REQUIRE(total < (int64_t)2000000000, "tensor too large for one launch (%lld rows): split the batch", (long long)total);
  const int64_t work = total * ((Wo + kI2cTile - 1) / kI2cTile);
  HF_REQUIRE(work < (int64_t)2000000000, "im2col7x7s2: too many tiles (%lld): split the batch", (long long)work);
  const int grid = (int)std::min<int64_t>(work, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    im2col7x7s2_kernel<HF_BF16><<<grid, 256, 0, st>>>(x, (uint16_t*)y16, H, W, Ho, Wo, total);
  else
    im2col7x7s2_kernel<HF_F16><<<grid, 256, 0, st>>>(x, (uint16_t*)y16, H, W, Ho, Wo, total);
  HF_LAUNCH_OK("im2col7x7s2");
  count_launch();
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.MaxPool2d(kernel_size=3, stride=2, padding=1) (resnet.py:62,71) on NHWC 16-bit; padding never wins the max.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) maxpool3x3s2_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y,
                                                           int H, int W, int Ho, int Wo, int C8, int64_t total8) {
  const int C = C8 * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total8; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int c = (int)(i % C8) * 8;
    int t = i / C8;
    const int ox = (int)(t % Wo); t /= Wo;
    const int oy = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float m[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) m[k] = -3.0e38f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const int yy = 2 * oy + dy;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int xx = 2 * ox + dx;
        if (xx < 0 || xx >= W) continue;
        float v[8];
        unpack8s<DT>(__ldg(reinterpret_cast<const uint4*>(x + (((size_t)b * H + yy) * W + xx) * C + c)), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) m[k] = fmaxf(m[k], v[k]);
      }
    }
    *reinterpret_cast<uint4*>(y + (size_t)i * 8) = pack8s<DT>(m);
  }
}

int launch_maxpool3x3s2(const void* x16, void* y16, int B, int H, int W, int C, int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && y16 && C % 8 == 0 && B > 0 && H > 0 && W > 0, "maxpool: bad arguments");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total8 = (int64_t)B * Ho * Wo * C / 8;
  HF_REQUIRE(total8 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total8);
  const int grid = (int)std::min<int64_t>((total8 + 255) / 256, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    maxpool3x3s2_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, (uint16_t*)y16, H, W, Ho, Wo, C / 8, total8);
  else
    maxpool3x3s2_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, (uint16_t*)y16, H, W, Ho, Wo, C / 8, total8);
  HF_LAUNCH_OK("maxpool3x3s2");
  count_launch();
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// 1x1 convolution of the globally pooled feature (+ folded BatchNorm + activation):
//   out[b,o] = act((sum_c w[o,c] * mean_hw(x)[b,c]) * scale[o] + shift[o])
// AttentionRefinementModule attention (model.py:82-86: sigmoid) and ContextPath.conv_avg (model.py:114-115: ReLU).
// Stage 1 is the shared deterministic pooling (channel_sum_partial_kernel); this is stage 2, one CTA per sample.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pooled_fc_kernel(const float* __restrict__ part, int S, float inv_hw,
                                                        const float* __restrict__ w, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, int act,
                                                        float* __restrict__ out, int C, int Cout) {
  extern __shared__ float mean[];
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int c = tid; c < C; c += 256) {
    float t = 0.f;
    for (int s = 0; s < S; ++s) t += part[((size_t)b * S + s) * C + c];
    mean[c] = t * inv_hw;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int o = warp; o < Cout; o += 8) {
    float t = 0.f;
    for (int c = lane; c < C; c += 32) t = fmaf(__ldg(w + (size_t)o * C + c), mean[c], t);
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) t += __shfl_xor_sync(0xFFFFFFFFu, t, k);
    if (lane == 0) {
      float v = fmaf(t, scale ? __ldg(scale + o) : 1.f, shift ? __ldg(shift + o) : 0.f);
      if (act == 2) v = 1.f / (1.f + __expf(-v));
      else if (act == 1) v = fmaxf(v, 0.f);
      out[(size_t)b * Cout + o] = v;
    }
  }
}

int launch_pooled_fc(const void* x16, const float* w, const float* scale, const float* shift, int act, float* out,
                     float* ws, int B, int HW, int C, int Cout, int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && w && out && ws, "pooled_fc: null pointer");
  HF_REQUIRE(C % 8 == 0 && C <= 8192 && Cout > 0 && act >= 0 && act <= 2, "pooled_fc: bad arguments");
  int S = 1;
  int rc = launch_channel_partial(x16, ws, B, HW, C, dtype, st, &S);
  if (rc) return rc;
  pooled_fc_kernel<<<B, 256, (size_t)C * sizeof(float), st>>>(ws, S, 1.f / (float)HW, w, scale, shift, act, out, C, Cout);
  HF_LAUNCH_OK("pooled_fc");
  count_launch();
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// y[b,Y,X,c] = x[b,Y/up,X/up,c] * gate[b,c] + addvec[b,c] + addt[b,Y/up,X/up,c]      (up = 1 or 2, nearest)
// ContextPath (model.py:116-128): feat*atten (+ the pooled branch | + the upsampled coarser branch), then
// F.interpolate(mode='nearest') to the next finer level.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) gate_add_up_kernel(const uint16_t* __restrict__ x, const float* __restrict__ gate,
                                                          const float* __restrict__ addvec,
                                                          const uint16_t* __restrict__ addt, uint16_t* __restrict__ y,
                                                          int h, int w, int up, int C8, int64_t total8) {
  const int C = C8 * 8, H = h * up, W = w * up;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total8; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int c = (int)(i % C8) * 8;
    int t = i / C8;
    const int X = (int)(t % W); t /= W;
    const int Y = (int)(t % H);
    const int b = (int)(t / H);
    const size_t src = (((size_t)b * h + Y / up) * w + X / up) * C + c;
    float v[8];
    unpack8s<DT>(__ldg(reinterpret_cast<const uint4*>(x + src)), v);
    if (gate) {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] *= __ldg(gate + (size_t)b * C + c + k);
    }
    if (addvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] += __ldg(addvec + (size_t)b * C + c + k);
    }
    if (addt) {
      float a[8];
      unpack8s<DT>(__ldg(reinterpret_cast<const uint4*>(addt + src)), a);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] += a[k];
    }
    *reinterpret_cast<uint4*>(y + (size_t)i * 8) = pack8s<DT>(v);
  }
}

int launch_gate_add_up(const void* x16, const float* gate, const float* addvec, const void* addt16, void* y16, int B,
                       int h, int w, int C, int up, int dtype, cudaStream_t st) {
  HF_REQUIRE(x16 && y16 && C % 8 == 0 && (up == 1 || up == 2) && B > 0 && h > 0 && w > 0, "gate_add_up: bad arguments");
  const int64_t total8 = (int64_t)B * h * up * w * up * C / 8;
  HF_REQUIRE(total8 < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total8);
  const int grid = (int)std::min<int64_t>((total8 + 255) / 256, (int64_t)num_sms() * 16);
  if (dtype == HF_BF16)
    gate_add_up_kernel<HF_BF16><<<grid, 256, 0, st>>>((const uint16_t*)x16, gate, addvec, (const uint16_t*)addt16,
                                                      (uint16_t*)y16, h, w, up, C / 8, total8);
  else
    gate_add_up_kernel<HF_F16><<<grid, 256, 0, st>>>((const uint16_t*)x16, gate, addvec, (const uint16_t*)addt16,
                                                     (uint16_t*)y16, h, w, up, C / 8, total8);
  HF_LAUNCH_OK("gate_add_up");
  count_launch();
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// Fused stem (round 2): Resnet18.conv1 7x7/s2/p3 + bn1 + ReLU (resnet.py:60-61,69-70) in ONE kernel, fp32 NCHW image in,
// 16-bit NHWC [B,Ho,Wo,64] out -- the [B,Ho,Wo,160] im2col tensor (21 MB per 512^2 image, written by one kernel and
// read back by the next: 0.84 ms of a B=48 call) no longer exists.
// Roofline: 1.23 GFLOP against 3 MB in + 8.4 MB out per 512^2 image = 108 FLOP/B, far left of the ridge (~260): the
// kernel is HBM-bound, so the contraction runs on warp-level mma.sync.m16n8k16 fragments built straight from a
// shared-memory copy of the input window (K = 7 rows x 24 [= 7 taps x 3 channels + 3 zero-weight pads] = 168 -> 176);
// a tensor-core tile would need the same im2col rows materialised in the swizzled operand layout first.
// CTA = 8 x 32 output pixels x 64 channels, 8 warps (one output row each: 2 m16 tiles x 8 n8 tiles x 11 k16 steps).
// ------------------------------------------------------------------------------------------------
constexpr int kSfRows = 8, kSfCols = 32;                 // output tile
constexpr int kSfInRows = 2 * kSfRows + 6;               // 22 (one spare row for the zero-weight K padding)
constexpr int kSfInPitch = 216;                          // (2*32 + 8) * 3 interleaved [x][c] 16-bit elements
constexpr int kSfK = 176, kSfWPitch = 184;               // packed weight row: [n][k], k = ky*24 + kx*3 + c

template <int DT>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  if (DT == HF_BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int DT>
__global__ void __launch_bounds__(256, 2) stem7x7s2_fused_kernel(const float* __restrict__ x,
                                                                 const uint16_t* __restrict__ wp,
                                                                 const float* __restrict__ shift,
                                                                 uint16_t* __restrict__ y, int H, int W, int Ho, int Wo,
                                                                 int tiles_x, int tiles_y, int total_tiles) {
  // persistent CTA: the 23 KB of packed weights are loaded ONCE and stay in shared memory while the CTA walks over its
  // tiles (first version: one tile per CTA re-read them 12 k times per launch and ran at 82 TFLOP/s)
  extern __shared__ __align__(16) uint8_t stem_smem[];
  uint16_t* w_s = reinterpret_cast<uint16_t*>(stem_smem);                       // [64][184]
  uint16_t* in_s = w_s + 64 * kSfWPitch;                                          // [22][216]
  uint16_t* out_s = in_s + kSfInRows * kSfInPitch;                                // [256][64], chunk ^ (pixel & 7)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 64 * kSfWPitch / 8; i += 256)
    reinterpret_cast<uint4*>(w_s)[i] = __ldg(reinterpret_cast<const uint4*>(wp) + i);
  const int g4 = lane >> 2, q2 = (lane & 3) * 2;
  float sh[8][2];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sh[j][0] = __ldg(shift + j * 8 + q2); sh[j][1] = __ldg(shift + j * 8 + q2 + 1); }
  const int fr = threadIdx.x >> 6, fc = threadIdx.x & 63;                        // fill: 4 rows x 64 columns per pass

  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int tx = tile % tiles_x, t2 = tile / tiles_x, ty = t2 % tiles_y, b = t2 / tiles_y;
    const int oy0 = ty * kSfRows, ox0 = tx * kSfCols;
    const float* xb = x + (size_t)b * 3 * H * W;
    // ---- stage the 22 x 72 x 3 input window (zero outside the image = the conv padding), interleaved [row][x*3 + c]
    const int gy0 = 2 * oy0 - 3, gx0 = 2 * ox0 - 3;
    {
      // columns fc (0..63) of rows fr, fr+4, ..., fr+20: six loads per channel in flight before the first store;
      // then the 8 tail columns 64..71 (threads with fc < 8)
      const int gxa = gx0 + fc, gxb = gx0 + 64 + fc;
      const bool cola = gxa >= 0 && gxa < W, colb = fc < 8 && gxb >= 0 && gxb < W;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* xc = xb + (size_t)c * H * W;
        float va[6], vb[6];
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
          const int r = fr + 4 * kk, gy = gy0 + r;
          const bool row_ok = r < kSfInRows && gy >= 0 && gy < H;
          const float* xr = xc + (size_t)(row_ok ? gy : 0) * W;
          va[kk] = (row_ok && cola) ? __ldg(xr + gxa) : 0.f;
          vb[kk] = (row_ok && colb) ? __ldg(xr + gxb) : 0.f;
        }
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) {
          const int r = fr + 4 * kk;
          if (r < kSfInRows) {
            in_s[r * kSfInPitch + fc * 3 + c] = Half2T<DT>::one(va[kk]);
            if (fc < 8) in_s[r * kSfInPitch + (64 + fc) * 3 + c] = Half2T<DT>::one(vb[kk]);
          }
        }
      }
    }
    __syncthreads();

    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
    // A[pixel (warp, ox)][k = ky*24 + t] = in_s[2*warp + ky][6*ox + t]
    const uint16_t* a_row = in_s + (2 * warp) * kSfInPitch;
#pragma unroll
    for (int ks = 0; ks < kSfK / 16; ++ks) {
      int off[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int kk = ks * 16 + 8 * j + q2;
        off[j] = (kk / 24) * kSfInPitch + (kk % 24);
      }
      uint32_t a[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int oxa = i * 16 + g4;
        a[i][0] = *reinterpret_cast<const uint32_t*>(a_row + 6 * oxa + off[0]);
        a[i][1] = *reinterpret_cast<const uint32_t*>(a_row + 6 * (oxa + 8) + off[0]);
        a[i][2] = *reinterpret_cast<const uint32_t*>(a_row + 6 * oxa + off[1]);
        a[i][3] = *reinterpret_cast<const uint32_t*>(a_row + 6 * (oxa + 8) + off[1]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bf[2];
        const uint16_t* wrow = w_s + (j * 8 + g4) * kSfWPitch + ks * 16 + q2;
        bf[0] = *reinterpret_cast<const uint32_t*>(wrow);
        bf[1] = *reinterpret_cast<const uint32_t*>(wrow + 8);
        mma16816<DT>(acc[0][j], a[0], bf);
        mma16816<DT>(acc[1][j], a[1], bf);
      }
    }
    // ---- epilogue: + shift (BatchNorm folded: scale lives in the weights), ReLU, 16-bit, swizzled staging (its own
    // buffer: the previous tile's copy-out finished before this tile's fill barrier)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pix = warp * 32 + i * 16 + g4 + 8 * h;
          const float v0 = fmaxf(acc[i][j][2 * h] + sh[j][0], 0.f), v1 = fmaxf(acc[i][j][2 * h + 1] + sh[j][1], 0.f);
          *reinterpret_cast<uint32_t*>(out_s + pix * 64 + ((j ^ (pix & 7)) * 8) + q2) = Half2T<DT>::pack(v0, v1);
        }
      }
    __syncthreads();                                     // staging complete; also: everyone is done reading in_s
    for (int i = threadIdx.x; i < 256 * 8; i += 256) {
      const int pix = i >> 3, ch = i & 7;
      const int oy = oy0 + (pix >> 5), ox = ox0 + (pix & 31);
      if (oy < Ho && ox < Wo) {
        const uint4 v = *reinterpret_cast<const uint4*>(out_s + pix * 64 + ((ch ^ (pix & 7)) * 8));
        *reinterpret_cast<uint4*>(y + (((size_t)b * Ho + oy) * Wo + ox) * 64 + ch * 8) = v;
      }
    }
    // the next iteration's fill writes in_s (free since the barrier above) and its first barrier orders the out_s
    // reads above against the next epilogue's writes
  }
}

// ------------------------------------------------------------------------------------------------
// Fused 3x3 RGB stem of the IR-SE / iresnet encoders (round 2): Conv2d(3, 64, 3, 1, 1) + BatchNorm + PReLU
// (encoder4editing/models/encoders/psp_encoders.py:176-178 `input_layer`; FeatureStyleEncoder/arcface/iresnet.py:92-95
// conv1/bn1/prelu as taken by nets/feature_style_encoder.py:27; models/Net.py:347) in ONE kernel: fp32 NCHW image in,
// the raw 16-bit NHWC [B,H,W,64] activation AND its BatchNorm-affined copy for the first block out.  It replaces an
// NCHW->NHWC(32) layout pass plus an implicit-GEMM convolution whose K = 9 x 32 was 90 % zero padding (Cin 3 -> 32).  Same
// scheme as the 7x7 stem above (HBM-bound: 0.8 MB in, 16.8 MB out per 256^2 image): window gathered in shared memory
// interleaved [row][x*4 + c] (c = 3 is a zero lane so that every k pair is one aligned 32-bit word), k = ky*16 + kx*4 + c
// (K = 48), mma.sync fragments, persistent CTAs with the 7 KB of packed weights resident.
// ------------------------------------------------------------------------------------------------
constexpr int kS3InRows = kSfRows + 2, kS3InPitch = (kSfCols + 2) * 4;       // 10 rows x 136 elements
constexpr int kS3K = 48, kS3WPitch = 56;

template <int DT>
__global__ void __launch_bounds__(256, 2) stem3x3_fused_kernel(const float* __restrict__ x,
                                                               const uint16_t* __restrict__ wp,
                                                               const float* __restrict__ shift,
                                                               const float* __restrict__ slope,
                                                               const float* __restrict__ s2,
                                                               const float* __restrict__ b2,
                                                               uint16_t* __restrict__ y, uint16_t* __restrict__ yb,
                                                               int H, int W, int tiles_x, int tiles_y, int total_tiles) {
  __shared__ __align__(16) uint16_t w_s[64 * kS3WPitch];
  __shared__ __align__(16) uint16_t in_s[kS3InRows * kS3InPitch + 16];
  __shared__ __align__(16) uint16_t out_s[256 * 64];
  __shared__ float ep_s[4][64];                          // shift, slope, s2, b2
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 64 * kS3WPitch / 8; i += 256)
    reinterpret_cast<uint4*>(w_s)[i] = __ldg(reinterpret_cast<const uint4*>(wp) + i);
  for (int i = threadIdx.x; i < kS3InRows * kS3InPitch + 16; i += 256) in_s[i] = 0;      // the c = 3 lanes stay zero
  if (threadIdx.x < 64) {
    ep_s[0][threadIdx.x] = __ldg(shift + threadIdx.x);
    ep_s[1][threadIdx.x] = __ldg(slope + threadIdx.x);
    ep_s[2][threadIdx.x] = s2 ? __ldg(s2 + threadIdx.x) : 1.f;
    ep_s[3][threadIdx.x] = b2 ? __ldg(b2 + threadIdx.x) : 0.f;
  }
  const int g4 = lane >> 2, q2 = (lane & 3) * 2;
  const int fcx = threadIdx.x % (kSfCols + 2), fr0 = threadIdx.x / (kSfCols + 2);         // fill: 7 rows x 34 columns per pass
  __syncthreads();

  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int tx = tile % tiles_x, t2 = tile / tiles_x, ty = t2 % tiles_y, b = t2 / tiles_y;
    const int oy0 = ty * kSfRows, ox0 = tx * kSfCols;
    const float* xb = x + (size_t)b * 3 * H * W;
    // ---- stage the 10 x 34 x 3 window (zero outside the image = the conv padding)
    if (fr0 < 7) {
      const int gx = ox0 - 1 + fcx;
      const bool col_ok = gx >= 0 && gx < W;
      float v[3][2];
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 2; ++k) {                    // rows fr0 and fr0 + 7: all six loads in flight together
          const int r = fr0 + 7 * k, gy = oy0 - 1 + r;
          v[c][k] = (r < kS3InRows && col_ok && gy >= 0 && gy < H) ? __ldg(xb + ((size_t)c * H + gy) * W + gx) : 0.f;
        }
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int r = fr0 + 7 * k;
          if (r < kS3InRows) in_s[r * kS3InPitch + fcx * 4 + c] = Half2T<DT>::one(v[c][k]);
        }
    }
    __syncthreads();
    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < kS3K / 16; ++ks) {            // ks = kernel row ky
      const uint16_t* a_row = in_s + (warp + ks) * kS3InPitch;
      uint32_t a[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int oxa = i * 16 + g4;
        a[i][0] = *reinterpret_cast<const uint32_t*>(a_row + 4 * oxa + q2);
        a[i][1] = *reinterpret_cast<const uint32_t*>(a_row + 4 * (oxa + 8) + q2);
        a[i][2] = *reinterpret_cast<const uint32_t*>(a_row + 4 * oxa + q2 + 8);
        a[i][3] = *reinterpret_cast<const uint32_t*>(a_row + 4 * (oxa + 8) + q2 + 8);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bf[2];
        const uint16_t* wrow = w_s + (j * 8 + g4) * kS3WPitch + ks * 16 + q2;
        bf[0] = *reinterpret_cast<const uint32_t*>(wrow);
        bf[1] = *reinterpret_cast<const uint32_t*>(wrow + 8);
        mma16816<DT>(acc[0][j], a[0], bf);
        mma16816<DT>(acc[1][j], a[1], bf);
      }
    }
    // ---- epilogue: v = prelu(acc + shift); pass 0 stores v, pass 1 stores v * s2 + b2 (the first block's BatchNorm)
    for (int pass = 0; pass < (yb ? 2 : 1); ++pass) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int n0 = j * 8 + q2;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int pix = warp * 32 + i * 16 + g4 + 8 * h;
            float v[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              float t = acc[i][j][2 * h + u] + ep_s[0][n0 + u];
              t = t > 0.f ? t : t * ep_s[1][n0 + u];
              if (pass) t = fmaf(t, ep_s[2][n0 + u], ep_s[3][n0 + u]);
              v[u] = t;
            }
            *reinterpret_cast<uint32_t*>(out_s + pix * 64 + ((j ^ (pix & 7)) * 8) + q2) = Half2T<DT>::pack(v[0], v[1]);
          }
        }
      __syncthreads();
      uint16_t* dst = pass ? yb : y;
      for (int i = threadIdx.x; i < 256 * 8; i += 256) {
        const int pix = i >> 3, ch = i & 7;
        const int oy = oy0 + (pix >> 5), ox = ox0 + (pix & 31);
        if (oy < H && ox < W) {
          const uint4 v = *reinterpret_cast<const uint4*>(out_s + pix * 64 + ((ch ^ (pix & 7)) * 8));
          *reinterpret_cast<uint4*>(dst + (((size_t)b * H + oy) * W + ox) * 64 + ch * 8) = v;
        }
      }
      __syncthreads();                                   // out_s (and, after the last pass, in_s) may be rewritten
    }
  }
}

int launch_stem3x3_fused(const float* x, const void* wpacked, const float* shift, const float* slope, const float* s2,
                         const float* b2, void* y16, void* y16b, int B, int H, int W, int dtype, cudaStream_t st) {
  HF_REQUIRE(x && wpacked && shift && slope && y16, "stem3x3: null pointer");
  HF_REQUIRE((y16b == nullptr) == (s2 == nullptr) && (s2 == nullptr) == (b2 == nullptr),
             "stem3x3: y16b, s2 and b2 come together");
  HF_REQUIRE(B > 0 && H > 0 && W > 0, "stem3x3: bad shape");
  HF_REQUIRE((((uintptr_t)wpacked | (uintptr_t)y16 | (uintptr_t)y16b) & 15) == 0, "stem3x3: buffers must be 16-byte aligned");
  const int tiles_x = cdiv_s(W, kSfCols), tiles_y = cdiv_s(H, kSfRows);
  const int64_t total = (int64_t)tiles_x * tiles_y * B;
  HF_REQUIRE(total < (int64_t)2000000000, "stem3x3: too many tiles");
  const int grid = (int)std::min<int64_t>(total, (int64_t)num_sms() * 2);
  if (dtype == HF_BF16)
    stem3x3_fused_kernel<HF_BF16><<<grid, 256, 0, st>>>(x, (const uint16_t*)wpacked, shift, slope, s2, b2, (uint16_t*)y16,
                                                        (uint16_t*)y16b, H, W, tiles_x, tiles_y, (int)total);
  else
    stem3x3_fused_kernel<HF_F16><<<grid, 256, 0, st>>>(x, (const uint16_t*)wpacked, shift, slope, s2, b2, (uint16_t*)y16,
                                                       (uint16_t*)y16b, H, W, tiles_x, tiles_y, (int)total);
  HF_LAUNCH_OK("stem3x3_fused");
  count_launch();
  return HF_OK;
}

int launch_stem7x7s2_fused(const float* x, const void* wpacked, const float* shift, void* y16, int B, int H, int W,
                           int dtype, cudaStream_t st) {
  HF_REQUIRE(x && wpacked && shift && y16, "stem7x7s2: null pointer");
  HF_REQUIRE(B > 0 && H > 0 && W > 0 && B <= 65535, "stem7x7s2: bad shape");
  HF_REQUIRE((((uintptr_t)wpacked | (uintptr_t)y16) & 15) == 0, "stem7x7s2: packed weights / output must be 16-byte aligned");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int tiles_x = cdiv_s(Wo, kSfCols), tiles_y = cdiv_s(Ho, kSfRows);
  const int64_t total = (int64_t)tiles_x * tiles_y * B;
  HF_REQUIRE(total < (int64_t)2000000000, "stem7x7s2: too many tiles");
  const size_t smem = (size_t)(64 * kSfWPitch + kSfInRows * kSfInPitch + 256 * 64) * sizeof(uint16_t);   // 65.8 KB
  const int grid = (int)std::min<int64_t>(total, (int64_t)num_sms() * 2);
  if (dtype == HF_BF16) {
    HF_CUDA_OK(cudaFuncSetAttribute(stem7x7s2_fused_kernel<HF_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stem7x7s2_fused_kernel<HF_BF16><<<grid, 256, smem, st>>>(x, (const uint16_t*)wpacked, shift, (uint16_t*)y16, H, W, Ho,
                                                             Wo, tiles_x, tiles_y, (int)total);
  } else {
    HF_CUDA_OK(cudaFuncSetAttribute(stem7x7s2_fused_kernel<HF_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stem7x7s2_fused_kernel<HF_F16><<<grid, 256, smem, st>>>(x, (const uint16_t*)wpacked, shift, (uint16_t*)y16, H, W, Ho,
                                                            Wo, tiles_x, tiles_y, (int)total);
  }
  HF_LAUNCH_OK("stem7x7s2_fused");
  count_launch();
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// F.interpolate(x, (H, W), mode='bilinear', align_corners=True) on fp32 NCHW (model.py:239-241): the first C of
// Cin channel planes of x (the logit convolution pads its 19 classes to 32 output channels).
// ------------------------------------------------------------------------------------------------
// the one interpolation expression of all three kernels below (explicit roundings: the fused arg-max kernel must
// reproduce the logits of the plain upsampling kernel bit for bit)
__device__ __forceinline__ float lerp_rn(float t, float a, float b) {
  return __fmaf_rn(t, b, __fmul_rn(__fsub_rn(1.f, t), a));
}

__global__ void __launch_bounds__(256) bilinear_up_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int C,
                                                               int Cin, int h, int w, int H, int W4, int64_t rows) {
  // One CTA per output row (b, c, Y), grid-stride.  The two source rows are blended once into shared memory
  // (w values), then every thread produces 4 consecutive output columns (float4 store) from it.  Same weights as
  // F.interpolate(align_corners=True); the association of the fp32 products differs by ~1 ulp.
  extern __shared__ float srow[];
  const int W = W4 * 4;
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int row = blockIdx.x; row < (int)rows; row += gridDim.x) {
    const int bc = row / H, Y = row - bc * H;
    const int b = bc / C, c = bc - b * C;
    const float fy = Y * ry;
    const int y0 = (int)fy;
    const int y1 = y0 + 1 < h ? y0 + 1 : y0;
    const float ly = fy - y0;
    const float* p0 = x + (((size_t)b * Cin + c) * h + y0) * w;
    const float* p1 = x + (((size_t)b * Cin + c) * h + y1) * w;
    __syncthreads();
    for (int xs = threadIdx.x; xs < w; xs += blockDim.x) srow[xs] = lerp_rn(ly, __ldg(p0 + xs), __ldg(p1 + xs));
    __syncthreads();
    float* yrow = y + (size_t)row * W;
    for (int X4 = threadIdx.x; X4 < W4; X4 += blockDim.x) {
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float fx = (X4 * 4 + j) * rx;
        const int x0 = (int)fx;
        const int x1 = x0 + 1 < w ? x0 + 1 : x0;
        const float lx = fx - x0;
        o[j] = lerp_rn(lx, srow[x0], srow[x1]);
      }
      *reinterpret_cast<float4*>(yrow + X4 * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

__global__ void __launch_bounds__(256) bilinear_up_nchw_scalar_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                      int C, int Cin, int h, int w, int H, int W,
                                                                      int64_t total) {
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (int)total; i += gridDim.x * blockDim.x) {   // 32-bit index math: 64-bit div/mod costs ~100 instructions
    const int X = (int)(i % W);
    int t = i / W;
    const int Y = (int)(t % H); t /= H;
    const int c = (int)(t % C);
    const int b = (int)(t / C);
    const float fy = Y * ry, fx = X * rx;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + 1 < h ? y0 + 1 : y0, x1 = x0 + 1 < w ? x0 + 1 : x0;
    const float ly = fy - y0, lx = fx - x0;
    const float* p = x + ((size_t)b * Cin + c) * h * w;
    const float a00 = __ldg(p + (size_t)y0 * w + x0), a01 = __ldg(p + (size_t)y0 * w + x1);
    const float a10 = __ldg(p + (size_t)y1 * w + x0), a11 = __ldg(p + (size_t)y1 * w + x1);
    y[i] = lerp_rn(lx, lerp_rn(ly, a00, a10), lerp_rn(ly, a01, a11));       // rows first, like the row kernel
  }
}

// Fused `F.interpolate(logits, (H, W), 'bilinear', align_corners=True)` + `argmax(dim=1)` (BiSeNet.forward
// model.py:239 followed by FaceParsing_tensor.parsing_img, my_parsing_util.py:87-88): the [B,C,H,W] fp32 logits
// (76 B per pixel for 19 classes) never exist; 8 B of label per pixel are written.  One CTA per output row (b, Y): the
// C vertically blended source rows go to shared memory, then every thread scans the C classes of its pixels with the
// same arithmetic as bilinear_up_nchw_kernel, keeping the FIRST maximum (torch.argmax's tie rule).
__global__ void __launch_bounds__(256) bilinear_argmax_kernel(const float* __restrict__ x, long long* __restrict__ labels,
                                                              int C, int Cin, int h, int w, int H, int W, int rows) {
  extern __shared__ float srow[];                       // [C][w]
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int b = row / H, Y = row - b * H;
    const float fy = Y * ry;
    const int y0 = (int)fy;
    const int y1 = y0 + 1 < h ? y0 + 1 : y0;
    const float ly = fy - y0;
    __syncthreads();
    for (int i = threadIdx.x; i < C * w; i += blockDim.x) {
      const int c = i / w, xs = i - c * w;
      const float* p = x + ((size_t)b * Cin + c) * h * w;
      srow[i] = lerp_rn(ly, __ldg(p + (size_t)y0 * w + xs), __ldg(p + (size_t)y1 * w + xs));
    }
    __syncthreads();
    long long* out = labels + (size_t)row * W;
    for (int X = threadIdx.x; X < W; X += blockDim.x) {
      const float fx = X * rx;
      const int x0 = (int)fx;
      const int x1 = x0 + 1 < w ? x0 + 1 : x0;
      const float lx = fx - x0;
      float best = lerp_rn(lx, srow[x0], srow[x1]);
      int arg = 0;
      for (int c = 1; c < C; ++c) {
        const float v = lerp_rn(lx, srow[c * w + x0], srow[c * w + x1]);
        if (v > best) { best = v; arg = c; }
      }
      out[X] = arg;
    }
  }
}

int launch_bilinear_argmax(const float* x, long long* labels, int B, int C, int Cin, int h, int w, int H, int W,
                           cudaStream_t st) {
  HF_REQUIRE(x && labels && B > 0 && C > 0 && Cin >= C && h > 0 && w > 0 && H > 0 && W > 0,
             "bilinear_argmax: bad arguments");
  const size_t smem = (size_t)C * w * sizeof(float);
  HF_REQUIRE(smem <= 200 * 1024, "bilinear_argmax: %d classes x %d source columns do not fit in shared memory", C, w);
  const int64_t rows = (int64_t)B * H;
  HF_REQUIRE(rows < (int64_t)2000000000, "bilinear_argmax: too many rows");
  if (smem > 48 * 1024)
    HF_CUDA_OK(cudaFuncSetAttribute(bilinear_argmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::min<int64_t>(rows, (int64_t)num_sms() * 8);
  bilinear_argmax_kernel<<<grid, 256, smem, st>>>(x, labels, C, Cin, h, w, H, W, (int)rows);
  HF_LAUNCH_OK("bilinear_argmax");
  count_launch();
  return HF_OK;
}

int launch_bilinear_up_nchw(const float* x, float* y, int B, int C, int Cin, int h, int w, int H, int W,
                            cudaStream_t st) {
  HF_REQUIRE(x && y && B > 0 && C > 0 && Cin >= C && h > 0 && w > 0 && H > 0 && W > 0, "bilinear_up: bad arguments");
  const int64_t total = (int64_t)B * C * H * W;
  HF_REQUIRE(total < (int64_t)2000000000, "tensor too large for one launch (%lld work items): split the batch", (long long)total);
  if (W % 4 == 0 && (((uintptr_t)y) & 15) == 0 && w <= 8192) {
    const int64_t rows = (int64_t)B * C * H;
    const int grid = (int)std::min<int64_t>(rows, (int64_t)num_sms() * 16);
    bilinear_up_nchw_kernel<<<grid, 256, (size_t)w * sizeof(float), st>>>(x, y, C, Cin, h, w, H, W / 4, rows);
  } else {
    const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 32);
    bilinear_up_nchw_scalar_kernel<<<grid, 256, 0, st>>>(x, y, C, Cin, h, w, H, W, total);
  }
  HF_LAUNCH_OK("bilinear_up_nchw");
  count_launch();
  return HF_OK;
}

}  // namespace hf
