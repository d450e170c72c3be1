// Stage glue around the networks (SURVEY 8f-4): BicubicDownSample (utils/bicubic.py:6-78), the separable
// 4*factor-tap bicubic decimation HairFast applies to every 1024^2 image (Embedding.py:66-67, Blending.py:64).
// HBM-bound SIMT, fp32, deterministic.
#include "hf_kernels.cuh"

namespace hf {

constexpr int kBicTileH = 8, kBicTileW = 64, kBicMaxFactor = 8;

__device__ __forceinline__ int reflect_index(int i, int n) {      // F.pad(mode='reflect'): edge not repeated
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// y[p, oy, ox] = sum_j k[j] * V[oy][ox*f + j - pl],  V[oy][c] = sum_i k[i] * x[p, refl(oy*f + i - pt), refl(c)]
// (reference order: reflect-pad H, 1-D conv over H with stride f, [clip/round], reflect-pad W, 1-D conv over W).
// One CTA = 8 x 64 outputs of one plane: the vertical pass of the (64 f + 3 f) needed columns goes to shared memory,
// the horizontal pass reads it back.
__global__ void __launch_bounds__(256) bicubic_down_kernel(const float* __restrict__ x, const float* __restrict__ k,
                                                           float* __restrict__ y, int H, int W, int Ho, int Wo, int f,
                                                           int clip_round) {
  extern __shared__ float sm[];
  const int taps = 4 * f;
  const int pad = taps - f, p0 = pad / 2;                 // pad_top = pad_left = (4f - f) // 2
  const int cols = kBicTileW * f + pad;                  // input columns one output row segment needs
  float* kf = sm;                                        // [taps]
  float* v = sm + 4 * kBicMaxFactor;                     // [kBicTileH][cols]
  const int plane = blockIdx.z, oy0 = blockIdx.y * kBicTileH, ox0 = blockIdx.x * kBicTileW;
  const float* xp = x + (size_t)plane * H * W;
  if (threadIdx.x < taps) kf[threadIdx.x] = __ldg(k + threadIdx.x);
  __syncthreads();
  const int ix0 = ox0 * f - p0;
  for (int i = threadIdx.x; i < kBicTileH * cols; i += blockDim.x) {
    const int r = i / cols, c = i - r * cols;
    const int oy = oy0 + r;
    float acc = 0.f;
    if (oy < Ho) {
      // columns right of the last valid output of a partial tile are never read back: clamp them into the plane
      // (a single reflection of ix0 + c >= 2W - 1 would land before the row start)
      const int xc = min(max(reflect_index(ix0 + c, W), 0), W - 1);
      const int iy0 = oy * f - p0;
      for (int t = 0; t < taps; ++t) acc = fmaf(kf[t], __ldg(xp + (size_t)reflect_index(iy0 + t, H) * W + xc), acc);
      if (clip_round) acc = fminf(fmaxf(rintf(acc), 0.f), 255.f);
    }
    v[i] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kBicTileH * kBicTileW; i += blockDim.x) {
    const int r = i / kBicTileW, c = i - r * kBicTileW;
    const int oy = oy0 + r, ox = ox0 + c;
    if (oy >= Ho || ox >= Wo) continue;
    const float* row = v + r * cols + c * f;
    float acc = 0.f;
    for (int t = 0; t < taps; ++t) acc = fmaf(kf[t], row[t], acc);
    if (clip_round) acc = fminf(fmaxf(rintf(acc), 0.f), 255.f);
    y[((size_t)plane * Ho + oy) * Wo + ox] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// DilateErosion.mask (utils/image_utils.py:42-55): `iterations` rounds of a 3x3 cross "convolution" with zero padding
// followed by a threshold -- dilation keeps sum > 0, erosion keeps sum == 5.  One launch per round, both masks at
// once, ping-pong between two caller-provided planes; the arithmetic is on exact small integers in fp32.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dilate_erode_step_kernel(const float* __restrict__ din,
                                                                const float* __restrict__ ein,
                                                                float* __restrict__ dout, float* __restrict__ eout,
                                                                int H, int W, int total) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int x = i % W, t = i / W, y = t % H;
    const float* dp = din + i;
    const float* ep = ein + i;
    float sd = __ldg(dp), se = __ldg(ep);                          // centre, up, down, left, right
    if (y > 0) { sd += __ldg(dp - W); se += __ldg(ep - W); }
    if (y + 1 < H) { sd += __ldg(dp + W); se += __ldg(ep + W); }
    if (x > 0) { sd += __ldg(dp - 1); se += __ldg(ep - 1); }
    if (x + 1 < W) { sd += __ldg(dp + 1); se += __ldg(ep + 1); }
    dout[i] = sd > 0.f ? 1.f : 0.f;
    eout[i] = se == 5.f ? 1.f : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// F-space alignment (models/Alignment.py:139-159; the same blend with one stage is the Embedding mixing,
// models/Embedding.py:86-92).
//   masks  = [1 - (1 - HM1)(1 - HMX),  HMX,  HM2 * HMX]                                     (:139-143)  hf_align_masks_f32
//   w_s    = scale_a + scale_b * bicubic_down(free_mask_s, 256^2 -> 32^2)                    (:153-154)
//   F      = src_s + w_s * (F - src_s),  s = 0 .. n_stage-1,  F starting from `first`         (:157-159)  hf_fspace_blend_f32
// `F.interpolate(mode='bicubic')` = PyTorch's upsample_bicubic2d, align_corners=False, A = -0.75: source coordinate
// (i + 0.5) * in / out - 0.5, four taps around its floor with clamped indices.  One launch: every CTA first evaluates
// the n_stage interpolated weights of its 256 pixels (shared memory), then streams its channel slice with 16-byte
// accesses (4-byte ones when P % 4 != 0, past the last full quad, or when a tensor is not 16-byte aligned).  fp32
// throughout; the only difference from the torch expression is fma contraction (<= 1e-6).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) align_masks_kernel(const float* __restrict__ hm1, const float* __restrict__ hm2,
                                                          const float* __restrict__ hmx, float* __restrict__ out,
                                                          int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float a = __ldg(hm1 + i), b = __ldg(hm2 + i), x = __ldg(hmx + i);
    out[i] = 1.f - (1.f - a) * (1.f - x);
    out[n + i] = x;
    out[2 * n + i] = b * x;
  }
}

__device__ __forceinline__ void cubic_coeffs(float t, float* w) {
  const float A = -0.75f;                         // ATen UpSample.h: cubic_convolution1 / cubic_convolution2
  const float x0 = t + 1.f, x1 = t, x2 = 1.f - t, x3 = 2.f - t;
  w[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
  w[1] = ((A + 2.f) * x1 - (A + 3.f)) * x1 * x1 + 1.f;
  w[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  w[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}

constexpr int kBlendMaxStage = 4;
struct BlendArgs {
  const float* first;                  // [C, P]
  const float* src[kBlendMaxStage];    // [C, P] each
  const float* mask[kBlendMaxStage];   // [Hm, Wm] each
  float scale_a[kBlendMaxStage], scale_b[kBlendMaxStage];
  float* out;                          // [C, P]
  int n_stage, C, Ho, Wo, Hm, Wm, ch_per_block;
  int aligned;                         // first, every src[s] and out 16-byte aligned: the float4 path may run
};

__global__ void __launch_bounds__(256) fspace_blend_kernel(const BlendArgs a) {
  __shared__ float w_sm[kBlendMaxStage][256];
  const int P = a.Ho * a.Wo;
  const int p0 = blockIdx.x * 256;
  const int p = p0 + threadIdx.x;
  if (p < P) {
    const int oy = p / a.Wo, ox = p - oy * a.Wo;
    const float sy = (oy + 0.5f) * ((float)a.Hm / (float)a.Ho) - 0.5f;
    const float sx = (ox + 0.5f) * ((float)a.Wm / (float)a.Wo) - 0.5f;
    const float fy = floorf(sy), fx = floorf(sx);
    float wy[4], wx[4];
    cubic_coeffs(sy - fy, wy);
    cubic_coeffs(sx - fx, wx);
    const int iy = (int)fy, ix = (int)fx;
    for (int s = 0; s < a.n_stage; ++s) {
      float acc = 0.f;
      for (int j = 0; j < 4; ++j) {
        const int yy = min(max(iy - 1 + j, 0), a.Hm - 1);
        float row = 0.f;
        for (int i = 0; i < 4; ++i) {
          const int xx = min(max(ix - 1 + i, 0), a.Wm - 1);
          row += __ldg(a.mask[s] + (size_t)yy * a.Wm + xx) * wx[i];
        }
        acc += row * wy[j];
      }
      w_sm[s][threadIdx.x] = a.scale_a[s] + a.scale_b[s] * acc;
    }
  }
  __syncthreads();
  const int c0 = blockIdx.y * a.ch_per_block, c1 = min(c0 + a.ch_per_block, a.C);
  // 64 threads x float4 cover the 256 pixels of this CTA; 4 channel rows in flight per pass
  const int lane4 = (threadIdx.x & 63) * 4, crow = threadIdx.x >> 6;
  const bool vec = a.aligned && (P % 4 == 0) && (p0 + lane4 + 3 < P);
  for (int c = c0 + crow; c < c1; c += 4) {
    const size_t off = (size_t)c * P + p0 + lane4;
    if (vec) {
      float4 f = __ldg(reinterpret_cast<const float4*>(a.first + off));
      for (int s = 0; s < a.n_stage; ++s) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(a.src[s] + off));
        const float* w = &w_sm[s][lane4];
        f.x = b.x + w[0] * (f.x - b.x); f.y = b.y + w[1] * (f.y - b.y);
        f.z = b.z + w[2] * (f.z - b.z); f.w = b.w + w[3] * (f.w - b.w);
      }
      *reinterpret_cast<float4*>(a.out + off) = f;
    } else {
      for (int e = 0; e < 4; ++e) {
        if (p0 + lane4 + e >= P) break;
        float f = __ldg(a.first + off + e);
        for (int s = 0; s < a.n_stage; ++s) {
          const float b = __ldg(a.src[s] + off + e);
          f = b + w_sm[s][lane4 + e] * (f - b);
        }
        a.out[off + e] = f;
      }
    }
  }
}

}  // namespace hf

using namespace hf;

extern "C" {

int hf_bicubic_downsample_f32(const float* x, const float* k, float* y, int planes, int H, int W, int factor,
                              int clip_round, void* stream) {
  HF_REQUIRE(x && k && y, "bicubic_down: null pointer");
  HF_REQUIRE(factor >= 1 && factor <= kBicMaxFactor, "bicubic_down: factor %d unsupported (1..%d)", factor, kBicMaxFactor);
  HF_REQUIRE(planes > 0 && planes <= 65535 && H > 0 && W > 0, "bicubic_down: bad shape");
  const int taps = 4 * factor, pad = taps - factor;
  HF_REQUIRE(pad / 2 < H && pad - pad / 2 < H && pad / 2 < W && pad - pad / 2 < W, "bicubic_down: image smaller than the reflect padding");
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int Ho = (H + pad - taps) / factor + 1, Wo = (W + pad - taps) / factor + 1;
  const size_t smem = (size_t)(4 * kBicMaxFactor + kBicTileH * (kBicTileW * factor + pad)) * sizeof(float);
  dim3 grid((Wo + kBicTileW - 1) / kBicTileW, (Ho + kBicTileH - 1) / kBicTileH, planes);
  bicubic_down_kernel<<<grid, 256, smem, st>>>(x, k, y, H, W, Ho, Wo, factor, clip_round);
  HF_LAUNCH_OK("bicubic_down");
  count_launch();
  return HF_OK;
}

int hf_dilate_erode_f32(const float* mask, float* dilate, float* erode, void* workspace, int planes, int H, int W,
                        int iterations, void* stream) {
  float* ws = (float*)workspace;
  HF_REQUIRE(mask && dilate && erode, "dilate_erode: null pointer");
  HF_REQUIRE(planes > 0 && H > 0 && W > 0 && iterations >= 0, "dilate_erode: bad arguments");
  const int64_t total = (int64_t)planes * H * W;
  HF_REQUIRE(total < (int64_t)2000000000, "dilate_erode: tensor too large for one launch");
  HF_REQUIRE(iterations <= 1 || ws, "dilate_erode: workspace (2 planes sets) needed for more than one iteration");
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = (size_t)total * sizeof(float);
  if (iterations == 0) {
    HF_CUDA_OK(cudaMemcpyAsync(dilate, mask, bytes, cudaMemcpyDeviceToDevice, st));
    HF_CUDA_OK(cudaMemcpyAsync(erode, mask, bytes, cudaMemcpyDeviceToDevice, st));
    return HF_OK;
  }
  const int grid = grid_for(total);
  // buffers: round r reads (d_in, e_in) and writes (d_out, e_out); the last round writes the outputs
  const float *d_in = mask, *e_in = mask;
  float* tmp_d[2] = {ws, ws ? ws + 2 * total : nullptr};
  float* tmp_e[2] = {ws ? ws + total : nullptr, ws ? ws + 3 * total : nullptr};
  for (int r = 0; r < iterations; ++r) {
    const bool last = r == iterations - 1;
    float* d_out = last ? dilate : tmp_d[r & 1];
    float* e_out = last ? erode : tmp_e[r & 1];
    dilate_erode_step_kernel<<<grid, 256, 0, st>>>(d_in, e_in, d_out, e_out, H, W, (int)total);
    HF_LAUNCH_OK("dilate_erode_step");
    count_launch();
    d_in = d_out; e_in = e_out;
  }
  return HF_OK;
}

int hf_align_masks_f32(const float* hm1, const float* hm2, const float* hmx, float* out, int n, void* stream) {
  HF_REQUIRE(hm1 && hm2 && hmx && out && n > 0, "align_masks: bad arguments");
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  align_masks_kernel<<<(n + 255) / 256, 256, 0, st>>>(hm1, hm2, hmx, out, n);
  HF_LAUNCH_OK("align_masks");
  count_launch();
  return HF_OK;
}

int hf_fspace_blend_f32(const float* first, const float* const* src, const float* const* mask, const float* scale_a,
                        const float* scale_b, float* out, int n_stage, int C, int Ho, int Wo, int Hm, int Wm,
                        void* stream) {
  HF_REQUIRE(first && src && mask && scale_a && scale_b && out, "fspace_blend: null pointer");
  HF_REQUIRE(n_stage >= 1 && n_stage <= kBlendMaxStage, "fspace_blend: 1..%d stages", kBlendMaxStage);
  HF_REQUIRE(C > 0 && Ho > 0 && Wo > 0 && Hm > 0 && Wm > 0, "fspace_blend: bad shape");
  BlendArgs a;
  a.first = first; a.out = out; a.n_stage = n_stage; a.C = C; a.Ho = Ho; a.Wo = Wo; a.Hm = Hm; a.Wm = Wm;
  uintptr_t bits = (uintptr_t)first | (uintptr_t)out;
  for (int s = 0; s < n_stage; ++s) {
    HF_REQUIRE(src[s] && mask[s], "fspace_blend: null stage pointer");
    a.src[s] = src[s]; a.mask[s] = mask[s]; a.scale_a[s] = scale_a[s]; a.scale_b[s] = scale_b[s];
    bits |= (uintptr_t)src[s];
  }
  // contiguous views may start at any 4-byte offset (fspace.py only calls .contiguous()): scalar path then
  a.aligned = (bits & 15) == 0;
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int P = Ho * Wo;
  a.ch_per_block = 16;
  dim3 grid((P + 255) / 256, (C + a.ch_per_block - 1) / a.ch_per_block);
  fspace_blend_kernel<<<grid, 256, 0, st>>>(a);
  HF_LAUNCH_OK("fspace_blend");
  count_launch();
  return HF_OK;
}

}  // extern "C"
