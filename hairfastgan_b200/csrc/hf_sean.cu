// SEAN's SPADE decoder (decode_sean, models/sean_codes/models/pix2pix_model.py:309-325) around the wgmma convolution:
// label maps, the one-hot convolutions as table lookups, the per-call ACE style tables, the ACE normalisation and the
// final RGB convolution.  HBM- / L2-bound SIMT, fp32 arithmetic, fixed summation orders (deterministic).
#include <string.h>

#include "hf_kernels.cuh"

namespace hf {
namespace {

constexpr int kClasses = 19;      // label_nc (SEAN_OPT)
constexpr int kStyle = 512;       // ACE.style_length (normalization.py:79)

// ------------------------------------------------------------------------------------------------
// Label maps.  F.interpolate(one_hot, size=(R, R), mode='nearest') of the size^2 map picks source pixel
// floor(i * size / R) (generator.py:75, normalization.py:115); R runs over size/32 .. size (six levels for 256).
// Labels outside 0..18 are counted in *bad (the reference's scatter_ would index out of range instead).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sean_labels_kernel(const long long* __restrict__ lab, int8_t* __restrict__ maps,
                                                          int* __restrict__ bad, int size, int levels) {
  const int n = size * size;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long v = lab[i];
    const bool ok = v >= 0 && v < kClasses;
    if (!ok) atomicAdd(bad, 1);
    const int y = i / size, x = i % size;
    int8_t* out = maps;
    for (int l = 0; l < levels; ++l) {
      const int R = size >> (levels - 1 - l), f = size / R;
      if (y % f == 0 && x % f == 0) out[(y / f) * R + x / f] = ok ? (int8_t)v : (int8_t)0;
      out += R * R;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 3x3 zero-padded convolution of a one-hot map as a lookup:  y[p, c] = act(bias[c] + sum_{tap, p+tap inside}
// table[tap][L(p+tap)][c]).  One thread = 8 channels of one pixel; table [9][19][C] fp32 stays in L2.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) sean_onehot_kernel(const int8_t* __restrict__ L, const float* __restrict__ table,
                                                          const float* __restrict__ bias, int act,
                                                          uint16_t* __restrict__ y, int R, int C8) {
  const int C = C8 * 8;
  const int total = R * R * C8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = (i % C8) * 8, p = i / C8, py = p / R, px = p % R;
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = bias ? __ldg(bias + c + k) : 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = py + tap / 3 - 1, xx = px + tap % 3 - 1;
      if (yy < 0 || yy >= R || xx < 0 || xx >= R) continue;
      const float* t = table + ((size_t)tap * kClasses + L[yy * R + xx]) * C + c;
      const float4 a = __ldg(reinterpret_cast<const float4*>(t)), b = __ldg(reinterpret_cast<const float4*>(t + 4));
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    if (act == 3) {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
    }
    st8<DT>(y + (size_t)p * C + c, v);
  }
}

// ------------------------------------------------------------------------------------------------
// ACE style tables, step 1: mu[a][j] = relu(fc_w[a][j] . code_j + fc_b[a][j])      (normalization.py:133-135)
// code_j = image_code[j] unless that row is all zero, then mean_code[j]         (pix2pix_model.py:312-315)
// One warp per output element row; grid (kStyle / 8, 19, n_ace).
// ------------------------------------------------------------------------------------------------
struct SeanAceJob {
  const float* fc_w;    // [19][512][512]
  const float* fc_b;    // [19][512]
  const float* tw;      // [9 * n2][512]: row tap * n2 + n of [a_g W_gamma; a_b W_beta][:, :, tap]
  float* table;         // [19][9][n2]
  int n2;
  int block_begin;      // first CTA of this ACE in the table launch
};
constexpr int kMaxAce = 16;
struct SeanAceJobs {
  SeanAceJob job[kMaxAce];
};

__global__ void __launch_bounds__(256) sean_fc_mu_kernel(const float* __restrict__ image_code,
                                                         const float* __restrict__ mean_code, const SeanAceJobs jobs,
                                                         float* __restrict__ mu) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.y, a = blockIdx.z;
  const int row = blockIdx.x * 8 + warp;
  const float* ic = image_code + (size_t)j * kStyle;
  bool nz = false;
  for (int k = lane; k < kStyle; k += 32) nz |= (ic[k] != 0.f);
  nz = __any_sync(0xffffffffu, nz);
  const float* code = nz ? ic : mean_code + (size_t)j * kStyle;
  const SeanAceJob& jb = jobs.job[a];
  const float* w = jb.fc_w + ((size_t)j * kStyle + row) * kStyle;
  float s = 0.f;
  for (int k = lane * 4; k < kStyle; k += 128) {
    const float4 wv = __ldg(reinterpret_cast<const float4*>(w + k));
    const float4 cv = __ldg(reinterpret_cast<const float4*>(code + k));
    s += wv.x * cv.x + wv.y * cv.y + wv.z * cv.z + wv.w * cv.w;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) mu[((size_t)a * kClasses + j) * kStyle + row] = fmaxf(s + __ldg(jb.fc_b + j * kStyle + row), 0.f);
}

// ------------------------------------------------------------------------------------------------
// ACE style tables, step 2: T[a][j][tap][n] = sum_k tw[a][tap * n2 + n][k] * mu[a][j][k].  The 3x3 convolution of the
// piecewise-constant middle_avg (normalization.py:172-173) is then a 9-tap gather of T (ace_apply below).  One warp
// per weight row: the row is read once from HBM and dotted with all 19 class vectors (held in shared memory).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sean_table_kernel(const SeanAceJobs jobs, int n_ace, const float* __restrict__ mu) {
  __shared__ float4 smu[kClasses * kStyle / 4];
  int a = 0;
  while (a + 1 < n_ace && (int)blockIdx.x >= jobs.job[a + 1].block_begin) ++a;
  const SeanAceJob& jb = jobs.job[a];
  const float4* src = reinterpret_cast<const float4*>(mu + (size_t)a * kClasses * kStyle);
  for (int i = threadIdx.x; i < kClasses * kStyle / 4; i += blockDim.x) smu[i] = src[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rows = 9 * jb.n2;
  const int row = ((int)blockIdx.x - jb.block_begin) * 8 + warp;
  if (row >= rows) return;
  const float* w = jb.tw + (size_t)row * kStyle;
  float4 wr[kStyle / 128];
#pragma unroll
  for (int q = 0; q < kStyle / 128; ++q) wr[q] = __ldg(reinterpret_cast<const float4*>(w + q * 128 + lane * 4));
  const int tap = row / jb.n2, n = row % jb.n2;
  for (int j = 0; j < kClasses; ++j) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < kStyle / 128; ++q) {
      const float4 m = smu[j * (kStyle / 4) + q * 32 + lane];
      s += wr[q].x * m.x + wr[q].y * m.y + wr[q].z * m.z + wr[q].w * m.w;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) jb.table[((size_t)j * 9 + tap) * jb.n2 + n] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// ACE.forward (normalization.py:108-189) for batch 1, plus the leaky_relu(0.2) of SPADEResnetBlock.actvn
// (architecture.py:95-96) when lrelu != 0:
//   v   = (x[p,c] + r[w*R + h] * noise_var[c]) * bn_scale[c] + bn_shift[c]     eval BatchNorm, affine=False
//   g   = gb[c][p]     + sum_{tap, p+tap inside} T[L(p+tap)][tap][c]           (blend weights folded into gb / T)
//   b   = gb[C + c][p] + sum_{tap, p+tap inside} T[L(p+tap)][tap][C + c]
//   out = v * (1 + g) + b
// gb = the SPADE gamma || beta convolution (fp32 NCHW [2C][R*R]).  CTA = 32 pixels x 64 channels: gb goes through
// shared memory from its NCHW rows to the NHWC order of x and out.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) sean_ace_kernel(const uint16_t* __restrict__ x, const float* __restrict__ rnd,
                                                       const float* __restrict__ noise_var,
                                                       const float* __restrict__ bn_scale,
                                                       const float* __restrict__ bn_shift, const float* __restrict__ gb,
                                                       const float* __restrict__ T, const int8_t* __restrict__ L,
                                                       int lrelu, uint16_t* __restrict__ y, int R, int C) {
  __shared__ float sgb[2][64][33];
  const int HW = R * R;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < 2 * 64 * 32; i += blockDim.x) {
    const int col = i & 31, row = i >> 5, half = row >> 6, cc = row & 63;
    sgb[half][cc][col] = __ldg(gb + (size_t)(half * C + c0 + cc) * HW + p0 + col);
  }
  __syncthreads();
  const int pl = threadIdx.x >> 3, cl = (threadIdx.x & 7) * 8;
  const int p = p0 + pl, c = c0 + cl, py = p / R, px = p % R;
  float g[8], b[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { g[k] = sgb[0][cl + k][pl]; b[k] = sgb[1][cl + k][pl]; }
  if (T) {
    const int n2 = 2 * C;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = py + tap / 3 - 1, xx = px + tap % 3 - 1;
      if (yy < 0 || yy >= R || xx < 0 || xx >= R) continue;
      const float* t = T + ((size_t)L[yy * R + xx] * 9 + tap) * n2 + c;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(t)), g1 = __ldg(reinterpret_cast<const float4*>(t + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(t + C)),
                   b1 = __ldg(reinterpret_cast<const float4*>(t + C + 4));
      g[0] += g0.x; g[1] += g0.y; g[2] += g0.z; g[3] += g0.w; g[4] += g1.x; g[5] += g1.y; g[6] += g1.z; g[7] += g1.w;
      b[0] += b0.x; b[1] += b0.y; b[2] += b0.z; b[3] += b0.w; b[4] += b1.x; b[5] += b1.y; b[6] += b1.z; b[7] += b1.w;
    }
  }
  float v[8];
  ld8<DT>(x + (size_t)p * C + c, v);
  const float r = __ldg(rnd + px * R + py);          // randn(1, W, H, 1) ... .transpose(1, 3): n[c, h, w] = r[w, h]
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    float t = (v[k] + r * __ldg(noise_var + c + k)) * __ldg(bn_scale + c + k) + __ldg(bn_shift + c + k);
    t = t * (1.f + g[k]) + b[k];
    v[k] = (lrelu && t < 0.f) ? 0.2f * t : t;
  }
  st8<DT>(y + (size_t)p * C + c, v);
}

// ------------------------------------------------------------------------------------------------
// conv_img(leaky_relu(x, 0.2)) + tanh (generator.py:107-108): Cout = 3, so one thread per output pixel with the
// weights in shared memory ([tap][c][3]); fp32 NCHW out.
// ------------------------------------------------------------------------------------------------
constexpr int kImgMaxC = 256;
template <int DT>
__global__ void __launch_bounds__(256) sean_conv_img_kernel(const uint16_t* __restrict__ x, const float* __restrict__ w,
                                                            const float* __restrict__ bias, float* __restrict__ y, int R,
                                                            int C) {
  __shared__ float sw[9 * kImgMaxC * 3];
  for (int i = threadIdx.x; i < 9 * C * 3; i += blockDim.x) {
    const int o = i % 3, c = (i / 3) % C, tap = i / (3 * C);
    sw[i] = w[((size_t)o * C + c) * 9 + tap];
  }
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R * R) return;
  const int py = p / R, px = p % R;
  float acc[3] = {__ldg(bias), __ldg(bias + 1), __ldg(bias + 2)};
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = py + tap / 3 - 1, xx = px + tap % 3 - 1;
    if (yy < 0 || yy >= R || xx < 0 || xx >= R) continue;
    const uint16_t* src = x + (size_t)(yy * R + xx) * C;
    const float* wt = sw + tap * C * 3;
    for (int c = 0; c < C; c += 8) {
      float v[8];
      ld8<DT>(src + c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float a = v[k] < 0.f ? 0.2f * v[k] : v[k];
        acc[0] += a * wt[(c + k) * 3];
        acc[1] += a * wt[(c + k) * 3 + 1];
        acc[2] += a * wt[(c + k) * 3 + 2];
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 3; ++o) y[(size_t)o * R * R + p] = tanhf(acc[o]);
}

// ------------------------------------------------------------------------------------------------
// Zencoder.forward's tail (architecture.py:177-207): codes[b][j][c] = mean over the class-j pixels of tanh(y[b][c]),
// 0 where class j has no pixel.  One CTA per (c, b) plane: thread t accumulates pixels t, t + 256, ... into its own
// column of per-class sums and counts in shared memory, then warp w reduces classes w, w + 8, w + 16 over the 256
// columns in a fixed order (no atomics: the result does not depend on scheduling).
// ------------------------------------------------------------------------------------------------
constexpr int kMeanThreads = 256;
__global__ void __launch_bounds__(kMeanThreads) sean_class_means_kernel(const float* __restrict__ y,
                                                                        const int8_t* __restrict__ labels,
                                                                        long long label_stride,
                                                                        float* __restrict__ codes, int C, int HW) {
  __shared__ float ssum[kClasses][kMeanThreads];
  __shared__ int scnt[kClasses][kMeanThreads];
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  for (int j = 0; j < kClasses; ++j) { ssum[j][tid] = 0.f; scnt[j][tid] = 0; }
  const float* plane = y + ((size_t)b * C + c) * HW;
  const int8_t* L = labels + (size_t)b * label_stride;
  for (int p = tid; p < HW; p += kMeanThreads) {
    const int j = L[p];
    if ((unsigned)j < (unsigned)kClasses) {
      ssum[j][tid] += tanhf(__ldg(plane + p));
      scnt[j][tid] += 1;
    }
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  for (int j = warp; j < kClasses; j += kMeanThreads / 32) {
    float s = 0.f;
    int n = 0;
#pragma unroll
    for (int k = 0; k < kMeanThreads / 32; ++k) { s += ssum[j][lane + 32 * k]; n += scnt[j][lane + 32 * k]; }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      n += __shfl_xor_sync(0xffffffffu, n, o);
    }
    if (lane == 0) codes[((size_t)b * kClasses + j) * C + c] = n > 0 ? s / (float)n : 0.f;
  }
}

}  // namespace
}  // namespace hf

using namespace hf;

extern "C" {

int hf_sean_labels(const long long* labels, int8_t* maps, int* bad, int size, void* stream) {
  HF_REQUIRE(labels && maps && bad, "hf_sean_labels: null pointer");
  HF_REQUIRE(size >= 32 && size % 32 == 0 && size <= 4096, "hf_sean_labels: size %d must be a multiple of 32", size);
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  HF_CUDA_OK(cudaMemsetAsync(bad, 0, sizeof(int), st));
  sean_labels_kernel<<<grid_for((int64_t)size * size), 256, 0, st>>>(labels, maps, bad, size, 6);
  HF_LAUNCH_OK("sean_labels");
  count_launch();
  return HF_OK;
}

int hf_sean_onehot_conv(const int8_t* labels, const float* table, const float* bias, int act, void* y16, int res,
                        int channels, int dtype, void* stream) {
  return with_dtype(dtype, "hf_sean_onehot_conv", [&](auto dt) -> int {
    HF_REQUIRE(labels && table && y16, "hf_sean_onehot_conv: null pointer");
    HF_REQUIRE(res > 0 && channels > 0 && channels % 8 == 0, "hf_sean_onehot_conv: bad shape %d^2 x %d", res, channels);
    HF_REQUIRE(act == 0 || act == 3, "hf_sean_onehot_conv: act %d (0 none, 3 ReLU)", act);
    HF_REQUIRE(((uintptr_t)table & 15) == 0 && ((uintptr_t)y16 & 15) == 0, "hf_sean_onehot_conv: unaligned pointer");
    int rc = ensure_device_current();
    if (rc) return rc;
    const int64_t total = (int64_t)res * res * (channels / 8);
    sean_onehot_kernel<dt><<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(labels, table, bias, act, (uint16_t*)y16,
                                                                              res, channels / 8);
    HF_LAUNCH_OK("sean_onehot");
    count_launch();
    return HF_OK;
  });
}

int hf_sean_style_tables(const float* image_code, const float* mean_code, const hf_sean_ace_tables* aces, int n_ace,
                         float* mu_workspace, void* stream) {
  HF_REQUIRE(image_code && mean_code && aces && mu_workspace, "hf_sean_style_tables: null pointer");
  HF_REQUIRE(n_ace >= 1 && n_ace <= kMaxAce, "hf_sean_style_tables: %d ACE layers (1..%d)", n_ace, kMaxAce);
  HF_REQUIRE(aligned16(image_code, mean_code, mu_workspace),
             "hf_sean_style_tables: image_code, mean_code and mu_workspace must be 16-byte aligned");
  SeanAceJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  int blocks = 0;
  for (int a = 0; a < n_ace; ++a) {
    const hf_sean_ace_tables& s = aces[a];
    HF_REQUIRE(s.fc_w && s.fc_b && s.tw && s.table, "hf_sean_style_tables: null pointer in ACE %d", a);
    HF_REQUIRE(s.n2 > 0 && s.n2 % 8 == 0, "hf_sean_style_tables: ACE %d width %d", a, s.n2);
    HF_REQUIRE(aligned16(s.fc_w, s.tw), "hf_sean_style_tables: fc_w and tw of ACE %d must be 16-byte aligned", a);
    jobs.job[a] = SeanAceJob{s.fc_w, s.fc_b, s.tw, s.table, s.n2, blocks};
    blocks += (9 * s.n2 + 7) / 8;
  }
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  sean_fc_mu_kernel<<<dim3(kStyle / 8, kClasses, n_ace), 256, 0, st>>>(image_code, mean_code, jobs, mu_workspace);
  HF_LAUNCH_OK("sean_fc_mu");
  sean_table_kernel<<<blocks, 256, 0, st>>>(jobs, n_ace, mu_workspace);
  HF_LAUNCH_OK("sean_table");
  count_launch(2);
  return HF_OK;
}

int hf_sean_ace_apply(const void* x16, const float* noise, const float* noise_var, const float* bn_scale,
                      const float* bn_shift, const float* gamma_beta, const float* table, const int8_t* labels,
                      int lrelu, void* y16, int res, int channels, int dtype, void* stream) {
  return with_dtype(dtype, "hf_sean_ace_apply", [&](auto dt) -> int {
    HF_REQUIRE(x16 && noise && noise_var && bn_scale && bn_shift && gamma_beta && y16 && (!table || labels),
               "hf_sean_ace_apply: null pointer");
    HF_REQUIRE(res > 0 && res * res % 32 == 0 && channels % 64 == 0 && channels > 0,
               "hf_sean_ace_apply: bad shape %d^2 x %d (pixels %% 32, channels %% 64)", res, channels);
    HF_REQUIRE(((uintptr_t)x16 & 15) == 0 && ((uintptr_t)y16 & 15) == 0 && ((uintptr_t)table & 15) == 0,
               "hf_sean_ace_apply: unaligned pointer");
    int rc = ensure_device_current();
    if (rc) return rc;
    const dim3 grid(res * res / 32, channels / 64);
    sean_ace_kernel<dt><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x16, noise, noise_var, bn_scale,
                                                                bn_shift, gamma_beta, table, labels, lrelu,
                                                                (uint16_t*)y16, res, channels);
    HF_LAUNCH_OK("sean_ace");
    count_launch();
    return HF_OK;
  });
}

int hf_sean_class_means(const float* y, const int8_t* labels, long long label_stride, float* codes, int batch,
                        int channels, int hw, void* stream) {
  HF_REQUIRE(y && labels && codes, "hf_sean_class_means: null pointer");
  HF_REQUIRE(batch > 0 && batch <= 65535 && channels > 0 && hw > 0 && label_stride >= hw,
             "hf_sean_class_means: bad shape B=%d C=%d HW=%d label stride %lld", batch, channels, hw, label_stride);
  int rc = ensure_device_current();
  if (rc) return rc;
  sean_class_means_kernel<<<dim3(channels, batch), kMeanThreads, 0, (cudaStream_t)stream>>>(y, labels, label_stride,
                                                                                           codes, channels, hw);
  HF_LAUNCH_OK("sean_class_means");
  count_launch();
  return HF_OK;
}

int hf_sean_conv_img(const void* x16, const float* weight, const float* bias, float* y, int res, int channels,
                     int dtype, void* stream) {
  return with_dtype(dtype, "hf_sean_conv_img", [&](auto dt) -> int {
    HF_REQUIRE(x16 && weight && bias && y, "hf_sean_conv_img: null pointer");
    HF_REQUIRE(res > 0 && channels > 0 && channels % 8 == 0 && channels <= kImgMaxC,
               "hf_sean_conv_img: bad shape %d^2 x %d (channels %% 8, <= %d)", res, channels, kImgMaxC);
    HF_REQUIRE(aligned16(x16), "hf_sean_conv_img: x16 must be 16-byte aligned");
    int rc = ensure_device_current();
    if (rc) return rc;
    const int grid = (res * res + 255) / 256;
    sean_conv_img_kernel<dt><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x16, weight, bias, y, res,
                                                                     channels);
    HF_LAUNCH_OK("sean_conv_img");
    count_launch();
    return HF_OK;
  });
}

}  // extern "C"
