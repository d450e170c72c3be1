// CtrlHair's shape adaptor (models/CtrlHair/shape_branch/model.py:146-199, Alignment.mask_generator): label map,
// the one-hot first encoder layer as a lookup, the split-K "skinny" GEMM of the weight-streaming layers, the
// whole-sample LayerNorm + LeakyReLU, and the 19 logits + argmax.  The GEMM itself lives in hf_splitk_gemm.cuh.
// Fixed summation orders everywhere (deterministic); the only atomic is the out-of-range label count.
#include <algorithm>

#include "hf_splitk_gemm.cuh"

namespace hf {
namespace {

constexpr int kLabels = 20;       // 19 classes + 19, the all-zero one-hot of 255 (mask_label_to_one_hot)
constexpr int kOutClasses = 19;
constexpr int kHairIdx = 13;      // HAIR_IDX (global_value_utils.py:52)
constexpr int kOutC = 32;         // channels of both decoders' last LayerNorm layer

// ------------------------------------------------------------------------------------------------
// Label map.  mask_label_to_one_hot (shape_util.py:6-14) rewrites 255 -> 19 in the caller's long tensor and scatters
// into 20 channels, dropping the last: 19 is the all-zero one-hot.  Labels outside {0..19, 255} are counted in *bad
// (the reference's scatter_ would index out of range) and map to 19.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) shape_labels_kernel(long long* __restrict__ lab, int8_t* __restrict__ L,
                                                           int* __restrict__ bad, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    long long v = lab[i];
    if (v == 255) {
      v = 19;
      lab[i] = 19;
    }
    const bool ok = v >= 0 && v < kLabels;
    if (!ok) atomicAdd(bad, 1);
    L[i] = ok ? (int8_t)v : (int8_t)(kLabels - 1);
  }
}

// ------------------------------------------------------------------------------------------------
// MaskEncoder layer 0 (ZeroPad 1 + Conv 4x4 stride 2 over cat[one-hot, 40 positional channels]) as a lookup:
// y[p, c] = cmap[p, c] + sum_{tap, source inside} table[tap][L(source)][c], where cmap is the positional channels'
// conv plus the bias (input independent, computed when packing) and table[tap][j] the one-hot weights of label j
// (zero rows for the labels the encoder does not see).  One thread = 8 channels of one pixel; output 16-bit NHWC.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) shape_onehot_s2_kernel(const int8_t* __restrict__ L, const float* __restrict__ table,
                                                              const float* __restrict__ cmap, uint16_t* __restrict__ y,
                                                              int R, int C8) {
  const int C = C8 * 8, S = 2 * R;
  const int total = R * R * C8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = (i % C8) * 8, p = i / C8, oy = p / R, ox = p % R;
    float v[8];
    const float4 c0 = __ldg(reinterpret_cast<const float4*>(cmap + (size_t)p * C + c));
    const float4 c1 = __ldg(reinterpret_cast<const float4*>(cmap + (size_t)p * C + c + 4));
    v[0] = c0.x; v[1] = c0.y; v[2] = c0.z; v[3] = c0.w; v[4] = c1.x; v[5] = c1.y; v[6] = c1.z; v[7] = c1.w;
#pragma unroll
    for (int tap = 0; tap < 16; ++tap) {
      const int yy = 2 * oy - 1 + tap / 4, xx = 2 * ox - 1 + tap % 4;
      if (yy < 0 || yy >= S || xx < 0 || xx >= S) continue;
      const float* t = table + ((size_t)tap * kLabels + L[yy * S + xx]) * C + c;
      const float4 a = __ldg(reinterpret_cast<const float4*>(t)), b = __ldg(reinterpret_cast<const float4*>(t + 4));
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    st8<DT>(y + (size_t)p * C + c, v);
  }
}

// ------------------------------------------------------------------------------------------------
// CtrlHair LayerNorm (my_torchlib/module.py:183-205) + LeakyReLU over one whole sample of 16-bit NHWC:
// (x - mean) / (std + eps) * gamma[c] + beta[c], std unbiased.  Pass 1: G block sums of x; pass 2: G block sums of
// (x - mean)^2, each block forming mean from pass 1's sums in order; apply: every block forms mean and std the same
// way.  Fixed-order block reductions, no atomics.
// ------------------------------------------------------------------------------------------------
constexpr int kLnThreads = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < kLnThreads / 32; ++i) t += red[i];
  return t;
}

__device__ __forceinline__ float ordered_sum(const float* part, int G) {
  float t = 0.f;
  for (int g = 0; g < G; ++g) t += part[g];
  return t;
}

template <int DT, bool CENTER>
__global__ void __launch_bounds__(kLnThreads) shape_ln_partial_kernel(const uint16_t* __restrict__ x, int64_t n8,
                                                                      int64_t chunk8, const float* __restrict__ sums,
                                                                      int G, float* __restrict__ part) {
  __shared__ float red[kLnThreads / 32];
  __shared__ float s_mean;
  float m = 0.f;
  if (CENTER) {
    if (threadIdx.x == 0) s_mean = ordered_sum(sums, G) / (float)(n8 * 8);
    __syncthreads();
    m = s_mean;
  }
  float acc = 0.f;
  const int64_t end = min(n8, (int64_t)(blockIdx.x + 1) * chunk8);
  for (int64_t i = blockIdx.x * chunk8 + threadIdx.x; i < end; i += kLnThreads) {
    float v[8];
    ld8<DT>(x + i * 8, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (CENTER) {
        const float d = v[k] - m;
        acc = fmaf(d, d, acc);
      } else {
        acc += v[k];
      }
    }
  }
  const float t = block_sum(acc, red);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

template <int DT>
__global__ void __launch_bounds__(kLnThreads) shape_ln_apply_kernel(const uint16_t* __restrict__ x,
                                                                    const float* __restrict__ sums,
                                                                    const float* __restrict__ sqsums, int G, int64_t n8,
                                                                    int C8, const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, float eps,
                                                                    float slope, uint16_t* __restrict__ y) {
  __shared__ float s_mean, s_inv;
  if (threadIdx.x == 0) {
    const float n = (float)(n8 * 8);
    s_mean = ordered_sum(sums, G) / n;
    s_inv = 1.f / (sqrtf(ordered_sum(sqsums, G) / (n - 1.f)) + eps);
  }
  __syncthreads();
  const float m = s_mean, inv = s_inv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8) * 8;
    float v[8];
    ld8<DT>(x + i * 8, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float t = (v[k] - m) * inv * __ldg(gamma + c + k) + __ldg(beta + c + k);
      v[k] = t > 0.f ? t : t * slope;
    }
    st8<DT>(y + i * 8, v);
  }
}

int ln_blocks(int64_t n8) { return (int)std::max<int64_t>(1, std::min<int64_t>(2 * num_sms(), n8 / 512)); }

// ------------------------------------------------------------------------------------------------
// Both decoders' out_layer (Conv 3x3 pad 1, 32 -> 1 | 18) and argmax over cat[face[:13], hair, face[13:]]
// (model.py:180-183; softmax is monotone and is not computed).  table [19][9][32] fp32 in that channel order, fp32
// arithmetic, ties to the first index (torch.argmax).  One thread = one pixel; int64 labels.
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) shape_logits_argmax_kernel(const uint16_t* __restrict__ hair,
                                                                  const uint16_t* __restrict__ face,
                                                                  const float* __restrict__ table,
                                                                  const float* __restrict__ bias,
                                                                  long long* __restrict__ out, int R) {
  __shared__ float sw[kOutClasses * 9 * kOutC];
  for (int i = threadIdx.x; i < kOutClasses * 9 * kOutC; i += blockDim.x) sw[i] = table[i];
  __syncthreads();
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < R * R; p += gridDim.x * blockDim.x) {
    const int py = p / R, px = p % R;
    float lg[kOutClasses];
#pragma unroll
    for (int j = 0; j < kOutClasses; ++j) lg[j] = __ldg(bias + j);
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = py + tap / 3 - 1, xx = px + tap % 3 - 1;
      if (yy < 0 || yy >= R || xx < 0 || xx >= R) continue;
      const size_t q = ((size_t)yy * R + xx) * kOutC;
#pragma unroll
      for (int c8 = 0; c8 < kOutC / 8; ++c8) {
        float fv[8], hv[8];
        ld8<DT>(face + q + c8 * 8, fv);
        ld8<DT>(hair + q + c8 * 8, hv);
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int j = 0; j < kOutClasses; ++j)
            lg[j] = fmaf(sw[(j * 9 + tap) * kOutC + c8 * 8 + k], j == kHairIdx ? hv[k] : fv[k], lg[j]);
      }
    }
    int best = 0;
#pragma unroll
    for (int j = 1; j < kOutClasses; ++j)
      if (lg[j] > lg[best]) best = j;
    out[p] = best;
  }
}

int gemm_shape(int mode, int cin, int hin, int win, GemmShape* g) {
  HF_REQUIRE(mode >= 0 && mode <= 2, "shape_gemm: mode %d (0 1x1, 1 conv 4x4 s2, 2 nearest-up conv 3x3)", mode);
  HF_REQUIRE(cin > 0 && cin % 8 == 0 && hin > 0 && win > 0, "shape_gemm: bad input %d x %d x %d (channels %% 8)", hin,
             win, cin);
  if (mode == 0) *g = GemmShape{hin * win, cin, hin, win, win};
  if (mode == 1) {
    HF_REQUIRE(hin % 2 == 0 && win % 2 == 0, "shape_gemm: stride-2 input %d x %d must be even", hin, win);
    *g = GemmShape{hin / 2 * (win / 2), 16 * cin, hin, win, win / 2};
  }
  if (mode == 2) *g = GemmShape{4 * hin * win, 9 * cin, hin, win, 2 * win};
  return HF_OK;
}

template <int DT, int BN>
int launch_gemm_mode(int mode, const uint16_t* w, const uint16_t* x, float* part, int cout, const GemmShape& g,
                     const int* pl, int cin, cudaStream_t st) {
  if (mode == 0) return launch_gemm<DT, BN, 0>(w, x, part, cout, g, pl, cin, st);
  if (mode == 1) return launch_gemm<DT, BN, 1>(w, x, part, cout, g, pl, cin, st);
  return launch_gemm<DT, BN, 2>(w, x, part, cout, g, pl, cin, st);
}

}  // namespace
}  // namespace hf

using namespace hf;

extern "C" {

int hf_shape_labels(long long* mask, int8_t* labels, int* bad, int n, void* stream) {
  HF_REQUIRE(mask && labels && bad, "hf_shape_labels: null pointer");
  HF_REQUIRE(n > 0, "hf_shape_labels: %d pixels", n);
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  HF_CUDA_OK(cudaMemsetAsync(bad, 0, sizeof(int), st));
  shape_labels_kernel<<<grid_for(n), 256, 0, st>>>(mask, labels, bad, n);
  HF_LAUNCH_OK("shape_labels");
  count_launch();
  return HF_OK;
}

int hf_shape_onehot_s2(const int8_t* labels, const float* table, const float* cmap, void* y16, int res, int channels,
                       int dtype, void* stream) {
  return with_dtype(dtype, "hf_shape_onehot_s2", [&](auto dt) -> int {
    HF_REQUIRE(labels && table && cmap && y16, "hf_shape_onehot_s2: null pointer");
    HF_REQUIRE(res > 0 && channels > 0 && channels % 8 == 0, "hf_shape_onehot_s2: bad shape %d^2 x %d", res, channels);
    HF_REQUIRE(((uintptr_t)table & 15) == 0 && ((uintptr_t)cmap & 15) == 0 && ((uintptr_t)y16 & 15) == 0,
               "hf_shape_onehot_s2: unaligned pointer");
    int rc = ensure_device_current();
    if (rc) return rc;
    const int64_t total = (int64_t)res * res * (channels / 8);
    shape_onehot_s2_kernel<dt><<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(labels, table, cmap, (uint16_t*)y16,
                                                                                  res, channels / 8);
    HF_LAUNCH_OK("shape_onehot_s2");
    count_launch();
    return HF_OK;
  });
}

int hf_shape_gemm_plan(int mode, int cin, int cout, int hin, int win, int sms, int* out) {
  HF_REQUIRE(out && cout > 0 && sms > 0, "hf_shape_gemm_plan: bad arguments");
  GemmShape g;
  int rc = gemm_shape(mode, cin, hin, win, &g);
  if (rc) return rc;
  gemm_plan(g, cout, sms, out);
  return HF_OK;
}

size_t hf_shape_gemm_workspace_bytes(int mode, int cin, int cout, int hin, int win) {
  GemmShape g;
  if (ensure_device_current() || cout <= 0 || gemm_shape(mode, cin, hin, win, &g)) return 0;
  int pl[5];
  gemm_plan(g, cout, num_sms(), pl);
  return (size_t)pl[1] * g.P * cout * sizeof(float);
}

int hf_shape_gemm(int mode, const void* w16, const void* x16, const float* bias, float* y32, void* y16, float* workspace,
                  int cin, int cout, int hin, int win, int dtype, void* stream) {
  return with_dtype(dtype, "hf_shape_gemm", [&](auto dt) -> int {
    HF_REQUIRE(w16 && x16 && workspace && (y32 || y16), "hf_shape_gemm: null pointer");
    HF_REQUIRE(((uintptr_t)w16 & 15) == 0 && ((uintptr_t)x16 & 15) == 0, "hf_shape_gemm: unaligned operand");
    HF_REQUIRE(cout > 0, "hf_shape_gemm: cout %d", cout);
    GemmShape g;
    int rc = gemm_shape(mode, cin, hin, win, &g);
    if (rc) return rc;
    if ((rc = ensure_device_current())) return rc;
    int pl[5];
    gemm_plan(g, cout, num_sms(), pl);
    cudaStream_t st = (cudaStream_t)stream;
    const uint16_t* w = (const uint16_t*)w16;
    const uint16_t* x = (const uint16_t*)x16;
    rc = pl[0] == 8 ? launch_gemm_mode<dt, 8>(mode, w, x, workspace, cout, g, pl, cin, st)
                    : launch_gemm_mode<dt, 64>(mode, w, x, workspace, cout, g, pl, cin, st);
    if (rc) return rc;
    const int64_t n = (int64_t)g.P * cout;
    shape_splitk_reduce_kernel<dt><<<grid_for(n), 256, 0, st>>>(workspace, pl[1], n, cout, n, bias, y32,
                                                                 (uint16_t*)y16);
    HF_LAUNCH_OK("shape_splitk_reduce");
    count_launch(2);
    return HF_OK;
  });
}

size_t hf_shape_layer_norm_workspace_bytes(long long n) {
  if (ensure_device_current() || n <= 0 || n % 8) return 0;
  return (size_t)2 * ln_blocks(n / 8) * sizeof(float);
}

int hf_shape_layer_norm_lrelu(const void* x16, const float* gamma, const float* beta, void* y16, float* workspace,
                              int pixels, int channels, float slope, int dtype, void* stream) {
  return with_dtype(dtype, "hf_shape_layer_norm_lrelu", [&](auto dt) -> int {
    HF_REQUIRE(x16 && gamma && beta && y16 && workspace, "hf_shape_layer_norm_lrelu: null pointer");
    HF_REQUIRE(pixels > 0 && channels > 0 && channels % 8 == 0 && (int64_t)pixels * channels > 1,
               "hf_shape_layer_norm_lrelu: bad shape %d x %d (channels %% 8)", pixels, channels);
    HF_REQUIRE(((uintptr_t)x16 & 15) == 0 && ((uintptr_t)y16 & 15) == 0,
               "hf_shape_layer_norm_lrelu: unaligned pointer");
    int rc = ensure_device_current();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n8 = (int64_t)pixels * channels / 8;
    const int G = ln_blocks(n8);
    const int64_t chunk8 = (n8 + G - 1) / G;
    float* sums = workspace;
    float* sqsums = workspace + G;
    const uint16_t* x = (const uint16_t*)x16;
    shape_ln_partial_kernel<dt, false><<<G, kLnThreads, 0, st>>>(x, n8, chunk8, nullptr, G, sums);
    shape_ln_partial_kernel<dt, true><<<G, kLnThreads, 0, st>>>(x, n8, chunk8, sums, G, sqsums);
    shape_ln_apply_kernel<dt><<<grid_for(n8), kLnThreads, 0, st>>>(x, sums, sqsums, G, n8, channels / 8, gamma, beta,
                                                                   1e-5f, slope, (uint16_t*)y16);
    HF_LAUNCH_OK("shape_layer_norm");
    count_launch(3);
    return HF_OK;
  });
}

int hf_shape_logits_argmax(const void* hair16, const void* face16, const float* table, const float* bias,
                           long long* labels, int res, int dtype, void* stream) {
  return with_dtype(dtype, "hf_shape_logits_argmax", [&](auto dt) -> int {
    HF_REQUIRE(hair16 && face16 && table && bias && labels, "hf_shape_logits_argmax: null pointer");
    HF_REQUIRE(res > 0 && res <= 4096, "hf_shape_logits_argmax: res %d", res);
    HF_REQUIRE(((uintptr_t)hair16 & 15) == 0 && ((uintptr_t)face16 & 15) == 0,
               "hf_shape_logits_argmax: unaligned input");
    int rc = ensure_device_current();
    if (rc) return rc;
    const int grid = (res * res + 255) / 256;
    shape_logits_argmax_kernel<dt><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)hair16,
                                                                           (const uint16_t*)face16, table, bias,
                                                                           labels, res);
    HF_LAUNCH_OK("shape_logits_argmax");
    count_launch();
    return HF_OK;
  });
}

}  // extern "C"
