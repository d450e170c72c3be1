// FFHQ face alignment after the landmarks (HairFast utils/shape_predictor.py:145-185) on uint8 RGB images, HWC with
// three channels and a row pitch in pixels.  Every stage reproduces the arithmetic of the library call it replaces
// (DESIGN.md, "Face alignment"):
//   * Pillow's LANCZOS resize: two separable passes (horizontal first) with coefficients normalised to 22-bit
//     fixed point, a uint8 intermediate, round-half-up and a clamp to 0..255 -- integer arithmetic, bit-exact;
//   * numpy's 'reflect' padding (edge not repeated) into float32;
//   * scipy.ndimage.gaussian_filter(img, [s, s, 0]): axis 0 then axis 1, each a correlation in double with scipy's
//     'reflect' extension (edge repeated), accumulated as w0 x[i] + sum_{j = r..1} w_j (x[i - j] + x[i + j]) in that
//     order, rounded to float32 after each axis -- the same operations in the same order, so bit-exact;
//   * the two blends with NumPy 2's float64 right-hand sides, each `img +=` rounded to float32, and the per-channel
//     median by an exact radix select on the float bits;
//   * Pillow's QUAD transform with BILINEAR sampling: double-precision coordinates, truncation to uint8, fill 0.
// No FMA contraction anywhere the library computes a separate multiply and add: the double paths spell out __dmul_rn /
// __dadd_rn.
#include "hf_kernels.cuh"

#include <cmath>
#include <vector>

namespace hf {

constexpr int kAlignPrecisionBits = 22;       // 32 - 8 - 2 fraction bits of the 8-bit resampling coefficients
constexpr int kAlignMaxRadius = 4096;         // Gaussian half width (qsize <= 51200 px)
constexpr int kMedianSel = 6;                 // (channel, lower / upper middle rank)

// ---- Lanczos resample ---------------------------------------------------------------------------------------------
// coeff row of output o: [first input, count, k_0 .. k_{taps-1}] (int32), stride taps + 2
__global__ void __launch_bounds__(256) resample_h_kernel(const uint8_t* __restrict__ src, int src_pitch,
                                                         uint8_t* __restrict__ dst, const int* __restrict__ coeff,
                                                         int taps, int rows, int out_w) {
  const int64_t n = (int64_t)rows * out_w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / out_w), o = (int)(i - (int64_t)y * out_w);
    const int* c = coeff + (size_t)o * (taps + 2);
    const int x0 = __ldg(c), cnt = __ldg(c + 1);
    const uint8_t* p = src + ((size_t)y * src_pitch + x0) * 3;
    int s0 = 1 << (kAlignPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < cnt; ++t) {
      const int k = __ldg(c + 2 + t);
      s0 += (int)__ldg(p + 3 * t) * k;
      s1 += (int)__ldg(p + 3 * t + 1) * k;
      s2 += (int)__ldg(p + 3 * t + 2) * k;
    }
    uint8_t* q = dst + (size_t)i * 3;
    q[0] = (uint8_t)min(max(s0 >> kAlignPrecisionBits, 0), 255);
    q[1] = (uint8_t)min(max(s1 >> kAlignPrecisionBits, 0), 255);
    q[2] = (uint8_t)min(max(s2 >> kAlignPrecisionBits, 0), 255);
  }
}

// one thread per (output row, column byte): coalesced along the row
__global__ void __launch_bounds__(256) resample_v_kernel(const uint8_t* __restrict__ src, int src_pitch,
                                                         uint8_t* __restrict__ dst, const int* __restrict__ coeff,
                                                         int taps, int out_h, int w) {
  const int row_bytes = w * 3;
  const int64_t n = (int64_t)out_h * row_bytes;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int o = (int)(i / row_bytes), b = (int)(i - (int64_t)o * row_bytes);
    const int* c = coeff + (size_t)o * (taps + 2);
    const int y0 = __ldg(c), cnt = __ldg(c + 1);
    const uint8_t* p = src + (size_t)y0 * src_pitch * 3 + b;
    int s = 1 << (kAlignPrecisionBits - 1);
    for (int t = 0; t < cnt; ++t) s += (int)__ldg(p + (size_t)t * src_pitch * 3) * __ldg(c + 2 + t);
    dst[i] = (uint8_t)min(max(s >> kAlignPrecisionBits, 0), 255);
  }
}

// ---- pad, blur, blend ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int numpy_reflect(int i, int n) {     // np.pad 'reflect': ... c b | a b c d | c b ...
  if (n == 1) return 0;
  const int period = 2 * (n - 1);
  i %= period;
  if (i < 0) i += period;
  return i < n ? i : period - i;
}
__device__ __forceinline__ int scipy_reflect(int i, int n) {     // ndimage 'reflect': ... b a | a b c d | d c ...
  const int period = 2 * n;
  i %= period;
  if (i < 0) i += period;
  return i < n ? i : period - 1 - i;
}

// P[y][x][c] = float(src[reflect(y - top)][reflect(x - left)][c])
__global__ void __launch_bounds__(256) pad_reflect_kernel(const uint8_t* __restrict__ src, int H, int W, int pitch,
                                                          int left, int top, float* __restrict__ P, int Hp, int Wp) {
  const int64_t n = (int64_t)Hp * Wp * 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = i / 3;
    const int c = (int)(i - pix * 3);
    const int y = (int)(pix / Wp), x = (int)(pix - (int64_t)y * Wp);
    const int sy = numpy_reflect(y - top, H), sx = numpy_reflect(x - left, W);
    P[i] = (float)__ldg(src + ((size_t)sy * pitch + sx) * 3 + c);
  }
}

// the float64 mask of :172-174, np.float32(x) / pad[0] promoted to float64 by the int64 pad array
__device__ __forceinline__ double pad_mask(int x, int y, int Wp, int Hp, int4 pad) {
  const double mx = fmin(__ddiv_rn((double)x, (double)pad.x), __ddiv_rn((double)(Wp - 1 - x), (double)pad.z));
  const double my = fmin(__ddiv_rn((double)y, (double)pad.y), __ddiv_rn((double)(Hp - 1 - y), (double)pad.w));
  return fmax(__dadd_rn(1.0, -mx), __dadd_rn(1.0, -my));
}

// One axis of gaussian_filter (float32 in, float32 out, double inside).  axis 0 runs down the columns (stride Wp * 3),
// axis 1 along the rows (stride 3).  BLEND (axis 1 only): the output is the first blend of :176,
//   out = f32(P + f64(f32(g - P)) * clip(3 mask + 1, 0, 1)).
template <int AXIS, bool BLEND>
__global__ void __launch_bounds__(256) gauss_axis_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                         const double* __restrict__ w, int radius, int Hp, int Wp,
                                                         const float* __restrict__ P, int4 pad) {
  const int64_t n = (int64_t)Hp * Wp * 3;
  const int len = AXIS == 0 ? Hp : Wp;
  const int64_t stride = AXIS == 0 ? (int64_t)Wp * 3 : 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = i / 3;
    const int c = (int)(i - pix * 3);
    const int y = (int)(pix / Wp), x = (int)(pix - (int64_t)y * Wp);
    const int pos = AXIS == 0 ? y : x;
    const float* line = in + (AXIS == 0 ? ((int64_t)x * 3 + c) : ((int64_t)y * Wp * 3 + c));
    double acc = __dmul_rn((double)__ldg(line + pos * stride), __ldg(w));
    if (pos - radius >= 0 && pos + radius < len) {               // interior: no extension needed
      const float* lp = line + (int64_t)pos * stride;
      for (int j = radius; j > 0; --j) {
        const double a = (double)__ldg(lp - j * stride), b = (double)__ldg(lp + j * stride);
        acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(a, b), __ldg(w + j)));
      }
    } else {
      for (int j = radius; j > 0; --j) {
        const double a = (double)__ldg(line + scipy_reflect(pos - j, len) * stride);
        const double b = (double)__ldg(line + scipy_reflect(pos + j, len) * stride);
        acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(a, b), __ldg(w + j)));
      }
    }
    float g = __double2float_rn(acc);
    if (BLEND) {
      const float p = __ldg(P + i);
      const double m = pad_mask(x, y, Wp, Hp, pad);
      const double k = fmin(fmax(__dadd_rn(__dmul_rn(m, 3.0), 1.0), 0.0), 1.0);
      g = __double2float_rn(__dadd_rn((double)p, __dmul_rn((double)__fsub_rn(g, p), k)));
    }
    out[i] = g;
  }
}

// ---- exact median of each channel: radix select, 8 bits per pass from the top --------------------------------------
__device__ __forceinline__ uint32_t float_key(float f) {         // order-preserving map of the float bits
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}
struct MedianState {
  uint32_t prefix[kMedianSel];      // key bits chosen so far, selection s = channel * 2 + (0 lower, 1 upper)
  uint32_t rank[kMedianSel];        // rank still to find among the keys that match the prefix
  uint32_t hist[kMedianSel][256];
};

__global__ void __launch_bounds__(256) median_hist_kernel(const float* __restrict__ x, int64_t pixels,
                                                          MedianState* __restrict__ st, int shift) {
  __shared__ uint32_t h[kMedianSel][256];
  __shared__ uint32_t pre[kMedianSel];
  for (int i = threadIdx.x; i < kMedianSel * 256; i += blockDim.x) (&h[0][0])[i] = 0;
  if (threadIdx.x < kMedianSel) pre[threadIdx.x] = st->prefix[threadIdx.x];
  __syncthreads();
  const int hi = shift + 8;                        // bits above this pass's digit must match the prefix
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < pixels * 3;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 3);
    const uint32_t k = float_key(__ldg(x + i));
    const uint32_t d = (k >> shift) & 255u;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int s = 2 * c + r;
      if (hi >= 32 || (k >> hi) == (pre[s] >> hi)) atomicAdd(&h[s][d], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kMedianSel * 256; i += blockDim.x) {
    const uint32_t v = (&h[0][0])[i];
    if (v) atomicAdd(&(&st->hist[0][0])[i], v);
  }
}

// one warp per selection: choose the digit, clear the histogram for the next pass; after the last pass write the
// median, numpy's mean of the two middle values for an even count (float32 sum, then halved)
__global__ void __launch_bounds__(32 * kMedianSel) median_select_kernel(MedianState* __restrict__ st, int shift,
                                                                        float* __restrict__ med, int last) {
  const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    uint32_t cum = 0, k = st->rank[s];
    int d = 0;
    for (; d < 256; ++d) {
      const uint32_t h = st->hist[s][d];
      if (cum + h > k) break;
      cum += h;
    }
    st->prefix[s] |= (uint32_t)d << shift;
    st->rank[s] = k - cum;
  }
  __syncwarp();
  for (int d = lane; d < 256; d += 32) st->hist[s][d] = 0;
  if (last) {
    __syncthreads();
    if (threadIdx.x < 3) {
      const float lo = key_float(st->prefix[2 * threadIdx.x]), up = key_float(st->prefix[2 * threadIdx.x + 1]);
      med[threadIdx.x] = __fmul_rn(__fadd_rn(lo, up), 0.5f);
    }
  }
}

__global__ void median_init_kernel(MedianState* __restrict__ st, int64_t pixels) {
  const int s = threadIdx.x;
  if (s < kMedianSel) {
    st->prefix[s] = 0;
    // odd count: both selections take the middle rank, so lo + up halves back to it exactly
    st->rank[s] = (uint32_t)((pixels & 1) ? pixels / 2 : pixels / 2 - 1 + (s & 1));
  }
  for (int i = threadIdx.x; i < kMedianSel * 256; i += blockDim.x) (&st->hist[0][0])[i] = 0;
}

// the second blend of :177 and the conversion of :178:
//   img = f32(img + f64(f32(median - img)) * clip(mask, 0, 1));  out = uint8(clip(rint(img), 0, 255))
__global__ void __launch_bounds__(256) blend_median_u8_kernel(const float* __restrict__ img,
                                                              const float* __restrict__ med, uint8_t* __restrict__ out,
                                                              int Hp, int Wp, int4 pad) {
  const int64_t n = (int64_t)Hp * Wp * 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = i / 3;
    const int c = (int)(i - pix * 3);
    const int y = (int)(pix / Wp), x = (int)(pix - (int64_t)y * Wp);
    const float v = __ldg(img + i);
    const double m = fmin(fmax(pad_mask(x, y, Wp, Hp, pad), 0.0), 1.0);
    const float r = __double2float_rn(__dadd_rn((double)v, __dmul_rn((double)__fsub_rn(__ldg(med + c), v), m)));
    out[i] = (uint8_t)fminf(fmaxf(rintf(r), 0.f), 255.f);
  }
}

// ---- QUAD transform, BILINEAR ---------------------------------------------------------------------------------------
struct QuadCoeffs {
  double a[8];
};
// output (x, y) samples source (a0 + a1 u + a2 v + a3 u v, a4 + a5 u + a6 v + a7 u v) at u = x + 0.5, v = y + 0.5;
// outside [0, W) x [0, H) -> 0; else bilinear between the pixel centres around it (indices clamped to the image,
// the lower row repeated past the bottom edge), truncated to uint8
__global__ void __launch_bounds__(256) quad_bilinear_kernel(const uint8_t* __restrict__ src, int H, int W, int pitch,
                                                            uint8_t* __restrict__ dst, int out_w, int out_h,
                                                            const QuadCoeffs q) {
  const int64_t n = (int64_t)out_w * out_h;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / out_w), ox = (int)(i - (int64_t)oy * out_w);
    const double u = (double)ox + 0.5, v = (double)oy + 0.5;
    const double uv1 = __dmul_rn(__dmul_rn(q.a[3], u), v), uv2 = __dmul_rn(__dmul_rn(q.a[7], u), v);
    double xs = __dadd_rn(__dadd_rn(__dadd_rn(q.a[0], __dmul_rn(q.a[1], u)), __dmul_rn(q.a[2], v)), uv1);
    double ys = __dadd_rn(__dadd_rn(__dadd_rn(q.a[4], __dmul_rn(q.a[5], u)), __dmul_rn(q.a[6], v)), uv2);
    uint8_t* o = dst + (size_t)i * 3;
    if (!(xs >= 0.0 && xs < (double)W && ys >= 0.0 && ys < (double)H)) {
      o[0] = o[1] = o[2] = 0;
      continue;
    }
    xs = __dadd_rn(xs, -0.5);
    ys = __dadd_rn(ys, -0.5);
    const double fx = floor(xs), fy = floor(ys);
    const int ix = (int)fx, iy = (int)fy;
    const double dx = __dadd_rn(xs, -fx), dy = __dadd_rn(ys, -fy);
    const int x0 = min(max(ix, 0), W - 1), x1 = min(max(ix + 1, 0), W - 1);
    const int y0 = min(max(iy, 0), H - 1);
    const bool row2 = iy + 1 >= 0 && iy + 1 < H;
    const uint8_t* r0 = src + (size_t)y0 * pitch * 3;
    const uint8_t* r1 = src + (size_t)(row2 ? iy + 1 : y0) * pitch * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int a0 = __ldg(r0 + x0 * 3 + c), b0 = __ldg(r0 + x1 * 3 + c);
      const double v1 = __dadd_rn((double)a0, __dmul_rn((double)(b0 - a0), dx));
      double v2 = v1;
      if (row2) {
        const int a1 = __ldg(r1 + x0 * 3 + c), b1 = __ldg(r1 + x1 * 3 + c);
        v2 = __dadd_rn((double)a1, __dmul_rn((double)(b1 - a1), dx));
      }
      const double r = __dadd_rn(v1, __dmul_rn(__dadd_rn(v2, -v1), dy));
      o[c] = (uint8_t)min(max((int)r, 0), 255);
    }
  }
}

// ---- host: Pillow's resampling coefficients for one axis (LANCZOS, support 3) ---------------------------------------
static double lanczos_weight(double x) {
  if (!(-3.0 <= x && x < 3.0)) return 0.0;
  auto sinc = [](double t) {
    if (t == 0.0) return 1.0;
    t = t * M_PI;
    return sin(t) / t;
  };
  return sinc(x) * sinc(x / 3.0);
}

static int lanczos_taps(int in_size, int out_size) {
  const double scale = (double)in_size / out_size;
  const double support = 3.0 * (scale > 1.0 ? scale : 1.0);
  return (int)ceil(support) * 2 + 1;
}

static void lanczos_table(int in_size, int out_size, int* table) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale > 1.0 ? scale : 1.0;
  const double support = 3.0 * filterscale, ss = 1.0 / filterscale;
  const int taps = lanczos_taps(in_size, out_size);
  std::vector<double> k(taps);
  for (int o = 0; o < out_size; ++o) {
    const double center = (o + 0.5) * scale;
    int lo = (int)(center - support + 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)(center + support + 0.5);
    if (hi > in_size) hi = in_size;
    const int cnt = hi - lo;
    double sum = 0.0;
    for (int t = 0; t < cnt; ++t) {
      k[t] = lanczos_weight((t + lo - center + 0.5) * ss);
      sum += k[t];
    }
    int* row = table + (size_t)o * (taps + 2);
    row[0] = lo;
    row[1] = cnt;
    for (int t = 0; t < taps; ++t) {
      double v = t < cnt ? k[t] : 0.0;
      if (t < cnt && sum != 0.0) v /= sum;
      const double s = v * (1 << kAlignPrecisionBits);
      row[2 + t] = (int)(v < 0.0 ? -0.5 + s : 0.5 + s);
    }
  }
}

static int launch_grid(int64_t n) { return grid_for(n); }

}  // namespace hf

using namespace hf;

extern "C" {

int hf_align_lanczos_taps(int in_size, int out_size) {
  if (in_size <= 0 || out_size <= 0) {
    set_error("align_lanczos_taps: sizes must be positive");
    return -1;
  }
  return lanczos_taps(in_size, out_size);
}

int hf_align_lanczos_coeffs(int in_size, int out_size, int* table) {
  HF_REQUIRE(in_size > 0 && out_size > 0 && table, "align_lanczos_coeffs: bad arguments");
  HF_REQUIRE(in_size <= (1 << 20) && out_size <= (1 << 20), "align_lanczos_coeffs: size over 2^20");
  lanczos_table(in_size, out_size, table);
  return HF_OK;
}

size_t hf_align_resample_workspace_bytes(int H, int W, int Ho, int Wo) {
  if (H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0) return 0;
  return (W != Wo && H != Ho) ? (size_t)H * Wo * 3 : 0;
}

int hf_align_resample_u8(const uint8_t* src, int H, int W, int src_pitch, uint8_t* dst, int Ho, int Wo,
                         const int* coeff_x, const int* coeff_y, uint8_t* workspace, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  HF_REQUIRE(src && dst, "align_resample: null pointer");
  HF_REQUIRE(H > 0 && W > 0 && Ho > 0 && Wo > 0 && src_pitch >= W, "align_resample: bad shape");
  const bool need_h = Wo != W, need_v = Ho != H;
  HF_REQUIRE(!need_h || coeff_x, "align_resample: horizontal coefficients missing");
  HF_REQUIRE(!need_v || coeff_y, "align_resample: vertical coefficients missing");
  HF_REQUIRE(!(need_h && need_v) || workspace, "align_resample: workspace missing");
  if (!need_h && !need_v) {
    HF_CUDA_OK(cudaMemcpy2DAsync(dst, (size_t)W * 3, src, (size_t)src_pitch * 3, (size_t)W * 3, H,
                                 cudaMemcpyDeviceToDevice, st));
    return HF_OK;
  }
  const uint8_t* vin = src;
  int vin_pitch = src_pitch;
  if (need_h) {
    uint8_t* hout = need_v ? workspace : dst;
    const int64_t n = (int64_t)H * Wo;
    resample_h_kernel<<<launch_grid(n), 256, 0, st>>>(src, src_pitch, hout, coeff_x, lanczos_taps(W, Wo), H, Wo);
    HF_LAUNCH_OK("align_resample_h");
    count_launch();
    vin = hout;
    vin_pitch = Wo;
  }
  if (need_v) {
    const int64_t n = (int64_t)Ho * Wo * 3;
    resample_v_kernel<<<launch_grid(n), 256, 0, st>>>(vin, vin_pitch, dst, coeff_y, lanczos_taps(H, Ho), Ho, Wo);
    HF_LAUNCH_OK("align_resample_v");
    count_launch();
  }
  return HF_OK;
}

size_t hf_align_pad_blend_workspace_bytes(int Hp, int Wp) {
  if (Hp <= 0 || Wp <= 0) return 0;
  const size_t plane = ((size_t)Hp * Wp * 3 * sizeof(float) + 255) / 256 * 256;
  return 3 * plane + (sizeof(MedianState) + 255) / 256 * 256 + 256;
}

static int gaussian_passes(const float* x, float* tmp, float* y, const double* weights, int radius, int Hp, int Wp,
                           const float* P, int4 pad, bool blend, cudaStream_t st) {
  const int64_t n = (int64_t)Hp * Wp * 3;
  gauss_axis_kernel<0, false><<<launch_grid(n), 256, 0, st>>>(x, tmp, weights, radius, Hp, Wp, nullptr, pad);
  HF_LAUNCH_OK("align_gauss_axis0");
  count_launch();
  if (blend)
    gauss_axis_kernel<1, true><<<launch_grid(n), 256, 0, st>>>(tmp, y, weights, radius, Hp, Wp, P, pad);
  else
    gauss_axis_kernel<1, false><<<launch_grid(n), 256, 0, st>>>(tmp, y, weights, radius, Hp, Wp, nullptr, pad);
  HF_LAUNCH_OK("align_gauss_axis1");
  count_launch();
  return HF_OK;
}

static int median_launch(const float* x, int64_t pixels, MedianState* state, float* med, cudaStream_t st) {
  median_init_kernel<<<1, 256, 0, st>>>(state, pixels);
  HF_LAUNCH_OK("align_median_init");
  count_launch();
  const int grid = std::min<int64_t>((pixels * 3 + 255) / 256, (int64_t)num_sms() * 4);
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    median_hist_kernel<<<grid, 256, 0, st>>>(x, pixels, state, shift);
    HF_LAUNCH_OK("align_median_hist");
    median_select_kernel<<<1, 32 * kMedianSel, 0, st>>>(state, shift, med, pass == 3);
    HF_LAUNCH_OK("align_median_select");
    count_launch(2);
  }
  return HF_OK;
}

int hf_align_gaussian_f32(const float* x, float* y, int Hp, int Wp, const double* weights, int radius,
                          float* workspace, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  HF_REQUIRE(x && y && weights && workspace, "align_gaussian: null pointer");
  HF_REQUIRE(Hp > 0 && Wp > 0 && (int64_t)Hp * Wp * 3 < ((int64_t)1 << 31), "align_gaussian: bad shape");
  HF_REQUIRE(radius >= 0 && radius <= kAlignMaxRadius, "align_gaussian: radius %d outside 0..%d", radius,
             kAlignMaxRadius);
  return gaussian_passes(x, workspace, y, weights, radius, Hp, Wp, nullptr, make_int4(1, 1, 1, 1), false,
                         (cudaStream_t)stream);
}

size_t hf_align_median_workspace_bytes(void) { return sizeof(MedianState); }

int hf_align_median_f32(const float* x, long long pixels, float* med, void* workspace, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  HF_REQUIRE(x && med && workspace, "align_median: null pointer");
  HF_REQUIRE(pixels > 0 && pixels * 3 < ((long long)1 << 32), "align_median: bad pixel count");
  return median_launch(x, pixels, (MedianState*)workspace, med, (cudaStream_t)stream);
}

int hf_align_pad_blend_u8(const uint8_t* src, int H, int W, int src_pitch, const int* pad, const double* weights,
                          int radius, uint8_t* dst, void* workspace, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  HF_REQUIRE(src && pad && weights && dst && workspace, "align_pad_blend: null pointer");
  HF_REQUIRE(H > 0 && W > 0 && src_pitch >= W, "align_pad_blend: bad shape");
  HF_REQUIRE(pad[0] > 0 && pad[1] > 0 && pad[2] > 0 && pad[3] > 0, "align_pad_blend: pads must be positive");
  HF_REQUIRE(radius >= 0 && radius <= kAlignMaxRadius, "align_pad_blend: radius %d outside 0..%d", radius,
             kAlignMaxRadius);
  const int Hp = H + pad[1] + pad[3], Wp = W + pad[0] + pad[2];
  const int64_t n = (int64_t)Hp * Wp * 3;
  HF_REQUIRE(n < ((int64_t)1 << 31), "align_pad_blend: padded image too large");
  const int4 pd = make_int4(pad[0], pad[1], pad[2], pad[3]);
  const size_t plane = ((size_t)n * sizeof(float) + 255) / 256 * 256;
  char* ws = (char*)workspace;
  float* P = (float*)ws;
  float* tmp = (float*)(ws + plane);
  float* img = (float*)(ws + 2 * plane);
  MedianState* state = (MedianState*)(ws + 3 * plane);
  float* med = (float*)(ws + 3 * plane + (sizeof(MedianState) + 255) / 256 * 256);
  pad_reflect_kernel<<<launch_grid(n), 256, 0, st>>>(src, H, W, src_pitch, pad[0], pad[1], P, Hp, Wp);
  HF_LAUNCH_OK("align_pad_reflect");
  count_launch();
  rc = gaussian_passes(P, tmp, img, weights, radius, Hp, Wp, P, pd, true, st);
  if (rc) return rc;
  rc = median_launch(img, (int64_t)Hp * Wp, state, med, st);
  if (rc) return rc;
  blend_median_u8_kernel<<<launch_grid(n), 256, 0, st>>>(img, med, dst, Hp, Wp, pd);
  HF_LAUNCH_OK("align_blend_median");
  count_launch();
  return HF_OK;
}

int hf_align_quad_u8(const uint8_t* src, int H, int W, int src_pitch, const double* coeffs, uint8_t* dst, int out_w,
                     int out_h, void* stream) {
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  HF_REQUIRE(src && coeffs && dst, "align_quad: null pointer");
  HF_REQUIRE(H > 0 && W > 0 && src_pitch >= W && out_w > 0 && out_h > 0, "align_quad: bad shape");
  QuadCoeffs q;
  for (int i = 0; i < 8; ++i) q.a[i] = coeffs[i];
  const int64_t n = (int64_t)out_w * out_h;
  quad_bilinear_kernel<<<launch_grid(n), 256, 0, st>>>(src, H, W, src_pitch, dst, out_w, out_h, q);
  HF_LAUNCH_OK("align_quad");
  count_launch();
  return HF_OK;
}

}  // extern "C"
