// HBM-bound SIMT kernels of the hot path: upfirdn2d, fused bias+activation, style affine /
// demodulation tables, NCHW->NHWC modulate+cast pre-pass, RGB combine (+ up-FIR of the skip),
// standalone ToRGB, weight packing.  All fp32 math; 16-bit only as storage for tensor-core operands.
#include "hf_kernels.cuh"
#include <type_traits>

namespace hf {

// =============================================================================================
// upfirdn2d  (reference semantics: models/stylegan2/op/upfirdn2d.py:159-200,
//             op/upfirdn2d_kernel.cu:107-207 -- zero-stuff, pad/crop, convolve (flipped taps), decimate)
// =============================================================================================

// up = 1, down in {1, 2}, 4x4 taps, pads 0..3, planes up to 1040 columns wide: the input side done by the TMA engine.
// Rows are only 4-byte aligned (width 2R+1 after the transposed convolution), so neither 16-byte per-row copies nor a
// tiled tensor map apply.  But a strip of full-width rows of one plane is ONE contiguous span of global memory, so it
// is fetched with 1-D bulk copies (`cp.async.bulk`) of whole-row spans.  A bulk copy needs a 16-byte aligned start and
// size, so the span is widened to the enclosing 16-byte boundaries; the widened span stays inside the tensor only
// because the launcher checks that the base is 16-byte aligned and the total element count a multiple of 4.
// One elected thread keeps up to S chunks of CR rows in flight per CTA (mbarrier complete_tx), so there are no
// per-element copy instructions and no per-element address arithmetic.  The stages are kept small (3 x 16 KB at 1025
// columns) so that several CTAs stay resident per SM and keep enough bytes in flight.  A thread owns the output
// columns t, t+256, ... (conflict-free 4-byte LDS whatever the row's alignment; 2-way for down = 2) and walks down the
// strip with the separable (or general) FIR in registers; padding columns are handled by a masked path that only the
// threads owning an edge column take, padding rows contribute nothing and are never fetched.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst_s, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst_s), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// Rows [lo, hi) of the plane that chunk c of a strip holds (strip row r = input row iy0 + r, nrows rows, CR per chunk)
// and the 16-byte aligned global byte span [a0, a0 + bytes) that contains them.
struct BulkSpan {
  int lo, hi;
  size_t a0;
  uint32_t bytes;
};
__device__ __forceinline__ BulkSpan bulk_span(int c, int CR, int iy0, int nrows, int in_h, int in_w, size_t plane_off) {
  BulkSpan sp;
  sp.lo = max(iy0 + c * CR, 0);
  sp.hi = min(iy0 + min((c + 1) * CR, nrows), in_h);
  const size_t g0 = (plane_off + (size_t)sp.lo * in_w) * 4, g1 = (plane_off + (size_t)max(sp.hi, sp.lo) * in_w) * 4;
  sp.a0 = g0 & ~(size_t)15;
  sp.bytes = (uint32_t)(((g1 + 15) & ~(size_t)15) - sp.a0);
  return sp;
}

template <int DOWN, int NC, int RS, int CR, int S>            // RS output rows per CTA, CR input rows per chunk, S stages
__global__ void __launch_bounds__(256) upfirdn2d_k4_bulk_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                const float* __restrict__ k, int in_h, int in_w,
                                                                int out_h, int out_w, int px0, int py0,
                                                                uint32_t stage_bytes) {
  static_assert(CR % 4 == 0 && (DOWN == 1 || DOWN == 2), "chunk rows keep the accumulator rotation static");
  constexpr int HALO = DOWN == 1 ? 3 : 2;
  constexpr int NACC = DOWN == 1 ? 4 : 2;
  extern __shared__ __align__(128) unsigned char bulk_smem[];
  __shared__ uint64_t full[S];
  const int t = threadIdx.x;
  const int oy0 = blockIdx.y * RS;
  float kr[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kr[i] = __ldg(k + 15 - i);           // flipped taps: kr[a*4+b] = k[3-a][3-b]
  float kx[4], ky[4];
  // rank-1 test on the flipped taps: kr[a][b] == ky[a] * kx[b] with kx = row 0, ky = column 0 / kr[0][0]
  bool separable = kr[0] != 0.f;
#pragma unroll
  for (int b = 0; b < 4; ++b) kx[b] = kr[b];
#pragma unroll
  for (int a = 0; a < 4; ++a) ky[a] = separable ? kr[a * 4] / kr[0] : 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      separable = separable && fabsf(ky[a] * kx[b] - kr[a * 4 + b]) <= 1e-6f * fabsf(kr[a * 4 + b]) + 1e-30f;
  const size_t plane_off = (size_t)blockIdx.z * in_h * in_w;          // elements
  float* yp = y + (size_t)blockIdx.z * out_h * out_w;
  const int nrows = DOWN * min(RS, out_h - oy0) + HALO;               // strip rows that feed a stored output row
  const int nchunks = (nrows + CR - 1) / CR;
  const int iy0 = DOWN * oy0 - py0;                                   // input row of strip row 0 (>= -3)
  const uint32_t smem_s = smem_u32(bulk_smem);
  auto issue_chunk = [&](int c) {                                     // one thread
    const BulkSpan sp = bulk_span(c, CR, iy0, nrows, in_h, in_w, plane_off);
    if (sp.lo >= sp.hi) return;                                       // only trailing chunks can be empty
    const int s = c % S;
    mbar_expect_tx(&full[s], sp.bytes);
    bulk_load_1d(smem_s + (uint32_t)s * stage_bytes, reinterpret_cast<const unsigned char*>(x) + sp.a0, sp.bytes,
                 &full[s]);
  };
  if (t == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (t == 0)
    for (int c = 0; c < S && c < nchunks; ++c) issue_chunk(c);

  // column state (row-invariant): byte offset of tap 0 inside a row; edge columns take the masked path
  uint32_t off[NC];
  uint32_t edge = 0, live = 0;
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const int ox = t + 256 * j, ix = DOWN * ox - px0;
    const bool in_img = ox < out_w;
    const bool inside = ix >= 0 && ix + 3 < in_w;
    off[j] = (in_img && inside) ? (uint32_t)ix * 4u : 0u;
    if (in_img) live |= 1u << j;
    if (in_img && !inside) edge |= 1u << j;
  }
  const bool any_edge = edge != 0;
  float* dst_row = yp + (size_t)oy0 * out_w + t;                       // next output row to complete (they complete in order)
  const uint32_t row_bytes = (uint32_t)in_w * 4u;

  // The whole strip loop is instantiated once per FIR kind so that the separable test is not re-evaluated per row.
  auto run = [&](auto sep_tag) {
    constexpr bool SEP = decltype(sep_tag)::value;
    float acc[NACC][NC];
#pragma unroll
    for (int i = 0; i < NACC; ++i)
#pragma unroll
      for (int j = 0; j < NC; ++j) acc[i][j] = 0.f;
#pragma unroll 1
    for (int c = 0; c < nchunks; ++c) {
      const BulkSpan sp = bulk_span(c, CR, iy0, nrows, in_h, in_w, plane_off);
      const int s = c % S;
      if (sp.lo < sp.hi) mbar_wait(&full[s], (uint32_t)(c / S) & 1u);
      // shared address of strip row c*CR (may lie before the span when that row is padding: never dereferenced then)
      uint32_t row_s = smem_s + (uint32_t)s * stage_bytes +
                       (uint32_t)(int32_t)((int64_t)((plane_off + (size_t)sp.lo * in_w) * 4 - sp.a0) +
                                           (int64_t)(iy0 + c * CR - sp.lo) * (int64_t)row_bytes);
#pragma unroll
      for (int u8 = 0; u8 < CR; ++u8, row_s += row_bytes) {
        const int r = c * CR + u8;
        if (r < nrows) {                                               // block-uniform
          const int iy = iy0 + r;
          const bool row_ok = iy >= sp.lo && iy < sp.hi;               // block-uniform: padding rows add nothing
          // DOWN 1: input row r feeds output rows r - a (tap row a), slot (r - a) & 3.  DOWN 2: r = 2m + e feeds
          // output m (tap row e, slot cur) and m - 1 (tap row e + 2, slot prev).  Static: chunks start at multiples of 4.
          const int u = u8 & 3, e = u8 & 1, cur = (u8 >> 1) & 1, prev = cur ^ 1;
          if (row_ok) {
            float v[NC][4];
#pragma unroll
            for (int j = 0; j < NC; ++j)
#pragma unroll
              for (int b = 0; b < 4; ++b) v[j][b] = lds_f32(row_s + off[j] + 4u * b);
            if (any_edge) {                                            // the few threads that own an edge column redo it
#pragma unroll
              for (int j = 0; j < NC; ++j)
                if (edge & (1u << j)) {
                  const int ix = DOWN * (t + 256 * j) - px0;
#pragma unroll
                  for (int b = 0; b < 4; ++b)
                    v[j][b] = (ix + b >= 0 && ix + b < in_w) ? lds_f32(row_s + (uint32_t)(ix + b) * 4u) : 0.f;
                }
            }
            if constexpr (SEP) {
#pragma unroll
              for (int j = 0; j < NC; ++j) {
                float h = v[j][0] * kx[0];
#pragma unroll
                for (int b = 1; b < 4; ++b) h = fmaf(v[j][b], kx[b], h);
                if constexpr (DOWN == 1) {
#pragma unroll
                  for (int a = 0; a < 4; ++a) acc[(u - a) & 3][j] = fmaf(h, ky[a], acc[(u - a) & 3][j]);
                } else {
                  acc[cur][j] = fmaf(h, ky[e], acc[cur][j]);
                  acc[prev][j] = fmaf(h, ky[e + 2], acc[prev][j]);
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < NC; ++j)
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                  if constexpr (DOWN == 1) {
#pragma unroll
                    for (int a = 0; a < 4; ++a)
                      acc[(u - a) & 3][j] = fmaf(v[j][b], kr[a * 4 + b], acc[(u - a) & 3][j]);
                  } else {
                    acc[cur][j] = fmaf(v[j][b], kr[e * 4 + b], acc[cur][j]);
                    acc[prev][j] = fmaf(v[j][b], kr[(e + 2) * 4 + b], acc[prev][j]);
                  }
                }
            }
          }
          // the output row that is complete once this input row has been added (row counts bound it by nrows)
          const int orow = DOWN == 1 ? r - 3 : (r >> 1) - 1;
          const int slot = DOWN == 1 ? (u + 1) & 3 : prev;
          if (DOWN == 1 || e == 1) {
            if (orow >= 0) {
#pragma unroll
              for (int j = 0; j < NC; ++j)
                if (live & (1u << j)) __stcs(dst_row + 256 * j, acc[slot][j]);
              dst_row += out_w;
            }
#pragma unroll
            for (int j = 0; j < NC; ++j) acc[slot][j] = 0.f;
          }
        }
      }
      __syncthreads();                                                 // every thread is done with stage s
      if (t == 0 && c + S < nchunks) issue_chunk(c + S);
    }
  };
  if (separable) run(std::true_type{});
  else run(std::false_type{});
}

// up = 2, down = 1, 4x4 taps, pad (2,1) (the RGB-skip Upsample) with the same TMA-fed strips: a thread owns the input
// columns t, t+256, ... and slides a 3-row x 3-column window; every input pixel yields a 2x2 output quad, stored as
// two 8-byte pairs (a warp writes 256 contiguous bytes per store).  Chunks are a multiple of 3 rows so that the
// window rotation is static.
template <int NC, int RS, int CR, int S>                      // RS INPUT rows per CTA
__global__ void __launch_bounds__(256) upfirdn2d_up2_k4_bulk_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                    const float* __restrict__ k, int in_h, int in_w,
                                                                    uint32_t stage_bytes) {
  static_assert(CR % 3 == 0, "chunk rows keep the window rotation static");
  extern __shared__ __align__(128) unsigned char bulk_smem[];
  __shared__ uint64_t full[S];
  const int t = threadIdx.x;
  const int y0 = blockIdx.y * RS;
  float kr[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kr[i] = __ldg(k + 15 - i);
  const size_t plane_off = (size_t)blockIdx.z * in_h * in_w;
  const int out_w = 2 * in_w;
  float* yp = y + (size_t)blockIdx.z * (2 * in_h) * out_w;
  const int nrows = min(RS, in_h - y0) + 2;                           // strip row r = input row y0 - 1 + r
  const int nchunks = (nrows + CR - 1) / CR;
  const int iy0 = y0 - 1;
  const uint32_t smem_s = smem_u32(bulk_smem);
  auto issue_chunk = [&](int c) {
    const BulkSpan sp = bulk_span(c, CR, iy0, nrows, in_h, in_w, plane_off);
    if (sp.lo >= sp.hi) return;
    const int s = c % S;
    mbar_expect_tx(&full[s], sp.bytes);
    bulk_load_1d(smem_s + (uint32_t)s * stage_bytes, reinterpret_cast<const unsigned char*>(x) + sp.a0, sp.bytes,
                 &full[s]);
  };
  if (t == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (t == 0)
    for (int c = 0; c < S && c < nchunks; ++c) issue_chunk(c);
  uint32_t off[NC];
  uint32_t edge = 0, live = 0;
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const int xx = t + 256 * j;
    const bool in_img = xx < in_w;
    const bool inside = xx >= 1 && xx + 1 < in_w;
    off[j] = (in_img && inside) ? (uint32_t)(xx - 1) * 4u : 0u;
    if (in_img) live |= 1u << j;
    if (in_img && !inside) edge |= 1u << j;
  }
  const bool any_edge = edge != 0;
  const uint32_t row_bytes = (uint32_t)in_w * 4u;
  float* dst_row = yp + (size_t)(2 * y0) * out_w + 2 * t;             // output rows are produced in order
  float win[3][NC][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < NC; ++j)
#pragma unroll
      for (int b = 0; b < 3; ++b) win[i][j][b] = 0.f;
#pragma unroll 1
  for (int c = 0; c < nchunks; ++c) {
    const BulkSpan sp = bulk_span(c, CR, iy0, nrows, in_h, in_w, plane_off);
    const int s = c % S;
    if (sp.lo < sp.hi) mbar_wait(&full[s], (uint32_t)(c / S) & 1u);
    uint32_t row_s = smem_s + (uint32_t)s * stage_bytes +
                     (uint32_t)(int32_t)((int64_t)((plane_off + (size_t)sp.lo * in_w) * 4 - sp.a0) +
                                         (int64_t)(iy0 + c * CR - sp.lo) * (int64_t)row_bytes);
#pragma unroll
    for (int u8 = 0; u8 < CR; ++u8, row_s += row_bytes) {
      const int r = c * CR + u8;
      if (r < nrows) {
        const int u = u8 % 3;                                          // strip row r lives in window slot r % 3 = u
        const int iy = iy0 + r;
        const bool row_ok = iy >= sp.lo && iy < sp.hi;
        if (row_ok) {
#pragma unroll
          for (int j = 0; j < NC; ++j)
#pragma unroll
            for (int b = 0; b < 3; ++b) win[u][j][b] = lds_f32(row_s + off[j] + 4u * b);
          if (any_edge) {
#pragma unroll
            for (int j = 0; j < NC; ++j)
              if (edge & (1u << j)) {
                const int ix = t + 256 * j - 1;
#pragma unroll
                for (int b = 0; b < 3; ++b)
                  win[u][j][b] = (ix + b >= 0 && ix + b < in_w) ? lds_f32(row_s + (uint32_t)(ix + b) * 4u) : 0.f;
              }
          }
        } else {
#pragma unroll
          for (int j = 0; j < NC; ++j)
#pragma unroll
            for (int b = 0; b < 3; ++b) win[u][j][b] = 0.f;
        }
        if (r >= 2) {                                                  // rows yy-1, yy, yy+1 = strip rows r-2, r-1, r
#pragma unroll
          for (int py = 0; py < 2; ++py) {
#pragma unroll
            for (int j = 0; j < NC; ++j) {
              float o[2];
#pragma unroll
              for (int px = 0; px < 2; ++px) {
                float sum = 0.f;
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                  for (int b = 0; b < 2; ++b)               // strip row r - 2 + py + a -> slot (u + 1 + py + a) % 3
                    sum = fmaf(win[(u + 1 + py + a) % 3][j][px + b], kr[(py + 2 * a) * 4 + px + 2 * b], sum);
                o[px] = sum;
              }
              if (live & (1u << j)) __stcs(reinterpret_cast<float2*>(dst_row + 512 * j), make_float2(o[0], o[1]));
            }
            dst_row += out_w;
          }
        }
      }
    }
    __syncthreads();
    if (t == 0 && c + S < nchunks) issue_chunk(c + S);
  }
}

// General path: any up/down/pad (incl. negative pads = crop) and any kernel size.
__global__ void __launch_bounds__(256) upfirdn2d_general_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                const float* __restrict__ k, int in_h, int in_w,
                                                                int out_h, int out_w, int kh, int kw, int up_x,
                                                                int up_y, int down_x, int down_y, int px0, int py0,
                                                                int64_t total) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int ox = (int)(idx % out_w);
    int64_t t = idx / out_w;
    int oy = (int)(t % out_h);
    int plane = (int)(t / out_h);
    const float* xp = x + (size_t)plane * in_h * in_w;
    float acc = 0.f;
    for (int ky = 0; ky < kh; ++ky) {
      int uy = oy * down_y + ky - py0;          // coordinate in the zero-stuffed image
      if (uy < 0 || uy % up_y != 0) continue;
      int iy = uy / up_y;
      if (iy >= in_h) continue;
      for (int kx = 0; kx < kw; ++kx) {
        int ux = ox * down_x + kx - px0;
        if (ux < 0 || ux % up_x != 0) continue;
        int ix = ux / up_x;
        if (ix >= in_w) continue;
        acc = fmaf(__ldg(xp + (size_t)iy * in_w + ix), __ldg(k + (kh - 1 - ky) * kw + (kw - 1 - kx)), acc);
      }
    }
    y[idx] = acc;
  }
}

// =============================================================================================
// fused bias + activation  (op/fused_bias_act_kernel.cu:19-49, forward, act in {1 linear, 3 lrelu})
// =============================================================================================
template <bool VEC>
__global__ void __launch_bounds__(256) bias_act_kernel(const float* __restrict__ x, const float* __restrict__ b,
                                                       float* __restrict__ y, int64_t n, int size_b,
                                                       int64_t step_b, int act, float alpha, float scale) {
  if (VEC) {
    const int64_t n4 = n >> 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
      float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
      // step_b % 4 == 0: one channel.  No bias adds -0, the identity of IEEE addition (+0 would turn -0 into +0)
      float bb = size_b ? __ldg(b + ((i * 4) / step_b) % size_b) : -0.f;
      float r[4] = {v.x + bb, v.y + bb, v.z + bb, v.w + bb};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float t = r[j];
        if (act == 3) t = (t > 0.f) ? t : t * alpha;
        r[j] = t * scale;
      }
      reinterpret_cast<float4*>(y)[i] = make_float4(r[0], r[1], r[2], r[3]);
    }
  } else {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      float t = x[i];
      if (size_b) t += __ldg(b + (i / step_b) % size_b);
      if (act == 3) t = (t > 0.f) ? t : t * alpha;
      y[i] = t * scale;
    }
  }
}

// Plane form of the vector path: blockIdx.y = (batch, channel) plane, so the bias index is computed once per CTA
// instead of two 64-bit divisions per float4 (measured: the flat form ran at about a third of the HBM rate).
__global__ void __launch_bounds__(256) bias_act_plane_kernel(const float* __restrict__ x, const float* __restrict__ b,
                                                             float* __restrict__ y, int quads_per_plane, int size_b,
                                                             int act, float alpha, float scale) {
  const int plane = blockIdx.y;
  const float bb = size_b ? __ldg(b + plane % size_b) : -0.f;        // -0: x + bb == x for every x, -0 included
  const float4* xp = reinterpret_cast<const float4*>(x) + (size_t)plane * quads_per_plane;
  float4* yp = reinterpret_cast<float4*>(y) + (size_t)plane * quads_per_plane;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < quads_per_plane; i += gridDim.x * blockDim.x) {
    const float4 v = __ldg(xp + i);
    float r[4] = {v.x + bb, v.y + bb, v.z + bb, v.w + bb};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = r[j];
      if (act == 3) t = (t > 0.f) ? t : t * alpha;
      r[j] = t * scale;
    }
    yp[i] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// =============================================================================================
// style affine (EqualLinear modulation, model.py:153-163 with bias_init=1) and demodulation table
// =============================================================================================
struct AffineJobs { AffineJob j[kMaxJobs]; int n; };
struct DemodJobs { DemodJob j[kMaxJobs]; int n; };

// One warp per output row i of one job; lanes split the D-long dot product (float4 loads).
__global__ void __launch_bounds__(256) affine_kernel(const __grid_constant__ AffineJobs jobs, int B, int D,
                                                     int64_t style_stride) {
  int jb = 0;
  while (jb + 1 < jobs.n && (int)blockIdx.x >= jobs.j[jb + 1].block_begin) ++jb;
  const AffineJob& job = jobs.j[jb];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = ((int)blockIdx.x - job.block_begin) * 8 + warp;
  if (i >= job.C) return;
  const float* wrow = job.mw + (size_t)i * D;
  const float mb = __ldg(job.mb + i);
  if (D == 512) {
    // the usual case (style_dim 512): the weight row lives in registers, four samples in flight per pass
    float4 w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) w[q] = __ldg(reinterpret_cast<const float4*>(wrow + lane * 4 + q * 128));
    for (int b0 = 0; b0 < B; b0 += 4) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int b = min(b0 + u, B - 1);
        const float* srow = job.style + (size_t)b * style_stride;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 s = __ldg(reinterpret_cast<const float4*>(srow + lane * 4 + q * 128));
          acc[u] = fmaf(w[q].x, s.x, acc[u]); acc[u] = fmaf(w[q].y, s.y, acc[u]);
          acc[u] = fmaf(w[q].z, s.z, acc[u]); acc[u] = fmaf(w[q].w, s.w, acc[u]);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], o);
      }
      if (lane < 4 && b0 + lane < B) {
        const float a = lane == 0 ? acc[0] : (lane == 1 ? acc[1] : (lane == 2 ? acc[2] : acc[3]));
        job.s[(size_t)(b0 + lane) * job.C + i] = fmaf(a, job.wscale, mb);
      }
    }
    return;
  }
  for (int b = 0; b < B; ++b) {
    const float* srow = job.style + (size_t)b * style_stride;
    float acc = 0.f;
    for (int j = lane * 4; j < D; j += 128) {
      float4 w = __ldg(reinterpret_cast<const float4*>(wrow + j));
      float4 s = __ldg(reinterpret_cast<const float4*>(srow + j));
      acc = fmaf(w.x, s.x, acc); acc = fmaf(w.y, s.y, acc); acc = fmaf(w.z, s.z, acc); acc = fmaf(w.w, s.w, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) job.s[(size_t)b * job.C + i] = fmaf(acc, job.wscale, mb);
  }
}

__global__ void __launch_bounds__(256) demod_kernel(const __grid_constant__ DemodJobs jobs, int B) {
  int jb = 0;
  while (jb + 1 < jobs.n && (int)blockIdx.x >= jobs.j[jb + 1].block_begin) ++jb;
  const DemodJob& job = jobs.j[jb];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = ((int)blockIdx.x - job.block_begin) * 8 + warp;
  if (o >= job.Cout) return;
  const float* wrow = job.wsq + (size_t)o * job.Cin;
  if (job.Cin <= 512) {
    // Wsq row in registers (<= 16 values per lane), four samples in flight per pass; same summation order as below
    float w[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) w[q] = (lane + 32 * q < job.Cin) ? __ldg(wrow + lane + 32 * q) : 0.f;
    for (int b0 = 0; b0 < B; b0 += 4) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float* srow = job.s + (size_t)min(b0 + u, B - 1) * job.Cin;
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          if (lane + 32 * q < job.Cin) {
            const float s = __ldg(srow + lane + 32 * q);
            acc[u] = fmaf(s * s, w[q], acc[u]);
          }
        }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], off);
      }
      if (lane < 4 && b0 + lane < B) {
        const float a = lane == 0 ? acc[0] : (lane == 1 ? acc[1] : (lane == 2 ? acc[2] : acc[3]));
        job.d[(size_t)(b0 + lane) * job.Cout + o] = rsqrtf(a + 1e-8f);
      }
    }
    return;
  }
  for (int b = 0; b < B; ++b) {
    const float* srow = job.s + (size_t)b * job.Cin;
    float acc = 0.f;
    for (int i = lane; i < job.Cin; i += 32) {
      float s = __ldg(srow + i);
      acc = fmaf(s * s, __ldg(wrow + i), acc);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) job.d[(size_t)b * job.Cout + o] = rsqrtf(acc + 1e-8f);
  }
}

int launch_affine(AffineJob* jobs, int njobs, int B, int D, int64_t style_stride, cudaStream_t st) {
  HF_REQUIRE(njobs > 0 && njobs <= kMaxJobs, "affine: bad job count %d", njobs);
  HF_REQUIRE(D % 4 == 0 && style_stride % 4 == 0, "affine: style_dim and stride must be multiples of 4");
  AffineJobs aj;
  aj.n = njobs;
  int blocks = 0;
  for (int i = 0; i < njobs; ++i) {
    jobs[i].block_begin = blocks;
    blocks += cdiv(jobs[i].C, 8);
    aj.j[i] = jobs[i];
  }
  affine_kernel<<<blocks, 256, 0, st>>>(aj, B, D, style_stride);
  HF_LAUNCH_OK("affine");
  count_launch();
  return HF_OK;
}

int launch_demod(DemodJob* jobs, int njobs, int B, cudaStream_t st) {
  HF_REQUIRE(njobs > 0 && njobs <= kMaxJobs, "demod: bad job count %d", njobs);
  DemodJobs dj;
  dj.n = njobs;
  int blocks = 0;
  for (int i = 0; i < njobs; ++i) {
    jobs[i].block_begin = blocks;
    blocks += cdiv(jobs[i].Cout, 8);
    dj.j[i] = jobs[i];
  }
  demod_kernel<<<blocks, 256, 0, st>>>(dj, B);
  HF_LAUNCH_OK("demod");
  count_launch();
  return HF_OK;
}

// =============================================================================================
// pre-pass: NCHW fp32 -> NHWC 16-bit with the per-(b,cin) style scale folded in
// (the "x * s" of y = d * conv(x*s, W~), SURVEY Appendix C-1); optional FSE feature blend.
// =============================================================================================
template <int DT>
__global__ void __launch_bounds__(256) modulate_to_nhwc_kernel(const float* __restrict__ x, int64_t x_bstride,
                                                               const float* __restrict__ s,
                                                               const float* __restrict__ feat, float alpha,
                                                               uint16_t* __restrict__ xh, int C, int HW) {
  __shared__ float tile[64][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 64, p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* xb = x + (size_t)b * x_bstride;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int c = c0 + ty + 8 * k, p = p0 + tx;
    float v = 0.f;
    if (c < C && p < HW) {
      v = __ldg(xb + (size_t)c * HW + p);
      if (feat) v = (1.f - alpha) * v + alpha * __ldg(feat + ((size_t)b * C + c) * HW + p);
      v *= __ldg(s + (size_t)b * C + c);
    }
    tile[ty + 8 * k][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int p = p0 + ty + 8 * k, c = c0 + 2 * tx;
    if (p < HW && c < C) {
      uint32_t packed = Half2T<DT>::pack(tile[2 * tx][ty + 8 * k], tile[2 * tx + 1][ty + 8 * k]);
      *reinterpret_cast<uint32_t*>(xh + ((size_t)b * HW + p) * C + c) = packed;
    }
  }
}

int launch_modulate_to_nhwc(const float* x, int x_broadcast, const float* s, const float* feat, float alpha,
                            void* xh, int B, int C, int HW, int dtype, cudaStream_t st) {
  HF_REQUIRE(x && s && xh, "modulate_to_nhwc: null pointer");
  HF_REQUIRE(C % 2 == 0, "modulate_to_nhwc: C must be even");
  dim3 grid(cdiv(HW, 32), cdiv(C, 64), B);
  int64_t bstride = x_broadcast ? 0 : (int64_t)C * HW;
  return with_dtype(dtype, "modulate_to_nhwc", [&](auto dt) -> int {
    modulate_to_nhwc_kernel<dt><<<grid, 256, 0, st>>>(x, bstride, s, feat, alpha, (uint16_t*)xh, C, HW);
    HF_LAUNCH_OK("modulate_to_nhwc");
    count_launch();
    return HF_OK;
  });
}

// =============================================================================================
// RGB combine: bias + ordered sum of the per-N-tile ToRGB partials + Upsample(skip)
// (ToRGB.forward model.py:356-365; Upsample = upfirdn2d(up=2, pad=(2,1)), model.py:35-53)
// =============================================================================================
__global__ void __launch_bounds__(256) rgb_combine_kernel(const float* partial, int num_partials,
                                                          int64_t partial_stride, const float* __restrict__ bias,
                                                          const float* __restrict__ skip,
                                                          const float* __restrict__ upk, float* rgb,
                                                          int H, int W, int64_t total) {
  __shared__ float kf[16];
  if (threadIdx.x < 16) kf[threadIdx.x] = upk ? upk[15 - threadIdx.x] : 0.f;
  __syncthreads();
  const int h2 = H >> 1, w2 = W >> 1;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int X = (int)(idx % W);
    int64_t t = idx / W;
    int Y = (int)(t % H);
    int plane = (int)(t / H);            // b*3 + j
    float acc = bias ? __ldg(bias + plane % 3) : 0.f;
    for (int q = 0; q < num_partials; ++q) acc += partial[q * partial_stride + idx];   // may alias rgb (in place)
    if (skip) {
      const float* sp = skip + (size_t)plane * h2 * w2;
      const int ky0 = Y & 1, kx0 = X & 1;      // pad0 = 2: Y + ky - 2 even
      float up = 0.f;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        int ky = ky0 + 2 * a;
        int uy = Y + ky - 2;
        int iy = uy >> 1;
        if (uy < 0 || iy >= h2) continue;
#pragma unroll
        for (int bq = 0; bq < 2; ++bq) {
          int kx = kx0 + 2 * bq;
          int ux = X + kx - 2;
          int ix = ux >> 1;
          if (ux >= 0 && ix < w2) up = fmaf(__ldg(sp + (size_t)iy * w2 + ix), kf[ky * 4 + kx], up);
        }
      }
      acc += up;
    }
    rgb[idx] = acc;
  }
}

// W % 4 == 0: four consecutive outputs per thread, float4 partial loads / stores; the 2x2-tap up-FIR of the
// skip reads a 2x4 window of the half-resolution image (columns 2q-1 .. 2q+2 for outputs 4q .. 4q+3).
__global__ void __launch_bounds__(256) rgb_combine_vec4_kernel(const float* partial, int num_partials,
                                                               int64_t partial_stride,
                                                               const float* __restrict__ bias,
                                                               const float* __restrict__ skip,
                                                               const float* __restrict__ upk, float* rgb, int H, int W,
                                                               int64_t total4) {
  __shared__ float kf[16];
  if (threadIdx.x < 16) kf[threadIdx.x] = upk ? upk[15 - threadIdx.x] : 0.f;
  __syncthreads();
  const int h2 = H >> 1, w2 = W >> 1, wq = W >> 2;
  // 32-bit index math (the launcher checks total4 < 2^31): a 64-bit div/mod costs ~100 instructions
  for (int i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < (int)total4; i4 += gridDim.x * blockDim.x) {
    const int q = i4 % wq;
    const int t = i4 / wq;
    const int Y = t % H;
    const int plane = t / H;
    const float bv = bias ? __ldg(bias + plane % 3) : 0.f;
    float acc[4] = {bv, bv, bv, bv};
    for (int s = 0; s < num_partials; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(partial + s * partial_stride + (size_t)i4 * 4);   // may alias rgb
      acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
    }
    if (skip) {
      const float* sp = skip + (size_t)plane * h2 * w2;
      const int ky0 = Y & 1;
      float up[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int ky = ky0 + 2 * a;
        const int uy = Y + ky - 2;
        const int iy = uy >> 1;
        if (uy < 0 || iy >= h2) continue;
        const float* row = sp + (size_t)iy * w2;
        float c[4];                                      // columns 2q-1 .. 2q+2
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int ix = 2 * q - 1 + m;
          c[m] = (ix >= 0 && ix < w2) ? __ldg(row + ix) : 0.f;
        }
        // even X (4q, 4q+2): taps kx 0,2 on columns (X/2-1, X/2); odd X: taps kx 1,3 on ((X-1)/2, (X+1)/2)
        up[0] = fmaf(c[0], kf[ky * 4 + 0], fmaf(c[1], kf[ky * 4 + 2], up[0]));
        up[1] = fmaf(c[1], kf[ky * 4 + 1], fmaf(c[2], kf[ky * 4 + 3], up[1]));
        up[2] = fmaf(c[1], kf[ky * 4 + 0], fmaf(c[2], kf[ky * 4 + 2], up[2]));
        up[3] = fmaf(c[2], kf[ky * 4 + 1], fmaf(c[3], kf[ky * 4 + 3], up[3]));
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += up[j];
    }
    *reinterpret_cast<float4*>(rgb + (size_t)i4 * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}

int launch_rgb_combine(const float* partial, int num_partials, const float* bias, const float* skip,
                       const float* up_kernel, float* rgb, int B, int H, int W, cudaStream_t st) {
  HF_REQUIRE(rgb && (partial || num_partials == 0), "rgb_combine: null pointer");
  HF_REQUIRE(!skip || up_kernel, "rgb_combine: skip given without an upsample kernel");
  int64_t total = (int64_t)B * 3 * H * W;
  if (W % 4 == 0 && ((((uintptr_t)partial | (uintptr_t)rgb) & 15) == 0) && total / 4 < (int64_t)2000000000) {
    int64_t total4 = total / 4;
    rgb_combine_vec4_kernel<<<grid_for(total4), 256, 0, st>>>(partial, num_partials, total, bias, skip, up_kernel,
                                                              rgb, H, W, total4);
    HF_LAUNCH_OK("rgb_combine");
    count_launch();
    return HF_OK;
  }
  rgb_combine_kernel<<<grid_for(total), 256, 0, st>>>(partial, num_partials, total, bias, skip, up_kernel, rgb, H, W,
                                                      total);
  HF_LAUNCH_OK("rgb_combine");
  count_launch();
  return HF_OK;
}

// =============================================================================================
// standalone ToRGB on an fp32 NCHW feature map (module-level API): one pass over x
// =============================================================================================
__global__ void __launch_bounds__(256) torgb_nchw_kernel(const float* __restrict__ x, const float* __restrict__ w1,
                                                         float w_scale, const float* __restrict__ s,
                                                         float* __restrict__ part, int C, int HW) {
  extern __shared__ float ws[];      // [3][C] = w1[j,i] * scale * s[b,i]
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 3 * C; i += 256) {
    int c = i % C;
    ws[i] = __ldg(w1 + i) * w_scale * __ldg(s + (size_t)b * C + c);
  }
  __syncthreads();
  const float* xb = x + (size_t)b * C * HW;
  for (int p = blockIdx.x * 256 + threadIdx.x; p < HW; p += gridDim.x * 256) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll 4
    for (int c = 0; c < C; ++c) {
      float v = __ldg(xb + (size_t)c * HW + p);
      a0 = fmaf(v, ws[c], a0);
      a1 = fmaf(v, ws[C + c], a1);
      a2 = fmaf(v, ws[2 * C + c], a2);
    }
    float* pb = part + (size_t)b * 3 * HW;
    pb[p] = a0; pb[HW + p] = a1; pb[2 * (size_t)HW + p] = a2;
  }
}

int launch_torgb_nchw(const float* x, const float* w1, float w_scale, const float* s, const float* bias,
                      const float* skip, const float* up_kernel, float* y, int B, int C, int H, int W,
                      cudaStream_t st) {
  HF_REQUIRE(x && w1 && s && y, "torgb: null pointer");
  HF_REQUIRE(3 * C * sizeof(float) <= 48 * 1024, "torgb: too many channels (%d)", C);
  const int HW = H * W;
  dim3 grid(std::min(cdiv(HW, 256), num_sms() * 4), B);
  // y doubles as the partial buffer; rgb_combine then adds bias + upsampled skip in place.
  torgb_nchw_kernel<<<grid, 256, 3 * C * sizeof(float), st>>>(x, w1, w_scale, s, y, C, HW);
  HF_LAUNCH_OK("torgb_nchw");
  count_launch();
  return launch_rgb_combine(y, 1, bias, skip, up_kernel, y, B, H, W, st);
}

// =============================================================================================
// weight packing (once per weight load)
// =============================================================================================
// plain: wpk[o][tap*Cin + c] = W[o,c,dy,dx] * scale (tap = dy*3+dx, correlation form of F.conv2d)
// up   : the stride-2 transposed conv (model.py:260) composed with the 4x4 blur (pad (1,1), model.py:263)
//        as four 3x3 correlations, one per output parity (py,px); N row = (o/32)*128 + (py*2+px)*32 + o%32
//        Kp[py,px][dy,dx] = sum_{a,b} W[a,b] * blur[2-a+u, 2-b+v],  u = py+2-2dy, v = px+2-2dx
template <int DT>
__global__ void __launch_bounds__(256) pack_conv_kernel(const float* __restrict__ w, const float* __restrict__ blur,
                                                        uint16_t* __restrict__ wpk, float* __restrict__ wsq,
                                                        int Cout, int Cin, int ksize, int up, float scale) {
  const int taps = ksize * ksize;
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= (int64_t)Cout * Cin) return;
  const int c = (int)(idx % Cin), o = (int)(idx / Cin);
  float wv[9];
  float sq = 0.f;
  for (int t = 0; t < taps; ++t) {
    wv[t] = w[((size_t)o * Cin + c) * taps + t] * scale;
    sq = fmaf(wv[t], wv[t], sq);
  }
  if (wsq) wsq[idx] = sq;
  const size_t K = (size_t)taps * Cin;
  if (!up) {
    for (int t = 0; t < taps; ++t) wpk[(size_t)o * K + (size_t)t * Cin + c] = Half2T<DT>::one(wv[t]);
  } else {
    float bk[16];
    for (int i = 0; i < 16; ++i) bk[i] = blur[i];
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const size_t row = (size_t)(o / 32) * 128 + (size_t)(py * 2 + px) * 32 + (o % 32);
        for (int dy = 0; dy < 3; ++dy)
          for (int dx = 0; dx < 3; ++dx) {
            const int u = py + 2 - 2 * dy, v = px + 2 - 2 * dx;
            float acc = 0.f;
            for (int a = 0; a < 3; ++a)
              for (int b = 0; b < 3; ++b) {
                int iy = 2 - a + u, ix = 2 - b + v;
                if (iy >= 0 && iy < 4 && ix >= 0 && ix < 4) acc = fmaf(wv[a * 3 + b], bk[iy * 4 + ix], acc);
              }
            wpk[row * K + (size_t)(dy * 3 + dx) * Cin + c] = Half2T<DT>::one(acc);
          }
      }
  }
}

int launch_pack_conv(const float* w, const float* blur, void* wpk, float* wsq, int Cout, int Cin, int ksize,
                     int up, int nc, int dtype, cudaStream_t st) {
  (void)nc;
  HF_REQUIRE(w && wpk, "pack_conv: null pointer");
  HF_REQUIRE(ksize == 3 || ksize == 1, "pack_conv: kernel size %d unsupported", ksize);
  HF_REQUIRE(!up || (ksize == 3 && blur && Cout % 32 == 0), "pack_conv: upsample needs 3x3, blur kernel, Cout%%32==0");
  const float scale = 1.0f / sqrtf((float)(Cin * ksize * ksize));
  int64_t total = (int64_t)Cout * Cin;
  int grid = cdiv(total, 256);
  return with_dtype(dtype, "pack_conv", [&](auto dt) -> int {
    pack_conv_kernel<dt><<<grid, 256, 0, st>>>(w, blur, (uint16_t*)wpk, wsq, Cout, Cin, ksize, up, scale);
    HF_LAUNCH_OK("pack_conv");
    count_launch();
    return HF_OK;
  });
}

__global__ void scale_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t n, float scale) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = src[i] * scale;
}
int launch_scale_copy(const float* src, float* dst, int64_t n, float scale, cudaStream_t st) {
  HF_REQUIRE(src && dst, "scale_copy: null pointer");
  if (n == 0) return HF_OK;
  int grid = (int)std::min<int64_t>((n + 255) / 256, 4096);
  scale_copy_kernel<<<grid, 256, 0, st>>>(src, dst, n, scale);
  HF_LAUNCH_OK("scale_copy");
  count_launch();
  return HF_OK;
}

}  // namespace hf

using namespace hf;

extern "C" {

int hf_upfirdn2d_f32(const float* x, float* y, const float* k, int planes, int in_h, int in_w, int kh, int kw,
                     int up_x, int up_y, int down_x, int down_y, int px0, int px1, int py0, int py1, void* stream) {
  reset_launch_count();
  if (planes == 0) return HF_OK;
  HF_REQUIRE(x && y && k, "upfirdn2d: null pointer");
  HF_REQUIRE(planes >= 0 && in_h > 0 && in_w > 0 && kh > 0 && kw > 0, "upfirdn2d: bad shape");
  HF_REQUIRE(up_x > 0 && up_y > 0 && down_x > 0 && down_y > 0, "upfirdn2d: up/down must be positive");
  const int out_h = (in_h * up_y + py0 + py1 - kh) / down_y + 1;
  const int out_w = (in_w * up_x + px0 + px1 - kw) / down_x + 1;
  HF_REQUIRE(in_h * up_y + py0 + py1 - kh >= 0 && in_w * up_x + px0 + px1 - kw >= 0,
             "upfirdn2d: output would be empty (in %dx%d up %d pad %d,%d k %d)", in_h, in_w, up_y, py0, py1, kh);
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const bool k4 = (kh == 4 && kw == 4);
  const bool sym = (up_x == up_y && down_x == down_y);
  const bool pads03 = px0 >= 0 && py0 >= 0 && px1 >= 0 && py1 >= 0 && px0 <= 3 && px1 <= 3 && py0 <= 3 && py1 <= 3;
  // TMA-fed strip kernels (see upfirdn2d_k4_bulk_kernel): full-width rows, 16-byte aligned tensor, pads 0..3
  const bool bulk_ok = k4 && sym && planes <= 65535 && in_w >= 64 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                       ((size_t)planes * in_h * in_w) % 4 == 0;
  auto bulk_stage = [&](int CR) {
    return (uint32_t)((((size_t)CR * in_w * 4 + 15) / 16 * 16 + 32 + 127) / 128 * 128);
  };
  auto bulk_go = [&](auto kern, int rows_per_cta, int CR, int S, auto... tail) {
    const uint32_t stage = bulk_stage(CR);                 // <= 25 KB for the widths admitted below
    // per launch like the convolution kernels: the attribute is per device, a cache would have to be too
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    dim3 grid(1, cdiv(up_x == 2 ? in_h : out_h, rows_per_cta), planes);
    kern<<<grid, 256, S * stage, st>>>(x, y, k, in_h, in_w, tail..., stage);
  };
  if (bulk_ok && up_x == 1 && down_x == 1 && pads03 && out_w <= 1024 && in_w <= 1040) {
    if (out_w <= 512) bulk_go(upfirdn2d_k4_bulk_kernel<1, 2, 64, 4, 3>, 64, 4, 3, out_h, out_w, px0, py0);
    else bulk_go(upfirdn2d_k4_bulk_kernel<1, 4, 64, 4, 3>, 64, 4, 3, out_h, out_w, px0, py0);
  } else if (bulk_ok && up_x == 1 && down_x == 2 && pads03 && out_w <= 1024 && in_w <= 1040) {
    if (out_w <= 512) bulk_go(upfirdn2d_k4_bulk_kernel<2, 2, 32, 4, 3>, 32, 4, 3, out_h, out_w, px0, py0);
    else bulk_go(upfirdn2d_k4_bulk_kernel<2, 4, 32, 4, 3>, 32, 4, 3, out_h, out_w, px0, py0);
  } else if (bulk_ok && up_x == 2 && down_x == 1 && px0 == 2 && py0 == 2 && px1 == 1 && py1 == 1 && in_w <= 1024 &&
             (reinterpret_cast<uintptr_t>(y) & 7) == 0) {
    if (in_w <= 512) bulk_go(upfirdn2d_up2_k4_bulk_kernel<2, 32, 6, 3>, 32, 6, 3);
    else bulk_go(upfirdn2d_up2_k4_bulk_kernel<4, 32, 6, 3>, 32, 6, 3);
  } else {
    int64_t total = (int64_t)planes * out_h * out_w;
    upfirdn2d_general_kernel<<<grid_for(total), 256, 0, st>>>(x, y, k, in_h, in_w, out_h, out_w, kh, kw, up_x, up_y,
                                                              down_x, down_y, px0, py0, total);
  }
  HF_LAUNCH_OK("upfirdn2d");
  count_launch();
  return HF_OK;
}

int hf_bias_act_f32(const float* x, const float* b, float* y, int64_t n, int size_b, int64_t step_b, int act,
                    float alpha, float scale, void* stream) {
  reset_launch_count();
  if (n == 0) return HF_OK;
  HF_REQUIRE(x && y, "bias_act: null pointer");
  HF_REQUIRE(act == 1 || act == 3, "bias_act: act must be 1 (linear) or 3 (leaky relu), got %d", act);
  HF_REQUIRE(n >= 0 && size_b >= 0 && step_b >= 1, "bias_act: bad sizes");
  HF_REQUIRE(size_b == 0 || b, "bias_act: bias pointer is null");
  int rc = ensure_device_current();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (step_b % 4 == 0 && step_b >= 1024 && n % step_b == 0 && n / step_b <= 65535 &&
      step_b / 4 < (int64_t)2000000000 && ((((uintptr_t)x | (uintptr_t)y) & 15) == 0)) {
    const int planes = (int)(n / step_b), quads = (int)(step_b / 4);
    const int gx = std::max(1, std::min(cdiv(quads, 256), std::max(1, num_sms() * 16 / planes)));
    bias_act_plane_kernel<<<dim3(gx, planes), 256, 0, st>>>(x, b, y, quads, size_b, act, alpha, scale);
    HF_LAUNCH_OK("bias_act");
    count_launch();
    return HF_OK;
  }
  const bool vec = (step_b % 4 == 0) && (n % 4 == 0) && ((((uintptr_t)x | (uintptr_t)y) & 15) == 0);
  const int grid = grid_for(vec ? n / 4 : n);
  if (vec)
    bias_act_kernel<true><<<grid, 256, 0, st>>>(x, b, y, n, size_b, step_b, act, alpha, scale);
  else
    bias_act_kernel<false><<<grid, 256, 0, st>>>(x, b, y, n, size_b, step_b, act, alpha, scale);
  HF_LAUNCH_OK("bias_act");
  count_launch();
  return HF_OK;
}

}  // extern "C"
