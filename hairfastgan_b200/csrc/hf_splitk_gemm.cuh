// The split-K "skinny" GEMM that streams compact 16-bit weights (mma.sync m16n8k16, fp32 accumulation) and its
// fixed-order reduction.  Shared by CtrlHair's shape adaptor (hf_shape.cu) and HairFast's modulation stacks
// (hf_modulation.cu).  Partials are summed in split order, no atomics: results are deterministic.
#pragma once
#include <algorithm>

#include "hf_kernels.cuh"

namespace hf {
namespace {

// ------------------------------------------------------------------------------------------------
// part[s][g][p][co] = sum_{k in split s} W_g[co][k] * A_g[p][k] for G groups of equal shape, with compact 16-bit
// weights W_g = w + g * w_gs, [Cout][K] (k = tap * Cin + c, taps in the reference's ky, kx order) and the im2col A_g
// gathered on the fly from the small 16-bit NHWC input x + g * x_gs:
//   MODE 0  1x1 / Linear:                  A[p][k] = x[p * ldx + k]
//   MODE 1  ZeroPad 1 + Conv 4x4 stride 2: source (2 oy - 1 + ky, 2 ox - 1 + kx) of an Hi x Wi input
//   MODE 2  nearest 2x up + Conv 3x3 pad 1: upsampled (oy - 1 + ky, ox - 1 + kx) of a 2Hi x 2Wi grid = source >> 1
// CTA tile 128 couts x BN pixels x 64 k, 4 warps (32 couts each), 4-stage cp.async ring (zero fill outside the image
// and beyond K), XOR-swizzled 128-byte shared-memory rows.  blockIdx.z = g * splits + s.
// ------------------------------------------------------------------------------------------------
constexpr int kGemmBM = 128, kGemmBK = 64, kGemmStages = 4, kGemmThreads = 128, kGemmMinKt = 4;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t& r0, uint32_t& r1, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
// element (row, k) of a [rows][64] tile: 16-byte chunk k / 8 XOR row % 8
__device__ __forceinline__ int swz(int row, int chunk) { return row * kGemmBK + ((chunk ^ (row & 7)) << 3); }

template <int MODE>
__device__ __forceinline__ const uint16_t* gather(const uint16_t* x, int p, int k, int Cin, int ldx, int Hi, int Wi,
                                                  int Wo) {
  if (MODE == 0) return x + (size_t)p * ldx + k;
  const int tap = k / Cin, c = k - tap * Cin, oy = p / Wo, ox = p - oy * Wo;
  int iy, ix;
  if (MODE == 1) {
    iy = 2 * oy - 1 + (tap >> 2);
    ix = 2 * ox - 1 + (tap & 3);
  } else {
    const int uy = oy - 1 + tap / 3, ux = ox - 1 + tap % 3;
    if (uy < 0 || ux < 0 || uy >= 2 * Hi || ux >= 2 * Wi) return nullptr;
    iy = uy >> 1;
    ix = ux >> 1;
  }
  if (iy < 0 || ix < 0 || iy >= Hi || ix >= Wi) return nullptr;
  return x + ((size_t)iy * Wi + ix) * Cin + c;
}

template <int DT, int BN, int MODE>
__global__ void __launch_bounds__(kGemmThreads) shape_gemm_kernel(const uint16_t* __restrict__ w,
                                                                  const uint16_t* __restrict__ x,
                                                                  float* __restrict__ part, int Cout, int K, int P,
                                                                  int Cin, int Hi, int Wi, int Wo, int kt_total,
                                                                  int G, int64_t w_gs, int64_t x_gs, int ldx) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint16_t* sA = reinterpret_cast<uint16_t*>(smem_raw);
  uint16_t* sB = sA + kGemmStages * kGemmBM * kGemmBK;
  const int S = gridDim.z / G, g = blockIdx.z / S, s = blockIdx.z - g * S;
  const int m0 = blockIdx.x * kGemmBM, n0 = blockIdx.y * BN;
  const int kt0 = (int)((int64_t)kt_total * s / S), nkt = (int)((int64_t)kt_total * (s + 1) / S) - kt0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  w += g * w_gs;
  x += g * x_gs;

  auto load = [&](int stage, int kt) {
    const int kb = (kt0 + kt) * kGemmBK;
    uint16_t* a = sA + stage * kGemmBM * kGemmBK;
    uint16_t* b = sB + stage * BN * kGemmBK;
#pragma unroll
    for (int i = tid; i < kGemmBM * 8; i += kGemmThreads) {
      const int row = i >> 3, ch = i & 7, k = kb + ch * 8;
      const bool ok = m0 + row < Cout && k < K;
      cp_async16(smem_u32(a + swz(row, ch)), ok ? w + (size_t)(m0 + row) * K + k : w, ok ? 16 : 0);
    }
    for (int i = tid; i < BN * 8; i += kGemmThreads) {
      const int row = i >> 3, ch = i & 7, k = kb + ch * 8, p = n0 + row;
      const uint16_t* src = (p < P && k < K) ? gather<MODE>(x, p, k, Cin, ldx, Hi, Wi, Wo) : nullptr;
      cp_async16(smem_u32(b + swz(row, ch)), src ? src : x, src ? 16 : 0);
    }
  };

  float acc[2][BN / 8][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
  for (int st = 0; st < kGemmStages - 1; ++st) {
    if (st < nkt) load(st, st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int kt = 0; kt < nkt; ++kt) {
    asm volatile("cp.async.wait_group %0;" ::"n"(kGemmStages - 2) : "memory");
    __syncthreads();
    if (kt + kGemmStages - 1 < nkt) load((kt + kGemmStages - 1) % kGemmStages, kt + kGemmStages - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const uint16_t* a = sA + (kt % kGemmStages) * kGemmBM * kGemmBK;
    const uint16_t* b = sB + (kt % kGemmStages) * BN * kGemmBK;
#pragma unroll
    for (int kk = 0; kk < kGemmBK / 16; ++kk) {
      uint32_t af[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int row = warp * 32 + mi * 16 + (lane & 15);
        ldsm_x4(af[mi], smem_u32(a + swz(row, kk * 2 + (lane >> 4))));
      }
      if (BN == 8) {
        uint32_t b0, b1;
        const int row = lane & 7;
        ldsm_x2(b0, b1, smem_u32(b + swz(row, kk * 2 + ((lane >> 3) & 1))));
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) mma16816<DT>(acc[mi][0], af[mi], b0, b1);
      } else {
#pragma unroll
        for (int nj = 0; nj < BN / 16; ++nj) {
          uint32_t bf[4];
          const int row = nj * 16 + (lane & 7) + ((lane >> 4) << 3);
          ldsm_x4(bf, smem_u32(b + swz(row, kk * 2 + ((lane >> 3) & 1))));
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) {
            mma16816<DT>(acc[mi][2 * nj], af[mi], bf[0], bf[1]);
            mma16816<DT>(acc[mi][2 * nj + 1], af[mi], bf[2], bf[3]);
          }
        }
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");

  float* out = part + (size_t)(s * G + g) * P * Cout;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < BN / 8; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int co = m0 + warp * 32 + mi * 16 + (lane >> 2) + (q >> 1) * 8;
        const int p = n0 + ni * 8 + (lane & 3) * 2 + (q & 1);
        if (co < Cout && p < P) out[(size_t)p * Cout + co] = acc[mi][ni][q];
      }
}

// y[g][p][co] = bias[g][co] + sum_s part[s][g][p][co], s in order (n = G * P * Cout, pc = P * Cout); fp32 and / or
// 16-bit copies
template <int DT>
__global__ void __launch_bounds__(256) shape_splitk_reduce_kernel(const float* __restrict__ part, int S, int64_t n,
                                                                  int Cout, int64_t pc, const float* __restrict__ bias,
                                                                  float* __restrict__ y32, uint16_t* __restrict__ y16) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = bias ? __ldg(bias + i / pc * Cout + i % Cout) : 0.f;
    for (int s = 0; s < S; ++s) v += __ldg(part + (size_t)s * n + i);
    if (y32) y32[i] = v;
    if (y16) y16[i] = Half2T<DT>::one(v);
  }
}

struct GemmShape {
  int P, K, Hi, Wi, Wo;
};

// {BN, splits, k tiles, grid m, grid n}: enough splits over all groups for two CTAs per SM, at least kGemmMinKt k
// tiles per split
inline void gemm_plan(const GemmShape& g, int cout, int sms, int* out, int groups = 1) {
  const int bn = g.P <= 8 ? 8 : 64;
  const int gm = cdiv(cout, kGemmBM), gn = cdiv(g.P, bn), kt = cdiv(g.K, kGemmBK);
  const int splits = std::max(1, std::min(cdiv(2 * sms, groups * gm * gn), kt / kGemmMinKt));
  out[0] = bn; out[1] = splits; out[2] = kt; out[3] = gm; out[4] = gn;
}

// Group g reads w + g * w_gs and x + g * x_gs and writes part[s][g]; ldx is MODE 0's input row stride.
template <int DT, int BN, int MODE>
int launch_gemm(const uint16_t* w, const uint16_t* x, float* part, int cout, const GemmShape& g, const int* pl,
                int cin, cudaStream_t st, int groups = 1, int64_t w_gs = 0, int64_t x_gs = 0, int ldx = -1) {
  constexpr int smem = kGemmStages * (kGemmBM + BN) * kGemmBK * 2;
  static uint64_t attr_set = 0;          // per device: the opt-in above 48 KB of dynamic shared memory
  int dev = 0;
  HF_CUDA_OK(cudaGetDevice(&dev));
  if (!(attr_set >> (dev & 63) & 1)) {
    HF_CUDA_OK(cudaFuncSetAttribute(shape_gemm_kernel<DT, BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set |= 1ull << (dev & 63);
  }
  shape_gemm_kernel<DT, BN, MODE><<<dim3(pl[3], pl[4], pl[1] * groups), kGemmThreads, smem, st>>>(
      w, x, part, cout, g.K, g.P, cin, g.Hi, g.Wi, g.Wo, pl[2], groups, w_gs, x_gs, ldx < 0 ? g.K : ldx);
  HF_LAUNCH_OK("shape_gemm");
  return HF_OK;
}

}  // namespace
}  // namespace hf
