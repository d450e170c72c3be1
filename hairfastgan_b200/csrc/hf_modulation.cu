// HairFast's latent modulation stacks (models/Encoders.py:13-137): 5 ModulationModules of
//   x <- LeakyReLU(LayerNorm_[L,512](fc(x)) * (1 + gamma(e)) + beta(e))      (no LeakyReLU after the last)
// with gamma / beta = Linear -> LayerNorm([middle]) -> LeakyReLU -> Linear of the embedding e.
//
// The ten gamma / beta MLPs of a stack read only e, so they run before the chain as two weight-streaming GEMMs on
// hf_splitk_gemm.cuh's kernel: the ten first Linears stacked into one [10 middle, inp] GEMM (reduced with the row
// LayerNorm + LeakyReLU fused in), the ten second Linears as one grouped launch.  Only the fc chain is sequential; it
// runs in one launch on clusters of 8 CTAs per (stack, sample), each CTA owning 64 of the 512 fc outputs, with the
// whole-sample LayerNorm statistics and the next module's operand exchanged over distributed shared memory.
// Fixed summation orders everywhere: results are deterministic.
#include <cooperative_groups.h>

#include "hf_splitk_gemm.cuh"

namespace cg = cooperative_groups;

namespace hf {
namespace {

constexpr int kDim = 512;                  // fc width
constexpr int kModules = 5;
constexpr int kBranches = 2 * kModules;    // gamma / beta per module
constexpr int kMaxLayers = 24;
constexpr float kSlope = 0.01f;            // nn.LeakyReLU()
constexpr float kEps = 1e-5f;              // nn.LayerNorm

struct Desc {
  int L, inp, middle, stacks, rows, B;
};

int check_desc(const hf_mod_desc* d, int batch, const char* what, Desc* out) {
  HF_REQUIRE(d->layers >= 1 && d->layers <= kMaxLayers, "%s: layers %d (1..%d)", what, d->layers, kMaxLayers);
  HF_REQUIRE(d->stacks == 1 || d->stacks == 2, "%s: stacks %d (1 or 2)", what, d->stacks);
  HF_REQUIRE(d->inp > 0 && d->inp % kDim == 0 && d->inp / kDim * d->stacks <= 3,
             "%s: inp %d (512 n, n * stacks <= 3)", what, d->inp);
  HF_REQUIRE(d->middle >= 256 && d->middle <= 1024 && d->middle % 256 == 0, "%s: middle %d (256 n, <= 1024)", what,
             d->middle);
  HF_REQUIRE(batch >= 1 && (int64_t)batch * d->layers <= 65535, "%s: batch %d (batch * layers <= 65535)", what, batch);
  *out = Desc{d->layers, d->inp, d->middle, d->stacks, batch * d->layers, batch};
  return HF_OK;
}

// ------------------------------------------------------------------------------------------------
// Embedding rows to 16-bit: e16[s][p][k] = src[s * nseg + k / 512][b][l][k % 512], p = b L + l.
// ------------------------------------------------------------------------------------------------
struct Sources {
  hf_mod_rows r[3];
};

template <int DT>
__global__ void __launch_bounds__(256) mod_embed16_kernel(Sources src, uint16_t* __restrict__ e16, int L, int rows,
                                                          int inp, int stacks) {
  const int k8n = inp / 8, nseg = inp / kDim;
  const int64_t total = (int64_t)stacks * rows * k8n;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % k8n) * 8;
    const int64_t sp = i / k8n;
    const int s = (int)(sp / rows), p = (int)(sp % rows), b = p / L, l = p - b * L, seg = k / kDim;
    const int q = s * nseg + seg;
    const hf_mod_rows r = q == 0 ? src.r[0] : q == 1 ? src.r[1] : src.r[2];     // no local-memory copy
    const float* x = r.ptr + b * r.batch_stride + l * r.row_stride + (k - seg * kDim);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __ldg(x + j);
    st8<DT>(e16 + sp * inp + k, v);
  }
}

// ------------------------------------------------------------------------------------------------
// Style layer 1's reduction: one CTA per (stack s, branch j, row p) over the branch's `middle` columns,
//   v = bias + sum_split part (split order), LayerNorm (biased variance, two passes), affine, LeakyReLU -> 16-bit.
// part [splits][stacks][rows][10 middle]; h16 [rows][stacks 10 middle].
// ------------------------------------------------------------------------------------------------
constexpr int kLnThreads = 256;

// sum over the CTA, the same value in every thread: warp butterflies, then the warp sums in order
__device__ __forceinline__ float cta_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  __syncthreads();                          // red is free (a previous call has been read by every thread)
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < kLnThreads / 32; ++i) t += red[i];
  return t;
}

template <int DT>
__global__ void __launch_bounds__(kLnThreads) mod_hidden_ln_kernel(const float* __restrict__ part, int S, int rows,
                                                                   int middle, int stacks,
                                                                   const float* __restrict__ bias,
                                                                   const float* __restrict__ ln_w,
                                                                   const float* __restrict__ ln_b,
                                                                   uint16_t* __restrict__ h16) {
  __shared__ float red[kLnThreads / 32];
  const int sj = blockIdx.x, s = sj / kBranches, j = sj - s * kBranches, p = blockIdx.y;
  const int width = kBranches * middle, per = middle / kLnThreads;     // 1..4
  const int64_t split_stride = (int64_t)stacks * rows * width;
  const float* src = part + ((int64_t)s * rows + p) * width + j * middle;
  const float* b1 = bias + (int64_t)s * width + j * middle;
  float v[4];
  float sum = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (e >= per) break;
    const int n = threadIdx.x + e * kLnThreads;
    float t = __ldg(b1 + n);
    for (int sp = 0; sp < S; ++sp) t += __ldg(src + sp * split_stride + n);
    v[e] = t;
    sum += t;
  }
  const float mean = cta_sum(sum, red) / (float)middle;
  float sq = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (e >= per) break;
    const float c = v[e] - mean;
    sq = fmaf(c, c, sq);
  }
  const float rstd = 1.f / sqrtf(cta_sum(sq, red) / (float)middle + kEps);
  const float* g = ln_w + (int64_t)sj * middle;
  const float* bb = ln_b + (int64_t)sj * middle;
  uint16_t* dst = h16 + (int64_t)p * stacks * width + (int64_t)sj * middle;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (e >= per) break;
    const int n = threadIdx.x + e * kLnThreads;
    const float t = (v[e] - mean) * rstd * __ldg(g + n) + __ldg(bb + n);
    dst[n] = Half2T<DT>::one(t > 0.f ? t : t * kSlope);
  }
}

// ------------------------------------------------------------------------------------------------
// The fc chain.  Cluster of 8 CTAs per (stack s, sample b); CTA r owns fc outputs 64 r .. 64 r + 63.
//   shared: w ring [2][64][512] 16-bit (module m's weight slice in slot m % 2; module m + 2's is loaded while
//           module m's LayerNorm runs), x [8 NT][512] 16-bit = the full operand of the current module (every CTA
//           holds a copy), y [2][8 NT][64] fp32 = the two K halves of the current module's outputs.
//   prologue: PixelNorm over the L rows of each column (models/stylegan2/model.py:21), every CTA for all 512.
//   module m: y = x W_r^T (mma.sync, warp = 16 outputs x one K half) + bias; the sample's mean and centred sum of
//           squares, each a CTA sum then the 8 CTA sums read over DSMEM in rank order; (y - mean) rstd (1 + gamma) +
//           beta and LeakyReLU; the 16-bit slice goes into every CTA's x.
//   epilogue: out = base + 0.1 dt.  With two stacks the CTA of the second stack to finish a (sample, slice) adds
//           both: dt of the first is passed through global memory, the order found by a counter.
// x rows and w rows are 1024 bytes; 16-byte chunk c of row r is stored at chunk c ^ (r % 8) (conflict-free ldmatrix).
// ------------------------------------------------------------------------------------------------
constexpr int kCta = 8, kCols = kDim / kCta, kChainThreads = 256;

struct ChainArgs {
  const uint16_t* w;   // [stacks][5][512][512]
  const float* bias;   // [stacks][5][512]
  const float* gb;     // [10 stacks][rows][512]
  hf_mod_rows x0[2];
  hf_mod_rows base;
  float* out;          // [B][L][512]
  float* dt;           // [2][B][L][512], two stacks
  int* count;          // [B][8] zeroed, two stacks
  int L, B, stacks;
};

__device__ __forceinline__ int xsw(int row, int chunk) { return row * kDim + ((chunk ^ (row & 7)) << 3); }

template <int NT>
constexpr int chain_smem() {
  return (2 * kCols * kDim + NT * 8 * kDim) * 2 + 2 * NT * 8 * kCols * 4;
}

template <int DT, int NT>
__global__ void __cluster_dims__(kCta, 1, 1) __launch_bounds__(kChainThreads, 1) mod_chain_kernel(ChainArgs a) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint16_t* sw = reinterpret_cast<uint16_t*>(smem_raw);
  uint16_t* sx = sw + 2 * kCols * kDim;
  float* ys = reinterpret_cast<float*>(sx + NT * 8 * kDim);
  __shared__ float red[kModules][2];
  __shared__ float cta_red[kChainThreads / 32];
  __shared__ float stat[2];
  __shared__ int last;

  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank(), q = blockIdx.x / kCta, s = q / a.B, b = q - s * a.B;
  const int L = a.L, rows = a.B * L, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float inv_n = 1.f / (float)(L * kDim);
  const uint16_t* wsrc = a.w + ((size_t)s * kModules * kDim + r * kCols) * kDim;

  auto load_w = [&](int m) {
    uint16_t* dst = sw + (m & 1) * kCols * kDim;
    const uint16_t* src = wsrc + (size_t)m * kDim * kDim;
    for (int i = tid; i < kCols * kDim / 8; i += kChainThreads) {
      const int row = i >> 6, ch = i & 63;
      cp_async16(smem_u32(dst + xsw(row, ch)), src + (size_t)row * kDim + ch * 8, 16);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  load_w(0);
  load_w(1);

  // PixelNorm: x[l][c] * rsqrt(mean_l x[l][c]^2 + 1e-8); rows L .. 8 NT - 1 are zero
  {
    const hf_mod_rows x0 = a.x0[s];
    const float* xb = x0.ptr + b * x0.batch_stride;
    for (int c = tid; c < kDim; c += kChainThreads) {
      float ss = 0.f;
      for (int l = 0; l < L; ++l) {
        const float v = __ldg(xb + l * x0.row_stride + c);
        ss = fmaf(v, v, ss);
      }
      const float inv = 1.f / sqrtf(ss / (float)L + 1e-8f);
      for (int l = 0; l < NT * 8; ++l)
        sx[xsw(l, c >> 3) + (c & 7)] = Half2T<DT>::one(l < L ? __ldg(xb + l * x0.row_stride + c) * inv : 0.f);
    }
  }

  // this CTA's sum of v, added over the cluster in rank order: the same value in every CTA of the cluster
  auto cluster_sum = [&](float v, float* slot) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    if (lane == 0) cta_red[warp] = v;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
      for (int i = 0; i < kChainThreads / 32; ++i) t += cta_red[i];
      *slot = t;
    }
    cluster.sync();
    if (tid == 0) {
      float t = 0.f;
      for (int i = 0; i < kCta; ++i) t += *cluster.map_shared_rank(slot, i);
      stat[0] = t;
    }
    __syncthreads();
    return stat[0];
  };

  constexpr int kPer = NT * 8 * kCols / kChainThreads;      // elements per thread: 2 NT
  const int mi = warp & 3, kh = warp >> 2;
  for (int m = 0; m < kModules; ++m) {
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    {
      const uint16_t* wa = sw + (m & 1) * kCols * kDim;
      float acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[nt][i] = 0.f;
#pragma unroll 4
      for (int kk = 0; kk < kDim / 32; ++kk) {
        const int k16 = kh * (kDim / 32) + kk;
        uint32_t af[4];
        ldsm_x4(af, smem_u32(wa + xsw(mi * 16 + (lane & 15), 2 * k16 + (lane >> 4))));
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          uint32_t b0, b1;
          ldsm_x2(b0, b1, smem_u32(sx + xsw(nt * 8 + (lane & 7), 2 * k16 + ((lane >> 3) & 1))));
          mma16816<DT>(acc[nt], af, b0, b1);
        }
      }
      float* y = ys + kh * NT * 8 * kCols;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          y[(nt * 8 + (lane & 3) * 2 + (i & 1)) * kCols + mi * 16 + (lane >> 2) + (i >> 1) * 8] = acc[nt][i];
    }
    __syncthreads();
    if (m + 2 < kModules) {
      load_w(m + 2);
    } else {
      asm volatile("cp.async.commit_group;" ::: "memory");
    }

    const float* bias = a.bias + ((size_t)s * kModules + m) * kDim + r * kCols;
    float v[kPer];
    float sum = 0.f;
#pragma unroll
    for (int e = 0; e < kPer; ++e) {
      const int i = tid + e * kChainThreads, l = i / kCols, c = i % kCols;
      v[e] = 0.f;
      if (l < L) {
        v[e] = ys[i] + ys[NT * 8 * kCols + i] + __ldg(bias + c);
        sum += v[e];
      }
    }
    const float mean = cluster_sum(sum, &red[m][0]) * inv_n;
    float sq = 0.f;
#pragma unroll
    for (int e = 0; e < kPer; ++e) {
      const int l = (tid + e * kChainThreads) / kCols;
      if (l < L) {
        const float d = v[e] - mean;
        sq = fmaf(d, d, sq);
      }
    }
    const float rstd = 1.f / sqrtf(cluster_sum(sq, &red[m][1]) * inv_n + kEps);
    const float* gam = a.gb + ((size_t)(s * kBranches + 2 * m) * rows + (size_t)b * L) * kDim + r * kCols;
    const float* bet = gam + (size_t)rows * kDim;
#pragma unroll
    for (int e = 0; e < kPer; ++e) {
      const int i = tid + e * kChainThreads, l = i / kCols, c = i % kCols;
      if (l < L) {
        const float t = (v[e] - mean) * rstd * (1.f + __ldg(gam + l * kDim + c)) + __ldg(bet + l * kDim + c);
        v[e] = m + 1 < kModules && t <= 0.f ? t * kSlope : t;
      }
    }
    if (m + 1 == kModules) {
      // every CTA of the cluster has read this CTA's red[] (second cluster_sum); the final sync lets none exit early
      const float* base = a.base.ptr + b * a.base.batch_stride;
      float* out = a.out + (size_t)b * L * kDim;
      if (a.stacks == 2) {
        float* mine = a.dt + ((size_t)s * rows + (size_t)b * L) * kDim;
        const float* other = a.dt + ((size_t)(1 - s) * rows + (size_t)b * L) * kDim;
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
          const int i = tid + e * kChainThreads, l = i / kCols, c = r * kCols + i % kCols;
          if (l < L) mine[l * kDim + c] = v[e];
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) last = atomicAdd(a.count + b * kCta + r, 1) == 1;
        __syncthreads();
        if (last) {
          __threadfence();
#pragma unroll
          for (int e = 0; e < kPer; ++e) {
            const int i = tid + e * kChainThreads, l = i / kCols, c = r * kCols + i % kCols;
            if (l < L) {
              const float o = __ldcg(other + l * kDim + c);
              const float face = s == 0 ? v[e] : o, hair = s == 0 ? o : v[e];
              out[l * kDim + c] = base[l * a.base.row_stride + c] + 0.1f * (face + hair);
            }
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
          const int i = tid + e * kChainThreads, l = i / kCols, c = r * kCols + i % kCols;
          if (l < L) out[l * kDim + c] = base[l * a.base.row_stride + c] + 0.1f * v[e];
        }
      }
      cluster.sync();
      break;
    }
    // every CTA has finished this module's MMA (it entered cluster_sum after it): x may be overwritten.  Own slice
    // first, then 16-byte copies of it into the 7 other CTAs.
#pragma unroll
    for (int e = 0; e < kPer; ++e) {
      const int i = tid + e * kChainThreads, l = i / kCols, c = r * kCols + i % kCols;
      if (l < L) sx[xsw(l, c >> 3) + (c & 7)] = Half2T<DT>::one(v[e]);
    }
    __syncthreads();
    for (int i = tid; i < (kCta - 1) * L * (kCols / 8); i += kChainThreads) {
      const int t = i / (L * (kCols / 8)), lc = i - t * (L * (kCols / 8)), l = lc / (kCols / 8);
      const int off = xsw(l, r * (kCols / 8) + lc % (kCols / 8));
      uint16_t* dst = cluster.map_shared_rank(sx, t < r ? t : t + 1);
      *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(sx + off);
    }
    cluster.sync();
  }
}

template <int DT, int NT>
int launch_chain(const ChainArgs& a, cudaStream_t st) {
  constexpr int smem = chain_smem<NT>();
  static uint64_t attr_set = 0;          // per device: the opt-in above 48 KB of dynamic shared memory
  int dev = 0;
  HF_CUDA_OK(cudaGetDevice(&dev));
  if (!(attr_set >> (dev & 63) & 1)) {
    HF_CUDA_OK(cudaFuncSetAttribute(mod_chain_kernel<DT, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set |= 1ull << (dev & 63);
  }
  mod_chain_kernel<DT, NT><<<kCta * a.stacks * a.B, kChainThreads, smem, st>>>(a);
  HF_LAUNCH_OK("mod_chain");
  return HF_OK;
}

// layer 1: stacks groups of [10 middle, inp]; layer 2: 10 stacks groups of [512, middle]
struct StyleGemm {
  GemmShape g;
  int groups, cout;
  int64_t w_gs, x_gs;
  int ldx;
};

int style_gemm(const Desc& d, int layer, const char* what, StyleGemm* o) {
  HF_REQUIRE(layer == 1 || layer == 2, "%s: layer %d (1 or 2)", what, layer);
  const int P = d.rows;
  if (layer == 1)
    *o = StyleGemm{GemmShape{P, d.inp, 1, P, P}, d.stacks, kBranches * d.middle, (int64_t)kBranches * d.middle * d.inp,
                   (int64_t)P * d.inp, d.inp};
  else
    *o = StyleGemm{GemmShape{P, d.middle, 1, P, P}, kBranches * d.stacks, kDim, (int64_t)kDim * d.middle, d.middle,
                   kBranches * d.stacks * d.middle};
  return HF_OK;
}

size_t partial_bytes(const StyleGemm& sg, const int* pl) {
  return (size_t)pl[1] * sg.groups * sg.g.P * sg.cout * sizeof(float);
}

template <int DT>
int run_style_gemm(const StyleGemm& sg, const void* w16, const void* x16, float* part, cudaStream_t st, int* pl) {
  gemm_plan(sg.g, sg.cout, num_sms(), pl, sg.groups);
  const uint16_t* w = (const uint16_t*)w16;
  const uint16_t* x = (const uint16_t*)x16;
  return pl[0] == 8 ? launch_gemm<DT, 8, 0>(w, x, part, sg.cout, sg.g, pl, 0, st, sg.groups, sg.w_gs, sg.x_gs, sg.ldx)
                    : launch_gemm<DT, 64, 0>(w, x, part, sg.cout, sg.g, pl, 0, st, sg.groups, sg.w_gs, sg.x_gs,
                                             sg.ldx);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace
}  // namespace hf

using namespace hf;

extern "C" {

size_t hf_mod_workspace_bytes(const hf_mod_desc* d, int batch) {
  Desc m;
  if (ensure_device_current() || !d || (d->dtype != HF_BF16 && d->dtype != HF_F16) ||
      check_desc(d, batch, "hf_mod_workspace_bytes", &m))
    return 0;
  size_t bytes = (size_t)2 * m.rows * kDim * sizeof(float) + (size_t)m.B * kCta * sizeof(int);     // hf_mod_chain
  for (int layer = 1; layer <= 2; ++layer) {
    StyleGemm sg;
    style_gemm(m, layer, "hf_mod_workspace_bytes", &sg);
    int pl[5];
    gemm_plan(sg.g, sg.cout, num_sms(), pl, sg.groups);
    bytes = std::max(bytes, partial_bytes(sg, pl));
  }
  return bytes;
}

int hf_mod_gemm_plan(const hf_mod_desc* d, int batch, int layer, int sms, int* out) {
  HF_REQUIRE(d && out && sms > 0, "hf_mod_gemm_plan: bad arguments");
  return with_dtype(d->dtype, "hf_mod_gemm_plan", [&](auto) -> int {
    Desc m;
    StyleGemm sg;
    int rc = check_desc(d, batch, "hf_mod_gemm_plan", &m);
    if (rc || (rc = style_gemm(m, layer, "hf_mod_gemm_plan", &sg))) return rc;
    gemm_plan(sg.g, sg.cout, sms, out, sg.groups);
    return HF_OK;
  });
}

int hf_mod_embed16(const hf_mod_desc* d, int batch, const hf_mod_rows* src, void* e16, void* stream) {
  HF_REQUIRE(d, "hf_mod_embed16: null descriptor");
  return with_dtype(d->dtype, "hf_mod_embed16", [&](auto dt) -> int {
    Desc m;
    int rc = check_desc(d, batch, "hf_mod_embed16", &m);
    if (rc) return rc;
    HF_REQUIRE(src && e16 && aligned16(e16), "hf_mod_embed16: null or unaligned pointer");
    Sources s{};
    const int n = m.inp / kDim * m.stacks;
    for (int i = 0; i < n; ++i) {
      HF_REQUIRE(src[i].ptr, "hf_mod_embed16: source %d is null", i);
      s.r[i] = src[i];
    }
    if ((rc = ensure_device_current())) return rc;
    const int64_t total = (int64_t)m.stacks * m.rows * m.inp / 8;
    mod_embed16_kernel<dt><<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(s, (uint16_t*)e16, m.L, m.rows, m.inp,
                                                                             m.stacks);
    HF_LAUNCH_OK("mod_embed16");
    count_launch();
    return HF_OK;
  });
}

int hf_mod_gemm(const hf_mod_desc* d, int batch, int layer, const void* w16, const void* x16, const float* bias,
                float* y32, float* workspace, void* stream) {
  HF_REQUIRE(d, "hf_mod_gemm: null descriptor");
  return with_dtype(d->dtype, "hf_mod_gemm", [&](auto dt) -> int {
    Desc m;
    StyleGemm sg;
    int rc;
    if ((rc = check_desc(d, batch, "hf_mod_gemm", &m)) || (rc = style_gemm(m, layer, "hf_mod_gemm", &sg))) return rc;
    HF_REQUIRE(w16 && x16 && y32 && workspace, "hf_mod_gemm: null pointer");
    HF_REQUIRE(aligned16(w16) && aligned16(x16), "hf_mod_gemm: unaligned operand");
    if ((rc = ensure_device_current())) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    int pl[5];
    if ((rc = run_style_gemm<dt>(sg, w16, x16, workspace, st, pl))) return rc;
    const int64_t pc = (int64_t)sg.g.P * sg.cout, n = sg.groups * pc;
    shape_splitk_reduce_kernel<dt><<<grid_for(n), 256, 0, st>>>(workspace, pl[1], n, sg.cout, pc, bias, y32, nullptr);
    HF_LAUNCH_OK("mod_gemm_reduce");
    count_launch(2);
    return HF_OK;
  });
}

int hf_mod_hidden(const hf_mod_desc* d, int batch, const void* w16, const void* e16, const float* bias,
                  const float* ln_w, const float* ln_b, void* h16, float* workspace, void* stream) {
  HF_REQUIRE(d, "hf_mod_hidden: null descriptor");
  return with_dtype(d->dtype, "hf_mod_hidden", [&](auto dt) -> int {
    Desc m;
    StyleGemm sg;
    int rc;
    if ((rc = check_desc(d, batch, "hf_mod_hidden", &m)) || (rc = style_gemm(m, 1, "hf_mod_hidden", &sg))) return rc;
    HF_REQUIRE(w16 && e16 && bias && ln_w && ln_b && h16 && workspace, "hf_mod_hidden: null pointer");
    HF_REQUIRE(aligned16(w16) && aligned16(e16), "hf_mod_hidden: unaligned operand");
    HF_REQUIRE(((uintptr_t)h16 & 1) == 0, "hf_mod_hidden: h16 must be 2-byte aligned");
    if ((rc = ensure_device_current())) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    int pl[5];
    if ((rc = run_style_gemm<dt>(sg, w16, e16, workspace, st, pl))) return rc;
    mod_hidden_ln_kernel<dt><<<dim3(kBranches * m.stacks, m.rows), kLnThreads, 0, st>>>(
        workspace, pl[1], m.rows, m.middle, m.stacks, bias, ln_w, ln_b, (uint16_t*)h16);
    HF_LAUNCH_OK("mod_hidden_ln");
    count_launch(2);
    return HF_OK;
  });
}

int hf_mod_chain(const hf_mod_desc* d, int batch, const void* fc_w16, const float* fc_b, const float* gb,
                 const hf_mod_rows* x0, const hf_mod_rows* base, float* out, float* workspace, void* stream) {
  HF_REQUIRE(d, "hf_mod_chain: null descriptor");
  return with_dtype(d->dtype, "hf_mod_chain", [&](auto dt) -> int {
    Desc m;
    int rc = check_desc(d, batch, "hf_mod_chain", &m);
    if (rc) return rc;
    HF_REQUIRE(fc_w16 && fc_b && gb && x0 && base && base->ptr && out && workspace, "hf_mod_chain: null pointer");
    HF_REQUIRE(aligned16(fc_w16), "hf_mod_chain: unaligned weights");
    for (int s = 0; s < m.stacks; ++s) HF_REQUIRE(x0[s].ptr, "hf_mod_chain: x0[%d] is null", s);
    if ((rc = ensure_device_current())) return rc;
    ChainArgs a{};
    a.w = (const uint16_t*)fc_w16;
    a.bias = fc_b;
    a.gb = gb;
    for (int s = 0; s < m.stacks; ++s) a.x0[s] = x0[s];
    a.base = *base;
    a.out = out;
    a.dt = workspace;
    a.count = reinterpret_cast<int*>(workspace + (size_t)2 * m.rows * kDim);
    a.L = m.L;
    a.B = m.B;
    a.stacks = m.stacks;
    cudaStream_t st = (cudaStream_t)stream;
    if (m.stacks == 2) HF_CUDA_OK(cudaMemsetAsync(a.count, 0, (size_t)m.B * kCta * sizeof(int), st));
    const int nt = cdiv(m.L, 8);
    rc = nt == 1 ? launch_chain<dt, 1>(a, st) : nt == 2 ? launch_chain<dt, 2>(a, st) : launch_chain<dt, 3>(a, st);
    if (rc) return rc;
    count_launch();
    return HF_OK;
  });
}

}  // extern "C"
