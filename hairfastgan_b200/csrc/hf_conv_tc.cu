// wgmma implicit-GEMM convolution for sm_90a: the ModulatedConv2d / StyledConv hot loop.
//
//   y[b,o,p] = act( d[b,o] * sum_{tap,c} W~[o,tap,c] * xh[b, p+tap, c]  + nw*noise[b,p] + bias[o] )
//
// (reference: models/stylegan2/model.py:238-279 + :288-293 + op/fused_act.py:73-82, restated in the
// shared-weight form of SURVEY Appendix C-1: the per-sample style scale s[b,c] is folded into the
// 16-bit NHWC activation `xh` by the producer of that tensor, the demodulation d[b,o] is applied to
// the fp32 accumulator in the epilogue).  The upsampling conv (conv_transpose2d stride 2 + 4x4 blur,
// model.py:252-263) runs as four 3x3 correlations, one per output parity, stacked along GEMM-N
// (Appendix C-2), so the same kernel serves both.
//
// GEMM view per tile:  D[128 pixels, n_tile] += A[128 pixels, KCHUNK ch] * B[n_tile, KCHUNK ch]^T over taps x
// channel chunks.  One TMA box per (tap, channel chunk), shifted by the tap offset, brings the activations into a
// swizzled K-major ring slot next to the matching weight box; TMA out-of-bounds zero fill *is* the conv zero
// padding, and the 128 GEMM rows may span several batch samples (4x4x8, 8x8x2).  Stride 2 walks every other input
// pixel through TMA element strides.
//
// conv_wgmma_kernel: persistent CTAs with a static schedule, three warpgroups.  Warpgroup 0 is the TMA producer
// (one thread); warpgroups 1 and 2 each own 64 of the 128 GEMM rows, issue wgmma m64 x n_tile x k16 with the
// fp32 accumulator in registers, release ring slots through mbarriers as their MMAs retire, and run the fused
// epilogue: the accumulator goes through a padded fp32 staging tile in shared memory so that one thread sees
// 32 consecutive channels of one pixel (two threads per pixel, alternating 32-channel chunks).  While the
// consumers run an epilogue the producer is already filling the ring for their next tile.
//
// The same kernel runs the plain convolutions of the encoders / PostProcess stack / BiSeNet (`epi == 1`:
// v = act(acc*scale[o] + shift[o]) (+ residual, before or after the activation), optional second output
// v*s2[o] + b2[o] for the next block's BatchNorm; stride 2; grouped heads).
#include <stdlib.h>
#include <string.h>

#include "hf_kernels.cuh"

namespace hf {

constexpr int kMaxStages = 8;
constexpr int kMaxDynSmem = 232448;   // 227 KB: opt-in dynamic shared memory per block on sm_90
constexpr int kTableBytes = 16384;   // 512 entries x 32 B
constexpr float kSqrt2 = 1.41421356237309515f;

struct ConvKernelParams {
  int B, H, W, Cin, Cout;
  int Ho, Wo;
  int taps, up, act;
  int TW, TH, TB, tiles_x, tiles_y;
  int n_tile, num_n_tiles, num_tiles;   // num_tiles = work items (M tiles x N tiles)
  int num_m_tiles;
  int num_kb;              // taps * Cin / KCHUNK
  int kc_per_tap;          // Cin / KCHUNK
  int stages;              // A+B ring stages
  uint32_t stage_bytes, a_bytes;
  const float* d;
  const float* noise;
  int64_t noise_bstride;
  const float* noise_w;
  const float* bias;
  const float* s_next;
  uint16_t* xhat_out;
  float* out_nchw;
  const float* rgb_w;
  const float* rgb_s;
  float* rgb_partial;
  // plain (encoder) convolution: epi == 1 -> v = act(acc*scale[o] + shift[o]) + residual;
  // y16 (= xhat_out) = v ; y16b = v*s2[o] + b2[o] ; out_nchw = v
  int dbg;
  int epi, stride, cin_g, cout_g, enc_act, enc_post;
  float enc_slope0;
  const float* enc_scale;
  const float* enc_shift;
  const float* enc_slope;
  const float* enc_s2;
  const float* enc_b2;
  const uint16_t* enc_residual;
  uint16_t* enc_y16b;
};

// generator: {d, bias, s_next, w_rgb0 | w_rgb1, w_rgb2, -, -};  encoder: {scale, shift, slope, - | s2, b2, -, -}.
// A warp-wide shared load costs one wavefront per 128 B of register write-back even when every lane reads the same
// address (ncu, round 2: the table look-ups were 60 % of the LSU shared pipe on the 1024^2 layer), so each variant
// fetches exactly the words it uses: LDS.64 + LDS.32 (3 wavefronts) instead of LDS.128 (4) without ToRGB,
// LDS.128 + LDS.64 (6) instead of 2 x LDS.128 (8) with it.
struct __align__(16) TableEntry {
  float d, bias, s_next, w0;
  float w1, w2, pad, pad2;
};

struct MTile {
  int x0, y0, bt;
};
__device__ __forceinline__ MTile decode_mtile(const ConvKernelParams& p, int mt) {
  MTile t;
  t.x0 = (mt % p.tiles_x) * p.TW;
  t.y0 = ((mt / p.tiles_x) % p.tiles_y) * p.TH;
  t.bt = mt / (p.tiles_x * p.tiles_y);
  return t;
}

// Per-tile table {demod, bias, next-layer style scale, ToRGB weights}, indexed [bb][channel in tile]
// (the four parity column groups of an up-conv share an entry).  Called by the 128 threads of one group.
__device__ __forceinline__ void fill_table(const ConvKernelParams& p, TableEntry* table, int etid, int bt, int n0) {
  const int nc_tile = p.up ? p.n_tile / 4 : p.n_tile;
  const int rows = p.epi == 1 ? 1 : p.TB;      // the encoder table is per channel only
  for (int e = etid; e < rows * nc_tile; e += 128) {
    const int ebb = e / nc_tile, ol = e - ebb * nc_tile;
    const int eb = bt * p.TB + ebb;
    const int o = (p.up ? (n0 >> 2) : n0) + ol;
    TableEntry t;
    t.d = 1.f; t.bias = 0.f; t.s_next = 1.f; t.pad = 0.f; t.w0 = t.w1 = t.w2 = 0.f; t.pad2 = 0.f;
    float enc_s2 = 1.f, enc_b2 = 0.f;
    if (p.epi == 1) {            // encoder: {scale, shift, slope, -, s2, b2}
      if (p.enc_scale) t.d = __ldg(p.enc_scale + o);
      if (p.enc_shift) t.bias = __ldg(p.enc_shift + o);
      // negative-side slope of the activation: none -> 1, PReLU -> per channel, LeakyReLU -> constant, ReLU -> 0
      t.s_next = p.enc_act == 0 ? 1.f
                 : p.enc_act == 3 ? 0.f
                 : (p.enc_act == 1 && p.enc_slope) ? __ldg(p.enc_slope + o) : p.enc_slope0;
      enc_s2 = p.enc_s2 ? __ldg(p.enc_s2 + o) : 1.f;
      enc_b2 = p.enc_b2 ? __ldg(p.enc_b2 + o) : 0.f;
      t.w1 = enc_s2; t.w2 = enc_b2;                // second half of the entry: {s2, b2}
    } else if (eb < p.B) {
      const size_t bo = (size_t)eb * p.Cout + o;
      if (p.d) t.d = __ldg(p.d + bo);
      if (p.bias) t.bias = __ldg(p.bias + o);
      if (p.s_next) t.s_next = __ldg(p.s_next + bo);
      if (p.rgb_w) {
        const float rs = __ldg(p.rgb_s + bo);
        t.w0 = __ldg(p.rgb_w + o) * rs;
        t.w1 = __ldg(p.rgb_w + p.Cout + o) * rs;
        t.w2 = __ldg(p.rgb_w + 2 * p.Cout + o) * rs;
      }
      if (p.act) { t.d *= kSqrt2; t.bias *= kSqrt2; }       // lrelu(a)*sqrt2 == lrelu(a*sqrt2)
    }
    table[e] = t;
  }
}

// raw noise for one pixel (plain: .x) or its 2x2 output quad (up: x,y = top row; z,w = bottom row); the caller
// multiplies by the noise weight when the value is USED, so the load can stay in flight behind other work
__device__ __forceinline__ float4 load_noise(const ConvKernelParams& p, int b, int y, int x, float nw) {
  float4 nz = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.noise) {
    const float* np_ = p.noise + (size_t)b * p.noise_bstride;
    if (p.up) {
      const float* r0 = np_ + (size_t)(2 * y) * p.Wo + 2 * x;
      const float2 a = __ldg(reinterpret_cast<const float2*>(r0));
      const float2 c = __ldg(reinterpret_cast<const float2*>(r0 + p.Wo));
      nz = make_float4(a.x, a.y, c.x, c.y);
    } else {
      nz.x = __ldg(np_ + (size_t)y * p.Wo + x);
    }
  }
  return nz;
}

__device__ __forceinline__ float2 lds64(uint32_t saddr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
  return v;
}
__device__ __forceinline__ float lds32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}

// 32 accumulator columns of one pixel through the encoder epilogue, 8 columns (one 16-byte store) at a time.
// Table entry = {scale, shift, slope, -, s2, b2, -, -}; the activation is a > 0 ? a : a*slope with slope = 1 (none)
// / 0 (ReLU) / per-channel (PReLU) / constant (LeakyReLU), so there is no per-element branch.
template <int DT, bool RES, bool Y16B, bool NCHW>
__device__ __forceinline__ void epi_chunk_enc(uint32_t ts, const uint32_t (&acc)[32], const uint4* res, uint4* dst,
                                              uint4* dst_b, float* onchw, size_t plane_o, bool post) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    uint32_t rw[4] = {0u, 0u, 0u, 0u};
    if (RES) {
      if (res) {
        const uint4 r = __ldg(res + g);
        rw[0] = r.x; rw[1] = r.y; rw[2] = r.z; rw[3] = r.w;
      }
    }
    uint32_t pk[4], pkb[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      float v[2], vb[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int j = g * 8 + h * 2 + u;
        const float2 t01 = lds64(ts + (uint32_t)j * 32u);             // scale, shift
        float4 ta;
        ta.x = t01.x; ta.y = t01.y; ta.z = lds32(ts + (uint32_t)j * 32u + 8u);   // slope
        float a = fmaf(__uint_as_float(acc[j]), ta.x, ta.y);
        if (RES) {
          const float r = Half2T<DT>::to_float((uint16_t)(u ? (rw[h] >> 16) : (rw[h] & 0xFFFFu)));
          if (post) {                      // ResNet BasicBlock: activation after the residual add (CTA-uniform)
            a += r;
            a = fmaf(fminf(a, 0.f), ta.z, fmaxf(a, 0.f));
          } else {
            a = fmaf(fminf(a, 0.f), ta.z, fmaxf(a, 0.f));
            a += r;
          }
        } else {
          a = fmaf(fminf(a, 0.f), ta.z, fmaxf(a, 0.f));
        }
        if (NCHW) { if (onchw) onchw[(size_t)j * plane_o] = a; }
        v[u] = a;
        if (Y16B) {
          const float2 tb = lds64(ts + (uint32_t)j * 32u + 16u);       // s2, b2
          vb[u] = fmaf(a, tb.x, tb.y);
        }
      }
      pk[h] = Half2T<DT>::pack(v[0], v[1]);
      if (Y16B) pkb[h] = Half2T<DT>::pack(vb[0], vb[1]);
    }
    if (dst) dst[g] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    if (Y16B) { if (dst_b) dst_b[g] = make_uint4(pkb[0], pkb[1], pkb[2], pkb[3]); }
  }
}

// 32 accumulator columns [32q, 32q + 32) of one pixel row of the fp32 staging tile (conflict-free 16-byte reads:
// the padded row pitch puts the eight rows of one shared-memory wavefront on different banks).
__device__ __forceinline__ void load_acc_chunk(const float* srow, int q, uint32_t (&acc)[32]) {
  const float4* s4 = reinterpret_cast<const float4*>(srow + q * 32);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = s4[i];
    acc[4 * i] = __float_as_uint(v.x); acc[4 * i + 1] = __float_as_uint(v.y);
    acc[4 * i + 2] = __float_as_uint(v.z); acc[4 * i + 3] = __float_as_uint(v.w);
  }
}

// Encoder epilogue (plain conv + folded BatchNorm / bias + PReLU | LeakyReLU | ReLU + residual):
//   v = act(acc*scale[o] + shift[o]) + residual ; y16 = v ; y16b = v*s2[o] + b2[o] ; y32 (NCHW) = v
// (reference: bottleneck_IR_SE / IBasicBlock conv stacks, encoder4editing/models/encoders/helpers.py:98-120,
//  FeatureStyleEncoder/arcface/iresnet.py:28-57; GradualStyleBlock psp_encoders.py:34-55)
// Chunks q0, q0 + 2, ... of the pixel's row.
template <int DT>
__device__ __forceinline__ void epilogue_tile_enc(const ConvKernelParams& p, const TableEntry* trow, const float* srow,
                                                  int q0, int n0, int b, int y, int x, bool valid) {
  const int chunks = p.n_tile / 32;
  const size_t plane_o = (size_t)p.Ho * p.Wo;
  const size_t pix = valid ? ((size_t)b * p.Ho + y) * p.Wo + x : 0;
  const uint32_t trow_s = smem_u32(trow);
  const int variant = p.out_nchw ? 3 : ((p.enc_residual ? 1 : 0) | (p.enc_y16b ? 2 : 0));
  const bool post = p.enc_post != 0;
  for (int q = q0; q < chunks; q += 2) {
    uint32_t acc[32];
    load_acc_chunk(srow, q, acc);
    const int o_base = n0 + q * 32;
    const size_t eo = pix * p.Cout + o_base;
    const uint4* res = (p.enc_residual && valid) ? reinterpret_cast<const uint4*>(p.enc_residual + eo) : nullptr;
    uint4* dst = (p.xhat_out && valid) ? reinterpret_cast<uint4*>(p.xhat_out + eo) : nullptr;
    uint4* dst_b = (p.enc_y16b && valid) ? reinterpret_cast<uint4*>(p.enc_y16b + eo) : nullptr;
    float* onchw = (p.out_nchw && valid) ? p.out_nchw + ((size_t)b * p.Cout + o_base) * plane_o + (size_t)y * p.Wo + x
                                         : nullptr;
    const uint32_t ts = trow_s + (uint32_t)(q * 32) * (uint32_t)sizeof(TableEntry);
    switch (variant) {       // uniform across the CTA
      case 0: epi_chunk_enc<DT, false, false, false>(ts, acc, res, dst, dst_b, onchw, plane_o, post); break;
      case 1: epi_chunk_enc<DT, true, false, false>(ts, acc, res, dst, dst_b, onchw, plane_o, post); break;
      case 2: epi_chunk_enc<DT, false, true, false>(ts, acc, res, dst, dst_b, onchw, plane_o, post); break;
      default: epi_chunk_enc<DT, true, true, true>(ts, acc, res, dst, dst_b, onchw, plane_o, post); break;
    }
  }
}

// 32 accumulator columns of one pixel through the StyledConv epilogue, 8 columns (one 16-byte store) at a time.
// `ts` = shared-window address of the table entry of column 0 (LDS.128, broadcast across the warp).  RGB:
// accumulate the fused ToRGB dot products; NCHW: also store the fp32 activation (feature outputs / module-level
// API); XOUT: produce the 16-bit operand of the next conv.
template <int DT, bool RGB, bool NCHW, bool XOUT>
__device__ __forceinline__ void epi_chunk(uint32_t ts, const uint32_t (&acc)[32], float nzv, float slope, uint4* dst,
                                          float& r0, float& r1, float& r2, float* onchw, size_t plane_o) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    uint32_t pk[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      float v[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int j = g * 8 + h * 2 + u;
        float4 ta;                                                   // d, bias, s_next, w_rgb0
        if (RGB) {
          ta = lds128(ts + (uint32_t)j * 32u);
        } else {
          const float2 t01 = lds64(ts + (uint32_t)j * 32u);
          ta.x = t01.x; ta.y = t01.y; ta.z = lds32(ts + (uint32_t)j * 32u + 8u); ta.w = 0.f;
        }
        float a = fmaf(__uint_as_float(acc[j]), ta.x, nzv + ta.y);
        a = fmaxf(a, slope * a);
        if (RGB) {
          const float2 tb = lds64(ts + (uint32_t)j * 32u + 16u);     // w_rgb1, w_rgb2 (ToRGB weights * style)
          r0 = fmaf(a, ta.w, r0); r1 = fmaf(a, tb.x, r1); r2 = fmaf(a, tb.y, r2);
        }
        if (NCHW) { if (onchw) onchw[(size_t)j * plane_o] = a; }
        v[u] = a * ta.z;
      }
      if (XOUT) pk[h] = Half2T<DT>::pack(v[0], v[1]);
    }
    if (XOUT) { if (dst) dst[g] = make_uint4(pk[0], pk[1], pk[2], pk[3]); }
  }
}

// staging tile -> fused epilogue -> global, for one pixel row and the chunks q0, q0 + 2, ... of it.
//   a = acc*d + nw*noise + bias ; a = lrelu(a)*sqrt2 ; rgb += a*wrgb ; out16 = a*s_next
// Returns this thread's share of the fused ToRGB dot products (plain, non-upsampling convolutions only;
// launch_conv checks); the caller adds the two shares of a pixel.
template <int DT>
__device__ __forceinline__ float3 epilogue_tile(const ConvKernelParams& p, const TableEntry* trow, const float* srow,
                                               int q0, int n0, int b, int y, int x, bool valid, float4 nz, float nw) {
  if (p.epi == 1) {
    epilogue_tile_enc<DT>(p, trow, srow, q0, n0, b, y, x, valid);
    return make_float3(0.f, 0.f, 0.f);
  }
  const int chunks = p.n_tile / 32;
  const size_t plane_o = (size_t)p.Ho * p.Wo;
  float r0 = 0.f, r1 = 0.f, r2 = 0.f;
  // the table already carries d*sqrt2 / bias*sqrt2 when the activation is on (fill_table): lrelu(a)*sqrt2 =
  // max(a', 0.2 a') with a' = a*sqrt2; slope 1 turns the max into the identity
  const float slope = p.act ? 0.2f : 1.f, nscale = (p.act ? kSqrt2 : 1.f) * nw;
  const uint32_t trow_s = smem_u32(trow);
  const int variant = (p.rgb_partial ? 1 : 0) | (p.out_nchw ? 2 : 0) | (p.xhat_out ? 4 : 0);

  for (int q = q0; q < chunks; q += 2) {
    uint32_t acc[32];
    load_acc_chunk(srow, q, acc);
    if (p.dbg & 1) { r0 += __uint_as_float(acc[0]); continue; }
    const int par = p.up ? (q & 3) : 0;
    const int t_base = p.up ? (q >> 2) * 32 : q * 32;          // channel offset inside the tile
    const int o_base = (p.up ? (n0 >> 2) : n0) + t_base;
    const int yo = p.up ? 2 * y + (par >> 1) : y;
    const int xo = p.up ? 2 * x + (par & 1) : x;
    const float nzv = nscale * (par == 0 ? nz.x : (par == 1 ? nz.y : (par == 2 ? nz.z : nz.w)));
    float* onchw = (p.out_nchw && valid) ? p.out_nchw + ((size_t)b * p.Cout + o_base) * plane_o +
                                              (size_t)yo * p.Wo + xo
                                            : nullptr;
    uint4* dst = (p.xhat_out && valid)
                     ? reinterpret_cast<uint4*>(p.xhat_out + (((size_t)b * p.Ho + yo) * p.Wo + xo) * p.Cout + o_base)
                     : nullptr;
    const uint32_t ts = trow_s + (uint32_t)t_base * (uint32_t)sizeof(TableEntry);
    switch (variant) {     // uniform across the CTA; one specialised, fully unrolled body per combination
      case 4: epi_chunk<DT, false, false, true>(ts, acc, nzv, slope, dst, r0, r1, r2, onchw, plane_o); break;
      case 5: epi_chunk<DT, true, false, true>(ts, acc, nzv, slope, dst, r0, r1, r2, onchw, plane_o); break;
      case 1: epi_chunk<DT, true, false, false>(ts, acc, nzv, slope, dst, r0, r1, r2, onchw, plane_o); break;
      default: epi_chunk<DT, true, true, true>(ts, acc, nzv, slope, dst, r0, r1, r2, onchw, plane_o); break;
    }
  }
  return make_float3(r0, r1, r2);
}

// =============================================================================================
// conv_wgmma_kernel
// =============================================================================================
constexpr int kConvThreads = 384;     // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue, 64 rows each
constexpr int kStagePad = 4;          // staging row pitch = n_tile + 4 floats
constexpr int kMaxNTile = 128;        // m64 x n128 fp32 accumulator = 64 registers per thread

// shared memory besides the ring: staging tiles, two epilogue tables, ToRGB exchange, barriers
__host__ __device__ constexpr size_t conv_fixed_smem(int n_tile) {
  return 1024 /*align*/ + (size_t)2 * 64 * (n_tile + kStagePad) * 4 + 2 * (size_t)kTableBytes + 2 * 64 * 4 * 4 +
         2 * kMaxStages * 8;
}

template <int KCHUNK, int DT, int NT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const ConvKernelParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int SP = NT + kStagePad;
  uint8_t* stage_base = smem;
  float* staging = reinterpret_cast<float*>(smem + (size_t)p.stages * p.stage_bytes);           // [2][64][SP]
  TableEntry* tables = reinterpret_cast<TableEntry*>(staging + 2 * 64 * SP);                     // [2][512]
  float* rgbx = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(tables) + 2 * kTableBytes);  // [2][64][4]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(rgbx + 2 * 64 * 4);                           // [kMaxStages]
  uint64_t* empty_bar = full_bar + kMaxStages;                                                   // [kMaxStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr uint32_t ROW_BYTES = KCHUNK * 2;
  constexpr uint32_t SBO = 8 * ROW_BYTES;
  constexpr uint32_t LAYOUT = (KCHUNK == 64) ? GMMA_LAYOUT_SW128 : GMMA_LAYOUT_SW64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);                 // lane 0 of each of the eight consumer warps
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================ TMA producer ================================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int pad = (p.taps == 9) ? 1 : 0;
      const uint32_t tx_bytes = p.stage_bytes;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int nt = tile % p.num_n_tiles;
        const MTile tc = decode_mtile(p, tile / p.num_n_tiles);
        const int b0 = tc.bt * p.TB, n0 = nt * p.n_tile;
        const int c_off = (n0 / p.cout_g) * p.cin_g;        // grouped weights: this N tile's input channels
        for (int tap = 0; tap < p.taps; ++tap) {
          const int dy = (p.taps == 9) ? tap / 3 : 0, dx = (p.taps == 9) ? tap % 3 : 0;
          for (int kc = 0; kc < p.kc_per_tap; ++kc) {
            mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
            uint8_t* a_dst = stage_base + (size_t)stage * p.stage_bytes;
            uint8_t* b_dst = a_dst + p.a_bytes;
            mbar_expect_tx(&full_bar[stage], tx_bytes);
            // stride 2: the tensor map walks every other input pixel (TMA element strides)
            tma_load_4d(a_dst, &tmA, &full_bar[stage], c_off + kc * KCHUNK, tc.x0 * p.stride + dx - pad,
                        tc.y0 * p.stride + dy - pad, b0);
            tma_load_2d(b_dst, &tmB, &full_bar[stage], tap * p.cin_g + kc * KCHUNK, n0);
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ================================ consumers: MMA + epilogue ============================
  const int cg = (threadIdx.x >> 7) - 1;       // GEMM rows [64 cg, 64 cg + 64)
  const int t = threadIdx.x & 127;
  const int cw = t >> 5;                       // warp within the warpgroup: accumulator rows [16 cw, 16 cw + 16)
  const int bar_id = 1 + cg;
  float* stg = staging + cg * 64 * SP;
  TableEntry* table = tables + cg * (kTableBytes / (int)sizeof(TableEntry));
  float* rx = rgbx + cg * 64 * 4;
  // epilogue: two threads per pixel row (t and t + 64), alternating 32-channel chunks
  const int er = t & 63, half = t >> 6;
  const int row = cg * 64 + er;
  const int w_l = row % p.TW, h_l = (row / p.TW) % p.TH, bb = row / (p.TW * p.TH);
  const float nw = p.noise_w ? __ldg(p.noise_w) : 0.f;
  const int nc_tile = p.up ? p.n_tile / 4 : p.n_tile;
  const size_t plane_o = (size_t)p.Ho * p.Wo;
  const uint32_t a_off = (uint32_t)cg * 64u * ROW_BYTES;
  const uint32_t smem_base_u32 = smem_u32(stage_base);
  int stage = 0;
  uint32_t phase = 0;
  int cached_bt = -1, cached_nt = -1;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int nt = tile % p.num_n_tiles;
    const MTile tc = decode_mtile(p, tile / p.num_n_tiles);
    const int x = tc.x0 + w_l, y = tc.y0 + h_l, b = tc.bt * p.TB + bb;
    const int n0 = nt * p.n_tile;
    const bool valid = b < p.B;
    if (tc.bt != cached_bt || nt != cached_nt) {     // table depends on (batch tile, N tile) only
      named_bar_sync(bar_id, 128);
      fill_table(p, table, t, tc.bt, n0);
      named_bar_sync(bar_id, 128);
      cached_bt = tc.bt; cached_nt = nt;
    }
    const float4 nz = valid ? load_noise(p, b, y, x, nw) : make_float4(0.f, 0.f, 0.f, 0.f);

    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait_nocall(&full_bar[stage], phase);
      const uint32_t a_addr = smem_base_u32 + (uint32_t)stage * p.stage_bytes;
      const uint64_t da = make_gmma_desc(a_addr + a_off, SBO, LAYOUT);
      const uint64_t db = make_gmma_desc(a_addr + p.a_bytes, SBO, LAYOUT);
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KCHUNK / 16; ++k) Wgmma<NT, DT>::mma(acc, da + 2 * k, db + 2 * k);
      wgmma_commit();
      wgmma_fence_regs(acc);
      wgmma_wait<1>();                              // the previous k-block's MMAs have retired: free its slot
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

    // accumulator fragment -> staging rows (m64nNk16: row 16*warp + lane/4 (+8), columns 8j + 2*(lane%4) (+1))
    {
      const int r0 = cw * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        *reinterpret_cast<float2*>(stg + r0 * SP + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r0 + 8) * SP + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    named_bar_sync(bar_id, 128);
    const float3 r = epilogue_tile<DT>(p, table + (p.epi == 1 ? 0 : bb * nc_tile), stg + er * SP, half, n0, b, y, x,
                                       valid, nz, nw);
    if (p.rgb_partial && half) { rx[er * 4] = r.x; rx[er * 4 + 1] = r.y; rx[er * 4 + 2] = r.z; }
    named_bar_sync(bar_id, 128);                   // staging tile and ToRGB shares consumed
    if (p.rgb_partial && !half && valid) {
      float* pp = p.rgb_partial + ((size_t)nt * p.B + b) * 3 * plane_o + (size_t)y * p.Wo + x;
      pp[0] = r.x + rx[er * 4]; pp[plane_o] = r.y + rx[er * 4 + 1]; pp[2 * plane_o] = r.z + rx[er * 4 + 2];
    }
  }
}
// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int conv_up_nc(int Cout) { return Cout < 32 ? Cout : 32; }

// Experiment knobs (HF_CONV_DBG: drop the epilogue -> WRONG outputs) exist only in
// -DHF_DEBUG builds; the shipped library never reads the environment on the launch path.
#ifdef HF_DEBUG
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}
#else
static constexpr int env_int(const char*, int dflt) { return dflt; }
#endif

int conv_plan(const ConvLaunch& a, ConvPlan* p) {
  HF_REQUIRE(a.B > 0 && a.H > 0 && a.W > 0, "conv: bad shape B=%d H=%d W=%d", a.B, a.H, a.W);
  HF_REQUIRE(a.taps == 9 || a.taps == 1, "conv: taps must be 9 or 1");
  const int stride = a.stride ? a.stride : 1, groups = a.groups ? a.groups : 1;
  HF_REQUIRE(stride == 1 || stride == 2, "conv: stride %d unsupported", stride);
  HF_REQUIRE(groups >= 1 && a.Cin % groups == 0 && a.Cout % groups == 0, "conv: bad group count %d", groups);
  HF_REQUIRE(!(a.up && (stride != 1 || groups != 1)), "conv: upsample excludes stride / groups");
  const int cin_g = a.Cin / groups;
  HF_REQUIRE(cin_g % 32 == 0 && cin_g >= 32, "conv: Cin per group = %d must be a multiple of 32", cin_g);
  HF_REQUIRE(a.Cout % 32 == 0 && a.Cout >= 32, "conv: Cout=%d must be a multiple of 32", a.Cout);
  HF_REQUIRE(!a.up || a.taps == 9, "conv: upsample needs a 3x3 kernel");
  HF_REQUIRE(stride == 1 || (a.H % 2 == 0 && a.W % 2 == 0) || (a.H == 1 && a.W == 1), "conv: stride 2 needs even H, W");
  // the GEMM rows are OUTPUT pixels (input pixels for the polyphase up-conv)
  const int MH = stride == 2 ? (a.H + 1) / 2 : a.H, MW = stride == 2 ? (a.W + 1) / 2 : a.W;
  p->halo = 0; p->G = 1; p->na_slots = 0; p->pitch = 0; p->b_resident = 0; p->a_slot_bytes = 0; p->ng = 2;
  p->TW = MW < 16 ? MW : 16;
  HF_REQUIRE(128 % p->TW == 0, "conv: width %d unsupported (tile width must divide 128)", MW);
  p->TH = MH < 128 / p->TW ? MH : 128 / p->TW;
  HF_REQUIRE(128 % (p->TW * p->TH) == 0, "conv: %dx%d image does not tile into 128 GEMM rows", MH, MW);
  p->TB = 128 / (p->TW * p->TH);
  HF_REQUIRE(MW % p->TW == 0 && MH % p->TH == 0, "conv: %dx%d not divisible by tile %dx%d", MH, MW, p->TH, p->TW);
  p->tiles_x = MW / p->TW;
  p->tiles_y = MH / p->TH;
  p->tiles_b = (a.B + p->TB - 1) / p->TB;
  p->num_m_tiles = p->tiles_x * p->tiles_y * p->tiles_b;
  p->kchunk = (cin_g % 64 == 0) ? 64 : 32;
  const int ntot = a.up ? 4 * a.Cout : a.Cout;
  const int cout_g = ntot / groups;                  // an N tile never straddles two groups
  const int nmin = a.up ? 128 : 32;
  const int sms = num_sms();
  const int table_cap = kTableBytes / (int)sizeof(TableEntry);   // entries per consumer warpgroup
  const int tb_rows = a.epi == 1 ? 1 : p->TB;      // encoder epilogue tables are per channel only
  int n_tile = 0;
  if (a.force_n_tile) {
    n_tile = a.force_n_tile;
  } else {
    for (int cand = kMaxNTile; cand >= nmin; cand >>= 1) {
      if (cout_g % cand || tb_rows * (a.up ? cand / 4 : cand) > table_cap) continue;
      n_tile = cand;
      if ((int64_t)p->num_m_tiles * (ntot / cand) >= sms) break;   // largest tile that still fills the GPU
    }
  }
  HF_REQUIRE(n_tile >= nmin && n_tile <= kMaxNTile && cout_g % n_tile == 0 && n_tile % 32 == 0 &&
                 tb_rows * (a.up ? n_tile / 4 : n_tile) <= table_cap,
             "conv: no valid N tile (Ntot=%d, n_tile=%d, TB=%d)", ntot, n_tile, p->TB);
  p->n_tile = n_tile;
  p->num_n_tiles = ntot / n_tile;
  p->nc = a.up ? n_tile / 4 : n_tile;
  const size_t fixed = conv_fixed_smem(n_tile);
  const size_t budget = kMaxDynSmem - fixed;
  const int row_bytes = p->kchunk * 2;
  const size_t stage_bytes = (size_t)128 * row_bytes + (size_t)n_tile * row_bytes;
  int stages = (int)(budget / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  HF_REQUIRE(stages >= 2, "conv: not enough shared memory for 2 stages");
  p->stages = stages;
  p->smem_bytes = fixed + stages * stage_bytes;
  p->num_tiles = p->num_m_tiles * p->num_n_tiles;
  p->grid = p->num_tiles < sms ? p->num_tiles : sms;
  return HF_OK;
}

template <int KCHUNK, int DT>
static int launch_conv_kernel(int n_tile, const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvKernelParams& kp,
                              const ConvPlan& pl, cudaStream_t st) {
  void (*kern)(const CUtensorMap, const CUtensorMap, const ConvKernelParams) =
      n_tile == 32 ? conv_wgmma_kernel<KCHUNK, DT, 32>
                   : (n_tile == 64 ? conv_wgmma_kernel<KCHUNK, DT, 64> : conv_wgmma_kernel<KCHUNK, DT, 128>);
  HF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
  kern<<<pl.grid, kConvThreads, pl.smem_bytes, st>>>(tmA, tmB, kp);
  HF_LAUNCH_OK("conv_wgmma");
  count_launch();
  return HF_OK;
}

int launch_conv(const ConvLaunch& a, cudaStream_t st, ConvPlan* plan_out) {
  ConvPlan pl;
  int rc = conv_plan(a, &pl);
  if (rc) return rc;
  HF_REQUIRE(a.xhat_in && a.wpk, "conv: null operand pointer");
  HF_REQUIRE(!a.rgb_partial || (a.rgb_w && a.rgb_s), "conv: rgb_partial needs rgb_w and rgb_s");
  HF_REQUIRE(!a.rgb_partial || !a.up, "conv: the fused ToRGB partial sums exist for non-upsampling convs only");
  HF_REQUIRE(!a.noise || a.noise_w, "conv: noise given without noise weight");
  HF_REQUIRE((((uintptr_t)a.xhat_in | (uintptr_t)a.wpk | (uintptr_t)a.xhat_out) & 15) == 0,
             "conv: 16-bit tensors must be 16-byte aligned");
  HF_REQUIRE(pl.n_tile == 32 || pl.n_tile == 64 || pl.n_tile == 128, "conv: N tile %d has no kernel", pl.n_tile);

  const int stride = a.stride ? a.stride : 1, groups = a.groups ? a.groups : 1;
  const int cin_g = a.Cin / groups;
  alignas(64) CUtensorMap tmA, tmB;
  {
    uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.B};
    uint64_t strides[3] = {(uint64_t)a.Cin * 2, (uint64_t)a.W * a.Cin * 2, (uint64_t)a.H * a.W * a.Cin * 2};
    uint32_t box[4] = {(uint32_t)pl.kchunk, (uint32_t)pl.TW, (uint32_t)pl.TH, (uint32_t)pl.TB};
    uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    // stride 2: the box is traversed with element stride 2, so it must span 2*T elements to deliver T samples
    if (stride == 2) { box[1] = (uint32_t)pl.TW * 2; box[2] = (uint32_t)pl.TH * 2; }
    rc = encode_tmap(&tmA, a.dtype, 4, const_cast<void*>(a.xhat_in), dims, strides, box, pl.kchunk * 2,
                     stride == 2 ? es : nullptr);
    if (rc) return rc;
  }
  {
    const uint64_t K = (uint64_t)a.taps * cin_g;
    const uint64_t N = a.up ? 4ull * a.Cout : (uint64_t)a.Cout;
    uint64_t dims[2] = {K, N};
    uint64_t strides[1] = {K * 2};
    uint32_t box[2] = {(uint32_t)pl.kchunk, (uint32_t)pl.n_tile};
    rc = encode_tmap(&tmB, a.dtype, 2, const_cast<void*>(a.wpk), dims, strides, box, pl.kchunk * 2);
    if (rc) return rc;
  }

  ConvKernelParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.B = a.B; kp.H = a.H; kp.W = a.W; kp.Cin = a.Cin; kp.Cout = a.Cout;
  kp.Ho = a.up ? 2 * a.H : (stride == 2 ? (a.H + 1) / 2 : a.H);
  kp.Wo = a.up ? 2 * a.W : (stride == 2 ? (a.W + 1) / 2 : a.W);
  kp.taps = a.taps; kp.up = a.up; kp.act = a.act;
  kp.TW = pl.TW; kp.TH = pl.TH; kp.TB = pl.TB; kp.tiles_x = pl.tiles_x; kp.tiles_y = pl.tiles_y;
  kp.n_tile = pl.n_tile; kp.num_n_tiles = pl.num_n_tiles; kp.num_tiles = pl.num_tiles;
  kp.num_m_tiles = pl.num_m_tiles;
  kp.kc_per_tap = cin_g / pl.kchunk;
  kp.num_kb = a.taps * kp.kc_per_tap;
  kp.stages = pl.stages;
  kp.a_bytes = 128u * pl.kchunk * 2;
  kp.stage_bytes = kp.a_bytes + (uint32_t)pl.n_tile * pl.kchunk * 2;
  kp.d = a.d;
  kp.noise = a.noise;
  kp.noise_bstride = (a.noise && a.noise_batch > 1) ? (int64_t)kp.Ho * kp.Wo : 0;
  kp.noise_w = a.noise ? a.noise_w : nullptr;
  kp.bias = a.bias;
  kp.s_next = a.s_next;
  kp.xhat_out = (uint16_t*)a.xhat_out;
  kp.out_nchw = a.out_nchw;
  kp.rgb_w = a.rgb_partial ? a.rgb_w : nullptr;
  kp.rgb_s = a.rgb_s;
  kp.rgb_partial = a.rgb_partial;
  kp.dbg = env_int("HF_CONV_DBG", 0);       // experiments only: 1 = epilogue reduced to the accumulator read
  kp.epi = a.epi; kp.stride = stride; kp.cin_g = cin_g; kp.enc_post = a.enc_post;
  kp.cout_g = (a.up ? 4 * a.Cout : a.Cout) / groups;
  kp.enc_act = a.enc_act; kp.enc_slope0 = a.enc_slope0;
  kp.enc_scale = a.enc_scale; kp.enc_shift = a.enc_shift; kp.enc_slope = a.enc_slope;
  kp.enc_s2 = a.enc_s2; kp.enc_b2 = a.enc_b2;
  kp.enc_residual = (const uint16_t*)a.enc_residual;
  kp.enc_y16b = (uint16_t*)a.enc_y16b;
  HF_REQUIRE(!a.epi || !a.up, "conv: the encoder epilogue has no upsampling form");
  if (plan_out) *plan_out = pl;

  const bool bf = a.dtype == HF_BF16;
  if (pl.kchunk == 64)
    return bf ? launch_conv_kernel<64, HF_BF16>(pl.n_tile, tmA, tmB, kp, pl, st)
              : launch_conv_kernel<64, HF_F16>(pl.n_tile, tmA, tmB, kp, pl, st);
  return bf ? launch_conv_kernel<32, HF_BF16>(pl.n_tile, tmA, tmB, kp, pl, st)
            : launch_conv_kernel<32, HF_F16>(pl.n_tile, tmA, tmB, kp, pl, st);
}

}  // namespace hf
