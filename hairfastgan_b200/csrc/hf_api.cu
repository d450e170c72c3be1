// C-ABI entry points (include/hairfast_b200.h) for the operator- and module-level calls, plus the
// process-wide plumbing: thread-local error string, device selection, TMA descriptor encoding.
#include <stdarg.h>
#include <string.h>

#include <algorithm>

#include "hf_kernels.cuh"

namespace hf {

static thread_local char g_err[512] = "";
static thread_local int g_launches = 0;
static thread_local int g_device = -1;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static thread_local long long g_launches_total = 0;
void count_launch(int n) { g_launches += n; g_launches_total += n; }
long long total_launch_count() { return g_launches_total; }
void reset_launch_count() { g_launches = 0; }

int num_sms() {
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (!sms[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    sms[dev] = n;
  }
  return sms[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap(CUtensorMap* map, int dtype, int rank, void* gaddr, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes,
                const uint32_t* elem_strides) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the CUDA driver");
    return HF_ERR_CUDA;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(map, dtype == HF_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                  (cuuint32_t)rank, gaddr, gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu,%llu,..] box [%u,%u,..] swizzle %d",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
              rank > 1 ? box[1] : 0, swizzle_bytes);
    return HF_ERR_CUDA;
  }
  return HF_OK;
}

static inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// packed blob of one conv: [wpk 16-bit N x K][wsq fp32 Cout x Cin]
static size_t conv_wpk_bytes(const hf_conv_desc* d) {
  const size_t K = (size_t)d->ksize * d->ksize * d->cin;
  const size_t N = d->upsample ? 4 * (size_t)d->cout : (size_t)d->cout;
  return align256(N * K * 2);
}

static int check_desc(const hf_conv_desc* d) {
  HF_REQUIRE(d, "conv: null descriptor");
  HF_REQUIRE(d->dtype == HF_BF16 || d->dtype == HF_F16, "conv: bad dtype %d", d->dtype);
  HF_REQUIRE(d->ksize == 3 || d->ksize == 1, "conv: kernel size %d unsupported (1 or 3)", d->ksize);
  HF_REQUIRE(d->cin >= 32 && d->cin % 32 == 0 && d->cout >= 32 && d->cout % 32 == 0,
             "conv: channels (%d -> %d) must be multiples of 32", d->cin, d->cout);
  HF_REQUIRE(!d->upsample || d->ksize == 3, "conv: upsample needs ksize 3");
  return HF_OK;
}

static int ensure_device() {
  if (g_device >= 0) {
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != g_device) HF_CUDA_OK(cudaSetDevice(g_device));
  }
  return HF_OK;
}
int ensure_device_current() { return ensure_device(); }

}  // namespace hf

using namespace hf;

extern "C" {

int hf_version(void) { return 90; }
const char* hf_last_error(void) { return g_err; }
int hf_last_launch_count(void) { return g_launches; }
long long hf_total_launch_count(void) { return hf::total_launch_count(); }

int hf_set_device(int device) {
  int n = 0;
  HF_CUDA_OK(cudaGetDeviceCount(&n));
  HF_REQUIRE(device >= 0 && device < n, "hf_set_device: device %d out of range (%d devices)", device, n);
  HF_CUDA_OK(cudaSetDevice(device));
  int major = 0, minor = 0;
  HF_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  HF_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  if (major != 9) {
    set_error("device %d is sm_%d%d; libhairfast_sm90 only contains sm_90a code and has no fallback", device,
              major, minor);
    return HF_ERR_UNSUPPORTED;
  }
  g_device = device;
  return HF_OK;
}

int hf_sm_count(void) {
  if (ensure_device()) return -1;
  return num_sms();
}

int hf_upfirdn2d_f32(const float* x, float* y, const float* kernel, int planes, int in_h, int in_w, int kernel_h,
                     int kernel_w, int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_x1, int pad_y0,
                     int pad_y1, void* stream) {
  int rc = ensure_device();
  if (rc) return rc;
  reset_launch_count();
  return launch_upfirdn2d(x, y, kernel, planes, in_h, in_w, kernel_h, kernel_w, up_x, up_y, down_x, down_y, pad_x0,
                          pad_x1, pad_y0, pad_y1, (cudaStream_t)stream);
}

int hf_bias_act_f32(const float* x, const float* bias, float* y, int64_t n, int size_b, int64_t step_b, int act,
                    float alpha, float scale, void* stream) {
  int rc = ensure_device();
  if (rc) return rc;
  reset_launch_count();
  return launch_bias_act(x, bias, y, n, size_b, step_b, act, alpha, scale, (cudaStream_t)stream);
}

size_t hf_conv_packed_bytes(const hf_conv_desc* d) {
  if (check_desc(d)) return 0;
  return conv_wpk_bytes(d) + align256((size_t)d->cout * d->cin * 4);
}

int hf_conv_pack(const hf_conv_desc* d, const float* weight, const float* blur_kernel, void* packed, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  HF_REQUIRE(weight && packed, "hf_conv_pack: null pointer");
  HF_REQUIRE(((uintptr_t)packed & 255) == 0, "hf_conv_pack: packed buffer must be 256-byte aligned");
  float* wsq = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(packed) + conv_wpk_bytes(d));
  return launch_pack_conv(weight, blur_kernel, packed, wsq, d->cout, d->cin, d->ksize, d->upsample, 0, d->dtype,
                          (cudaStream_t)stream);
}

size_t hf_conv_workspace_bytes(const hf_conv_desc* d, int batch, int height, int width) {
  if (check_desc(d) || batch <= 0 || height <= 0 || width <= 0) return 0;
  return align256((size_t)batch * d->cin * 4) + align256((size_t)batch * d->cout * 4) +
         align256((size_t)batch * height * width * d->cin * 2);
}

int hf_conv_plan_query(const hf_conv_desc* d, int batch, int height, int width, int* out) {
  int rc = check_desc(d);
  if (rc) return rc;
  HF_REQUIRE(out, "hf_conv_plan_query: null output");
  ConvLaunch cl;
  memset(&cl, 0, sizeof(cl));
  cl.B = batch; cl.H = height; cl.W = width; cl.Cin = d->cin; cl.Cout = d->cout;
  cl.taps = d->ksize * d->ksize; cl.up = d->upsample; cl.dtype = d->dtype;
  ConvPlan pl;
  if ((rc = conv_plan(cl, &pl))) return rc;
  const int v[12] = {pl.halo, pl.n_tile, pl.num_n_tiles, pl.G, pl.na_slots, pl.pitch, pl.b_resident, pl.stages,
                     (int)pl.smem_bytes, pl.num_tiles, pl.grid, pl.kchunk};
  for (int i = 0; i < 12; ++i) out[i] = v[i];
  return HF_OK;
}

static int conv_forward_impl(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, void* stream,
                             int time_iters, float* avg_ms);

int hf_conv_forward(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, void* stream) {
  return conv_forward_impl(d, packed, io, stream, 0, nullptr);
}

int hf_conv_time_kernel(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, int iters, float* avg_ms,
                        void* stream) {
  HF_REQUIRE(iters > 0 && avg_ms, "hf_conv_time_kernel: iters must be > 0 and avg_ms non-null");
  return conv_forward_impl(d, packed, io, stream, iters, avg_ms);
}

static int conv_forward_impl(const hf_conv_desc* d, const void* packed, const hf_conv_io* io, void* stream,
                             int time_iters, float* avg_ms) {
  int rc = check_desc(d);
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  reset_launch_count();
  HF_REQUIRE(packed && io && io->x && io->style && io->mod_weight && io->mod_bias && io->y && io->workspace,
             "hf_conv_forward: null pointer");
  HF_REQUIRE(io->batch > 0 && io->height > 0 && io->width > 0, "hf_conv_forward: bad shape");
  HF_REQUIRE(((uintptr_t)io->workspace & 255) == 0 && ((uintptr_t)packed & 255) == 0,
             "hf_conv_forward: workspace / packed must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = io->batch;
  uint8_t* ws = reinterpret_cast<uint8_t*>(io->workspace);
  float* s = reinterpret_cast<float*>(ws);
  float* dd = reinterpret_cast<float*>(ws + align256((size_t)B * d->cin * 4));
  void* xh = ws + align256((size_t)B * d->cin * 4) + align256((size_t)B * d->cout * 4);
  const float* wsq = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(packed) + conv_wpk_bytes(d));

  AffineJob aj;
  aj.mw = io->mod_weight; aj.mb = io->mod_bias; aj.style = io->style; aj.s = s; aj.C = d->cin;
  aj.wscale = 1.0f / sqrtf((float)io->style_dim);
  if ((rc = launch_affine(&aj, 1, B, io->style_dim, io->style_stride, st))) return rc;
  if (io->demodulate) {
    DemodJob dj;
    dj.wsq = wsq; dj.s = s; dj.d = dd; dj.Cout = d->cout; dj.Cin = d->cin;
    if ((rc = launch_demod(&dj, 1, B, st))) return rc;
  }
  if ((rc = launch_modulate_to_nhwc(io->x, io->x_batch_broadcast, s, nullptr, 0.f, xh, B, d->cin,
                                    io->height * io->width, d->dtype, st)))
    return rc;
  ConvLaunch cl;
  memset(&cl, 0, sizeof(cl));
  cl.B = B; cl.H = io->height; cl.W = io->width; cl.Cin = d->cin; cl.Cout = d->cout;
  cl.taps = d->ksize * d->ksize; cl.up = d->upsample; cl.dtype = d->dtype;
  cl.xhat_in = xh; cl.wpk = packed;
  cl.d = io->demodulate ? dd : nullptr;
  cl.noise = io->noise; cl.noise_batch = io->noise_batch; cl.noise_w = io->noise_weight;
  cl.bias = io->act_bias; cl.act = io->act;
  cl.out_nchw = io->y;
  if (time_iters <= 0) return launch_conv(cl, st, nullptr);
  // warm-up launch, then `time_iters` back-to-back launches bracketed by events on the launching stream
  if ((rc = launch_conv(cl, st, nullptr))) return rc;
  cudaEvent_t e0, e1;
  HF_CUDA_OK(cudaEventCreate(&e0));
  HF_CUDA_OK(cudaEventCreate(&e1));
  HF_CUDA_OK(cudaEventRecord(e0, st));
  for (int i = 0; i < time_iters; ++i)
    if ((rc = launch_conv(cl, st, nullptr))) return rc;
  HF_CUDA_OK(cudaEventRecord(e1, st));
  HF_CUDA_OK(cudaEventSynchronize(e1));
  float ms = 0.f;
  HF_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *avg_ms = ms / time_iters;
  return HF_OK;
}

int hf_torgb_forward(const float* x, const float* style, int64_t style_stride, int style_dim,
                     const float* conv_weight, const float* mod_weight, const float* mod_bias, const float* bias,
                     const float* up_kernel, const float* skip, float* y, int batch, int cin, int height, int width,
                     void* workspace, void* stream) {
  int rc = ensure_device();
  if (rc) return rc;
  reset_launch_count();
  HF_REQUIRE(x && style && conv_weight && mod_weight && mod_bias && y && workspace, "hf_torgb_forward: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  AffineJob aj;
  aj.mw = mod_weight; aj.mb = mod_bias; aj.style = style; aj.s = (float*)workspace; aj.C = cin;
  aj.wscale = 1.0f / sqrtf((float)style_dim);
  if ((rc = launch_affine(&aj, 1, batch, style_dim, style_stride, st))) return rc;
  return launch_torgb_nchw(x, conv_weight, 1.0f / sqrtf((float)cin), (const float*)workspace, bias, skip, up_kernel,
                           y, batch, cin, height, width, st);
}

}  // extern "C"
