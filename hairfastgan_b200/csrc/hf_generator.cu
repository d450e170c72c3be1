// Generator.forward (models/stylegan2/model.py:477-565) as one host-side chain of sm_90a kernels.
//
// Per forward: 1 affine launch (all style modulations), 1 demod launch, 1 NCHW->NHWC pre-pass for the
// first executed conv, then per layer {up-conv, conv, rgb_combine}.  Every conv epilogue applies
// demod + noise + bias + leaky-relu, multiplies by the NEXT conv's style scale while casting to the
// 16-bit NHWC activation, and (for the second conv of a layer) accumulates the ToRGB 1x1 conv.
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "hf_kernels.cuh"

namespace hf {

static inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

struct StyledL {
  int cin, cout, res_in, res_out, up;
  size_t wpk, wsq, mw, mb, noise_w, act_bias;   // byte offsets into the packed blob
};
struct RgbL {
  int cin, res;
  size_t w1, mw, mb, bias, upk;
};
struct GenLayout {
  int log_size, n_layers, n_styled, n_rgb, n_latent, style_dim;
  StyledL st[HF_MAX_STYLED];
  RgbL rgb[HF_MAX_TORGB];
  size_t const_in;
  size_t total;
};

static int channels_at(int res, int cm) {   // model.py:395-405
  switch (res) {
    case 4: case 8: case 16: case 32: return 512;
    case 64: return 256 * cm;
    case 128: return 128 * cm;
    case 256: return 64 * cm;
    case 512: return 32 * cm;
    case 1024: return 16 * cm;
  }
  return 0;
}

static int make_layout(const hf_gen_config* cfg, GenLayout* L) {
  HF_REQUIRE(cfg, "generator: null config");
  HF_REQUIRE(cfg->dtype == HF_BF16 || cfg->dtype == HF_F16, "generator: bad dtype");
  int ls = 0;
  while ((1 << ls) < cfg->size) ++ls;
  HF_REQUIRE((1 << ls) == cfg->size && ls >= 3 && ls <= 10, "generator: size %d unsupported", cfg->size);
  HF_REQUIRE(cfg->style_dim > 0 && cfg->style_dim % 4 == 0, "generator: style_dim must be a multiple of 4");
  HF_REQUIRE(channels_at(cfg->size, cfg->channel_multiplier) >= 32,
             "generator: channel_multiplier %d gives < 32 channels at %d^2 (unsupported)", cfg->channel_multiplier,
             cfg->size);
  memset(L, 0, sizeof(*L));
  L->log_size = ls;
  L->n_layers = ls - 2;
  L->n_styled = 2 * L->n_layers + 1;
  L->n_rgb = L->n_layers + 1;
  L->n_latent = 2 * ls - 2;
  L->style_dim = cfg->style_dim;
  const int D = cfg->style_dim;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align256(bytes); return o; };
  L->const_in = take((size_t)channels_at(4, cfg->channel_multiplier) * 16 * 4);
  for (int i = 0; i < L->n_styled; ++i) {
    StyledL& s = L->st[i];
    if (i == 0) {
      s.cin = s.cout = channels_at(4, cfg->channel_multiplier);
      s.res_in = s.res_out = 4; s.up = 0;
    } else {
      const int k = (i + 1) / 2;                // layer 1..n
      const int r_out = 4 << k;
      s.up = (i & 1);
      s.res_out = r_out;
      s.res_in = s.up ? r_out / 2 : r_out;
      s.cout = channels_at(r_out, cfg->channel_multiplier);
      s.cin = s.up ? channels_at(r_out / 2, cfg->channel_multiplier) : s.cout;
    }
    const size_t N = s.up ? 4 * (size_t)s.cout : (size_t)s.cout;
    s.wpk = take(N * 9 * s.cin * 2);
    s.wsq = take((size_t)s.cout * s.cin * 4);
    s.mw = take((size_t)s.cin * D * 4);
    s.mb = take((size_t)s.cin * 4);
    s.noise_w = take(4);
    s.act_bias = take((size_t)s.cout * 4);
  }
  for (int i = 0; i < L->n_rgb; ++i) {
    RgbL& r = L->rgb[i];
    r.res = 4 << i;
    r.cin = channels_at(r.res, cfg->channel_multiplier);
    r.w1 = take((size_t)3 * r.cin * 4);
    r.mw = take((size_t)r.cin * D * 4);
    r.mb = take((size_t)r.cin * 4);
    r.bias = take(3 * 4);
    r.upk = take(16 * 4);
  }
  L->total = off;
  return HF_OK;
}

struct WsLayout {
  size_t s_conv[HF_MAX_STYLED], d_conv[HF_MAX_STYLED], s_rgb[HF_MAX_TORGB];
  size_t xbuf[2], partial, rgbbuf[2];
  size_t total;
};

static void make_ws(const GenLayout& L, int B, int size, WsLayout* W) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align256(bytes); return o; };
  size_t max_x = 0, max_part = 0;
  for (int i = 0; i < L.n_styled; ++i) {
    W->s_conv[i] = take((size_t)B * L.st[i].cin * 4);
    W->d_conv[i] = take((size_t)B * L.st[i].cout * 4);
    size_t xin = (size_t)B * L.st[i].res_in * L.st[i].res_in * L.st[i].cin * 2;
    size_t xout = (size_t)B * L.st[i].res_out * L.st[i].res_out * L.st[i].cout * 2;
    max_x = xin > max_x ? xin : max_x;
    max_x = xout > max_x ? xout : max_x;
    size_t part = (size_t)(L.st[i].cout / 32) * B * 3 * L.st[i].res_out * L.st[i].res_out * 4;
    max_part = part > max_part ? part : max_part;
  }
  for (int i = 0; i < L.n_rgb; ++i) W->s_rgb[i] = take((size_t)B * L.rgb[i].cin * 4);
  W->xbuf[0] = take(max_x);
  W->xbuf[1] = take(max_x);
  W->partial = take(max_part);
  W->rgbbuf[0] = take((size_t)B * 3 * size * size * 4);
  W->rgbbuf[1] = take((size_t)B * 3 * size * size * 4);
  W->total = off;
}

}  // namespace hf

using namespace hf;

// Optional per-launch timing of the chain (HF_GEN_PROFILE=1): CUDA events around every conv / rgb_combine
// launch, printed to stderr after a stream sync.  Diagnostic only; off by default.
namespace {
struct ProfRec { char name[16]; int idx, cin, cout, res, up, ntile, halo; cudaEvent_t e0, e1; };
thread_local std::vector<ProfRec> g_prof;
thread_local cudaEvent_t g_prof_e0;
bool prof_on() { static int on = -1; if (on < 0) { const char* v = getenv("HF_GEN_PROFILE"); on = (v && atoi(v)) ? 1 : 0; } return on == 1; }
void prof_begin(cudaStream_t st) { if (!prof_on()) return; cudaEventCreate(&g_prof_e0); cudaEventRecord(g_prof_e0, st); }
void prof_end(cudaStream_t st, const char* name, int idx, int cin, int cout, int res, int up, int ntile, int halo) {
  if (!prof_on()) return;
  ProfRec r; snprintf(r.name, sizeof(r.name), "%s", name);
  r.idx = idx; r.cin = cin; r.cout = cout; r.res = res; r.up = up; r.ntile = ntile; r.halo = halo; r.e0 = g_prof_e0;
  cudaEventCreate(&r.e1); cudaEventRecord(r.e1, st); g_prof.push_back(r);
}
void prof_flush(cudaStream_t st, int B) {
  if (!prof_on()) return;
  cudaStreamSynchronize(st);
  float total = 0.f;
  for (auto& r : g_prof) {
    float ms = 0.f; cudaEventElapsedTime(&ms, r.e0, r.e1); total += ms;
    double gf = (strcmp(r.name, "conv") == 0) ? 2.0 * r.cin * r.cout * 9.0 * r.res * r.res * B * 1e-9 : 0.0;
    fprintf(stderr, "[hf_prof] %-12s #%-2d %4d->%-4d r_in=%-4d up=%d n_tile=%-3d halo=%d  %8.1f us  %7.1f TFLOP/s(alg)\n",
            r.name, r.idx, r.cin, r.cout, r.res, r.up, r.ntile, r.halo, ms * 1e3, gf / (ms * 1e-3) * 1e-3);
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  fprintf(stderr, "[hf_prof] B=%d sum of timed launches %.1f us\n", B, total * 1e3);
  g_prof.clear();
}
}  // namespace

extern "C" {

size_t hf_generator_packed_bytes(const hf_gen_config* cfg) {
  GenLayout L;
  if (make_layout(cfg, &L)) return 0;
  return L.total;
}

size_t hf_generator_workspace_bytes(const hf_gen_config* cfg, int batch) {
  GenLayout L;
  if (make_layout(cfg, &L) || batch <= 0) return 0;
  WsLayout W;
  make_ws(L, batch, cfg->size, &W);
  return W.total;
}

int hf_generator_pack(const hf_gen_config* cfg, const hf_gen_weights* w, void* packed, void* stream) {
  GenLayout L;
  int rc = make_layout(cfg, &L);
  if (rc) return rc;
  if ((rc = ensure_device_current())) return rc;
  HF_REQUIRE(w && packed, "hf_generator_pack: null pointer");
  HF_REQUIRE(((uintptr_t)packed & 255) == 0, "hf_generator_pack: packed buffer must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* P = reinterpret_cast<uint8_t*>(packed);
  const int D = cfg->style_dim;
  HF_REQUIRE(w->const_input, "hf_generator_pack: input.input is null");
  if ((rc = launch_scale_copy(w->const_input, (float*)(P + L.const_in), (int64_t)L.st[0].cin * 16, 1.f, st))) return rc;
  for (int i = 0; i < L.n_styled; ++i) {
    const StyledL& s = L.st[i];
    HF_REQUIRE(w->conv_weight[i] && w->conv_mod_weight[i] && w->conv_mod_bias[i] && w->conv_noise_weight[i] &&
                   w->conv_act_bias[i],
               "hf_generator_pack: styled conv %d has a null parameter", i);
    HF_REQUIRE(!s.up || w->conv_blur_kernel[i], "hf_generator_pack: upsampling conv %d has no blur kernel", i);
    if ((rc = launch_pack_conv(w->conv_weight[i], w->conv_blur_kernel[i], P + s.wpk, (float*)(P + s.wsq), s.cout,
                               s.cin, 3, s.up, 0, cfg->dtype, st)))
      return rc;
    if ((rc = launch_scale_copy(w->conv_mod_weight[i], (float*)(P + s.mw), (int64_t)s.cin * D, 1.f, st))) return rc;
    if ((rc = launch_scale_copy(w->conv_mod_bias[i], (float*)(P + s.mb), s.cin, 1.f, st))) return rc;
    if ((rc = launch_scale_copy(w->conv_noise_weight[i], (float*)(P + s.noise_w), 1, 1.f, st))) return rc;
    if ((rc = launch_scale_copy(w->conv_act_bias[i], (float*)(P + s.act_bias), s.cout, 1.f, st))) return rc;
  }
  for (int i = 0; i < L.n_rgb; ++i) {
    const RgbL& r = L.rgb[i];
    HF_REQUIRE(w->rgb_weight[i] && w->rgb_mod_weight[i] && w->rgb_mod_bias[i] && w->rgb_bias[i],
               "hf_generator_pack: to_rgb %d has a null parameter", i);
    HF_REQUIRE(i == 0 || w->rgb_up_kernel[i], "hf_generator_pack: to_rgb %d has no upsample kernel", i);
    // ModulatedConv2d(k=1).scale = 1/sqrt(cin) folded into the weights (model.py:220-221)
    if ((rc = launch_scale_copy(w->rgb_weight[i], (float*)(P + r.w1), 3 * (int64_t)r.cin, 1.f / sqrtf((float)r.cin), st)))
      return rc;
    if ((rc = launch_scale_copy(w->rgb_mod_weight[i], (float*)(P + r.mw), (int64_t)r.cin * D, 1.f, st))) return rc;
    if ((rc = launch_scale_copy(w->rgb_mod_bias[i], (float*)(P + r.mb), r.cin, 1.f, st))) return rc;
    if ((rc = launch_scale_copy(w->rgb_bias[i], (float*)(P + r.bias), 3, 1.f, st))) return rc;
    if (i > 0)
      if ((rc = launch_scale_copy(w->rgb_up_kernel[i], (float*)(P + r.upk), 16, 1.f, st))) return rc;
  }
  return HF_OK;
}

int hf_generator_forward(const hf_gen_config* cfg, const void* packed, const hf_gen_io* io, void* workspace,
                         int* early_exit, void* stream) {
  GenLayout L;
  int rc = make_layout(cfg, &L);
  if (rc) return rc;
  if ((rc = ensure_device_current())) return rc;
  reset_launch_count();
  HF_REQUIRE(packed && io && workspace, "hf_generator_forward: null pointer");
  HF_REQUIRE(((uintptr_t)packed & 255) == 0 && ((uintptr_t)workspace & 255) == 0,
             "hf_generator_forward: packed / workspace must be 256-byte aligned");
  HF_REQUIRE(io->batch > 0 && io->latent && io->out_rgb, "hf_generator_forward: batch/latent/out_rgb missing");
  const int n = L.n_layers, B = io->batch, D = cfg->style_dim;
  const int start = io->start_layer, end = io->end_layer;
  HF_REQUIRE(start >= 0 && start <= n && end >= 0, "hf_generator_forward: start_layer=%d end_layer=%d out of range (0..%d)",
             start, end, n);
  HF_REQUIRE(start == 0 || io->layer_in, "hf_generator_forward: start_layer=%d needs layer_in (model.py:546)", start);
  HF_REQUIRE(!(start > 0 && end == 0), "hf_generator_forward: start_layer>0 with end_layer=0 is not supported");
  bool any_feat = false;
  for (int i = 0; i < HF_MAX_STYLED; ++i) any_feat |= (io->feature_in[i] != nullptr);
  HF_REQUIRE(!any_feat || io->feature_alpha == 1.0f,
             "hf_generator_forward: insert_feature supports feature_scale == 1 only (got %f)", io->feature_alpha);
  HF_REQUIRE(!io->feature_in[0], "hf_generator_forward: feature_in[0] is never consumed (model.py insert_feature starts at 1)");
  // Which layers run (mirror of the loop at model.py:541-557)
  bool run[16] = {false};
  run[0] = (start == 0);
  int last = run[0] ? 0 : -1;
  if (end != 0)
    for (int k = 1; k <= n; ++k) {
      if (k < start) continue;
      if (k == start) { run[k] = true; last = k; continue; }
      if (k > end) break;
      run[k] = true; last = k;
    }
  HF_REQUIRE(last >= 0, "hf_generator_forward: nothing to execute");
  const bool early = last < n;
  if (early_exit) *early_exit = early ? 1 : 0;
  HF_REQUIRE(!early || io->out_feature, "hf_generator_forward: early exit at layer %d needs out_feature", last);

  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* P = reinterpret_cast<const uint8_t*>(packed);
  uint8_t* Wp = reinterpret_cast<uint8_t*>(workspace);
  WsLayout W;
  make_ws(L, B, cfg->size, &W);
  auto F = [&](size_t off) { return reinterpret_cast<const float*>(P + off); };
  auto WF = [&](size_t off) { return reinterpret_cast<float*>(Wp + off); };
  const int64_t lat_stride = (int64_t)L.n_latent * D;

  // ---- 1. style tables for every executed conv / to_rgb
  AffineJob aj[kMaxJobs];
  DemodJob dj[kMaxJobs];
  int na = 0, nd = 0;
  auto add_styled = [&](int i) {
    aj[na].mw = F(L.st[i].mw); aj[na].mb = F(L.st[i].mb); aj[na].style = io->latent + (size_t)i * D;
    aj[na].s = WF(W.s_conv[i]); aj[na].C = L.st[i].cin; aj[na].wscale = 1.f / sqrtf((float)D); ++na;
    dj[nd].wsq = F(L.st[i].wsq); dj[nd].s = WF(W.s_conv[i]); dj[nd].d = WF(W.d_conv[i]);
    dj[nd].Cout = L.st[i].cout; dj[nd].Cin = L.st[i].cin; ++nd;
  };
  auto add_rgb = [&](int k) {
    aj[na].mw = F(L.rgb[k].mw); aj[na].mb = F(L.rgb[k].mb); aj[na].style = io->latent + (size_t)(2 * k + 1) * D;
    aj[na].s = WF(W.s_rgb[k]); aj[na].C = L.rgb[k].cin; aj[na].wscale = 1.f / sqrtf((float)D); ++na;
  };
  for (int k = 0; k <= n; ++k) {
    if (!run[k]) continue;
    if (k == 0) add_styled(0); else { add_styled(2 * k - 1); add_styled(2 * k); }
    add_rgb(k);
  }
  if ((rc = launch_affine(aj, na, B, D, lat_stride, st))) return rc;
  if ((rc = launch_demod(dj, nd, B, st))) return rc;

  // ---- 2. chain
  int cur = 0;                               // which xbuf holds the current conv input
  const float* skip = nullptr;               // running RGB (fp32 NCHW at the previous resolution)
  int rgb_slot = 0;
  auto xb = [&](int i) { return (void*)(Wp + W.xbuf[i]); };

  auto run_conv = [&](int i, const void* xin, void* xout, const float* s_next, float* out_nchw, int rgb_k,
                      int* num_nt) -> int {
    const StyledL& s = L.st[i];
    ConvLaunch cl;
    memset(&cl, 0, sizeof(cl));
    cl.B = B; cl.H = s.res_in; cl.W = s.res_in; cl.Cin = s.cin; cl.Cout = s.cout; cl.taps = 9; cl.up = s.up;
    cl.dtype = cfg->dtype;
    cl.xhat_in = xin; cl.wpk = P + s.wpk;
    cl.d = WF(W.d_conv[i]);
    HF_REQUIRE(io->noise[i], "hf_generator_forward: noise[%d] is null (the host must draw it, model.py:288-291)", i);
    HF_REQUIRE(io->noise_batch[i] == 1 || io->noise_batch[i] == B, "hf_generator_forward: noise_batch[%d]=%d", i,
               io->noise_batch[i]);
    cl.noise = io->noise[i]; cl.noise_batch = io->noise_batch[i]; cl.noise_w = F(s.noise_w);
    cl.bias = F(s.act_bias); cl.act = 1;
    cl.s_next = s_next; cl.xhat_out = xout;
    cl.out_nchw = io->features_out[i + 1] ? io->features_out[i + 1] : out_nchw;    // return_features
    if (rgb_k >= 0) {
      cl.rgb_w = F(L.rgb[rgb_k].w1); cl.rgb_s = WF(W.s_rgb[rgb_k]); cl.rgb_partial = WF(W.partial);
    }
    ConvPlan pl;
    prof_begin(st);
    int r = launch_conv(cl, st, &pl);
    prof_end(st, "conv", i, s.cin, s.cout, s.res_in, s.up, pl.n_tile, pl.halo);
    if (num_nt) *num_nt = pl.num_n_tiles;
    return r;
  };
  auto combine = [&](int k, int num_nt, const float* skip_in, float* dst) -> int {
    const RgbL& r = L.rgb[k];
    prof_begin(st);
    int rr = launch_rgb_combine(WF(W.partial), num_nt, F(r.bias), skip_in, skip_in ? F(r.upk) : nullptr, dst, B,
                                r.res, r.res, st);
    prof_end(st, "rgb_combine", k, r.cin, 3, r.res, 0, num_nt, 0);
    return rr;
  };
  auto rgb_dst = [&](int k) -> float* {
    if (k == last) return io->out_rgb;
    rgb_slot ^= 1;
    return WF(W.rgbbuf[rgb_slot]);
  };

  if (io->features_out[0])
    for (int b = 0; b < B; ++b)
      if ((rc = launch_scale_copy(F(L.const_in), io->features_out[0] + (size_t)b * L.st[0].cin * 16,
                                  (int64_t)L.st[0].cin * 16, 1.f, st)))
        return rc;
  if (run[0]) {
    if ((rc = launch_modulate_to_nhwc(F(L.const_in), 1, WF(W.s_conv[0]), nullptr, 0.f, xb(cur), B, L.st[0].cin, 16,
                                      cfg->dtype, st)))
      return rc;
    const bool more = (last > 0);
    int nt = 0;
    if ((rc = run_conv(0, xb(cur), more ? xb(cur ^ 1) : nullptr, more ? WF(W.s_conv[1]) : nullptr,
                       (!more && early) ? io->out_feature : nullptr, 0, &nt)))
      return rc;
    cur ^= 1;
    float* dst = rgb_dst(0);
    if ((rc = combine(0, nt, nullptr, dst))) return rc;
    skip = dst;
  } else {
    skip = io->skip_in;
  }
  for (int k = 1; k <= n; ++k) {
    if (!run[k]) continue;
    const int iu = 2 * k - 1, ic = 2 * k;
    if (k == start || io->feature_in[iu]) {
      // layer_in (model.py:546) or the FSE feature insertion (alpha == 1): fresh NCHW fp32 input
      const float* src = io->feature_in[iu] ? io->feature_in[iu] : io->layer_in;
      if ((rc = launch_modulate_to_nhwc(src, 0, WF(W.s_conv[iu]), nullptr, 0.f, xb(cur), B, L.st[iu].cin,
                                        L.st[iu].res_in * L.st[iu].res_in, cfg->dtype, st)))
        return rc;
    }
    if ((rc = run_conv(iu, xb(cur), xb(cur ^ 1), WF(W.s_conv[ic]), nullptr, -1, nullptr))) return rc;
    cur ^= 1;
    if (io->feature_in[ic])      // insert_feature before the second conv of the layer
      if ((rc = launch_modulate_to_nhwc(io->feature_in[ic], 0, WF(W.s_conv[ic]), nullptr, 0.f, xb(cur), B,
                                        L.st[ic].cin, L.st[ic].res_in * L.st[ic].res_in, cfg->dtype, st)))
        return rc;
    const bool more = (k < last);
    int nt = 0;
    if ((rc = run_conv(ic, xb(cur), more ? xb(cur ^ 1) : nullptr, more ? WF(W.s_conv[ic + 1]) : nullptr,
                       (!more && early) ? io->out_feature : nullptr, k, &nt)))
      return rc;
    cur ^= 1;
    float* dst = rgb_dst(k);
    if ((rc = combine(k, nt, skip, dst))) return rc;
    skip = dst;
  }
  prof_flush(st, B);
  return HF_OK;
}

}  // extern "C"
