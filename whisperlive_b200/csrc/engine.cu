// libwlb200 engine: context, weights, encoder (K2-K7), decoder loop (K8-K13), alignment (K14) and their C ABI
// (include/wlb200.h).  Silero VAD, speaker embeddings and the kernel test hooks are in vad_engine.cu, spk_engine.cu and
// hooks.cu.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>

#include "ctx.cuh"

namespace wl {
void gemm_prime();
void attention_prime();
void search_prime();
void flash_attn_prime();
long other_launch_count();
void gemm_tl_bind(unsigned long long* p);
void attention_tl_bind(unsigned long long* p);
void elementwise_tl_bind(unsigned long long* p);
void search_tl_bind(unsigned long long* p);
}  // namespace wl

static std::string g_init_error;

// Rows of the per-stream metadata table of a decode call (stream_meta / search_meta -> upload_state_tables):
// slot, len, sot_index, use_ts, n_new, force_len, pre_n, pre_last, pre_penult, pre_lts, then the stream's search:
// smode, temperature (float bits), noise seed, noise key, rows
constexpr int META_ROWS = 15;

// Everything a context owns on the device and the host, and the context itself: wl_destroy, and wl_init when it
// fails part-way.
static void free_ctx(wl_ctx* c) {
  if (c->st || !c->mem.list.empty()) cudaSetDevice(c->mem.device);
  if (c->st) cudaStreamSynchronize(c->st);
  for (auto& g : c->graphs)
    if (g.second.exec) cudaGraphExecDestroy(g.second.exec);
  c->mem.release_from(0);
  if (c->h_int) cudaFreeHost(c->h_int);
  if (c->h_flt) cudaFreeHost(c->h_flt);
  if (c->ev0) cudaEventDestroy(c->ev0);
  if (c->ev1) cudaEventDestroy(c->ev1);
  if (c->pev0) cudaEventDestroy(c->pev0);
  if (c->pev1) cudaEventDestroy(c->pev1);
  for (cudaEvent_t e : c->vad.ev)
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : c->spk.ev)
    if (e) cudaEventDestroy(e);
  if (c->st) cudaStreamDestroy(c->st);
  delete c;
}

static void ensure_host(wl_ctx* c, size_t n_int, size_t n_flt) {
  if (n_int > c->h_int_cap) {
    if (c->h_int) cudaFreeHost(c->h_int);
    WL_CUDA(cudaMallocHost((void**)&c->h_int, n_int * sizeof(int)));
    c->h_int_cap = n_int;
  }
  if (n_flt > c->h_flt_cap) {
    if (c->h_flt) cudaFreeHost(c->h_flt);
    WL_CUDA(cudaMallocHost((void**)&c->h_flt, n_flt * sizeof(float)));
    c->h_flt_cap = n_flt;
  }
}

// device-resident decode state for Bm streams x Km rows (one per context, plus one per decode session)
static void alloc_decode_state(wl_ctx* c, DecodeState& s) {
  const size_t R = c->Rm, B = c->Bm;
  s.tok_in = c->mem.alloc<int>(R); s.pos = c->mem.alloc<int>(R); s.active = c->mem.alloc<int>(R); s.cum = c->mem.alloc<float>(R);
  s.gen_len = c->mem.alloc<int>(R); s.last_ts = c->mem.alloc<int>(R); s.row_done = c->mem.alloc<int>(R);
  s.hist = c->mem.alloc<int>(R * T_MAX); s.src = c->mem.alloc<short>(R * T_MAX);
  s.cand_val = c->mem.alloc<float>(R * MAX_CAND); s.cand_tok = c->mem.alloc<int>(R * MAX_CAND);
  s.nospeech_row = c->mem.alloc<float>(R);
  s.slot = c->mem.alloc<int>(B); s.prompt = c->mem.alloc<int>(B * T_MAX); s.prompt_len = c->mem.alloc<int>(B);
  s.fed = c->mem.alloc<int>(B); s.sot_index = c->mem.alloc<int>(B); s.use_ts = c->mem.alloc<int>(B); s.n_new = c->mem.alloc<int>(B);
  s.step = c->mem.alloc<int>(B); s.done = c->mem.alloc<int>(B); s.n_alive = c->mem.alloc<int>(B); s.no_speech = c->mem.alloc<float>(B);
  s.hyp_count = c->mem.alloc<int>(B); s.hyp_cum = c->mem.alloc<float>(B * MAX_HYPS); s.hyp_len = c->mem.alloc<int>(B * MAX_HYPS);
  s.hyp_tok = c->mem.alloc<int>(B * MAX_HYPS * T_MAX); s.steps_run = c->mem.alloc<int>(B); s.n_done = c->mem.alloc<int>(1);
  s.force_len = c->mem.alloc<int>(B); s.force_prob = c->mem.alloc<float>(B * T_MAX);
  s.steps_left = c->mem.alloc<int>(1);
  s.smode = c->mem.alloc<int>(B); s.temp = c->mem.alloc<float>(B); s.nseed = c->mem.alloc<unsigned>(B); s.nkey = c->mem.alloc<int>(B);
  s.nrows = c->mem.alloc<int>(B);
  s.pre_n = c->mem.alloc<int>(B); s.pre_last = c->mem.alloc<int>(B); s.pre_penult = c->mem.alloc<int>(B); s.pre_lts = c->mem.alloc<int>(B);
  s.brk = c->mem.alloc<int>(2);
  s.r_max_initial = s.r_suppress_blank = s.r_max_cand = s.r_beam = nullptr;   // the call's SearchOpts (a session adds its own)
  s.r_length_penalty = nullptr;
  s.r_mask = nullptr;
  s.mask_words = 0;
}

// Rows of a decode session's per-stream rule table (host shadow Session::rules -> DecodeState::r_*): max initial
// timestamp index, suppress_blank, max_cand, length penalty (float bits), beam width
constexpr int RULE_ROWS = 5;

// ------------------------------------------------------------------------------------------ init
extern "C" int wl_init(const wl_config* cfg, wl_ctx** out) {
  if (!cfg || !out) return WL_ERR_ARG;
  wl_ctx* c = new wl_ctx();
  try {
    WL_CHECK(cfg->abi_version == WL_ABI_VERSION, WL_ERR_ARG, "ABI version mismatch: header %d, caller %d", WL_ABI_VERSION,
             cfg->abi_version);
    c->cfg = *cfg;
    c->align_heads.assign(cfg->align_heads, cfg->align_heads + 2 * cfg->n_align_heads);
    c->cfg.align_heads = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    WL_CHECK(e == cudaSuccess && ndev > 0, WL_ERR_CUDA, "no CUDA device available (%s): libwlb200 has no CPU fallback",
             cudaGetErrorString(e));
    WL_CHECK(cfg->device >= 0 && cfg->device < ndev, WL_ERR_ARG, "device %d out of range (%d devices)", cfg->device, ndev);
    WL_CUDA(cudaSetDevice(cfg->device));
    c->mem.device = cfg->device;
    cudaDeviceProp prop;
    WL_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    WL_CHECK(prop.major == 9 && prop.minor == 0, WL_ERR_CUDA, "libwlb200 is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
    c->num_sms = prop.multiProcessorCount;
    c->d = cfg->d_model; c->H = cfg->n_heads; c->Le = cfg->enc_layers; c->Ld = cfg->dec_layers;
    c->n_mels = cfg->n_mels; c->V = cfg->vocab; c->Vld = (cfg->vocab + 3) / 4 * 4;
    c->Bm = cfg->max_streams; c->Km = cfg->max_beam; c->Rm = c->Bm * c->Km; c->NS = cfg->enc_slots;
    WL_CHECK(c->d % 64 == 0 && c->H * 64 == c->d && c->d <= 1280, WL_ERR_ARG, "d_model %d / heads %d unsupported", c->d, c->H);
    WL_CHECK(c->n_mels % 8 == 0 && c->n_mels <= 128, WL_ERR_ARG, "n_mels %d unsupported", c->n_mels);
    WL_CHECK(c->Km >= 1 && c->Km <= MAX_ROWS_PER_STREAM, WL_ERR_ARG, "max_beam %d must be in [1,%d]", c->Km, MAX_ROWS_PER_STREAM);
    WL_CHECK(c->Bm >= 1 && c->NS >= c->Bm, WL_ERR_ARG, "enc_slots %d must be >= max_streams %d", c->NS, c->Bm);
    WL_CUDA(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    c->mem.st = c->st;
    WL_CUDA(cudaEventCreate(&c->ev0));
    WL_CUDA(cudaEventCreate(&c->ev1));
    gemm_prime();
    dec_gemm_prime();
    wgemm_prime();
    attention_prime();
    search_prime();
    flash_attn_prime();
    if (const char* tl = getenv("WLB200_TIMELINE")) {
      c->tl_path = tl;
      c->tl_dev = c->mem.alloc<unsigned long long>(TL_CAP + 1);
      gemm_tl_bind(c->tl_dev); dec_gemm_tl_bind(c->tl_dev); wgemm_tl_bind(c->tl_dev); attention_tl_bind(c->tl_dev); elementwise_tl_bind(c->tl_dev); search_tl_bind(c->tl_dev);
    }
    c->enc.resize(c->Le);
    c->dec.resize(c->Ld);
    for (int i = c->NS - 1; i >= 0; --i) c->slot_free.push_back(i);
    c->slot_used.assign(c->NS, 0);
  } catch (const wl::Error& e) {
    // a failed init frees the stream, the events and the timeline buffer it had made: nothing stays on the device
    g_init_error = e.msg;
    free_ctx(c);
    return e.code;
  }
  *out = c;
  return WL_OK;
}

extern "C" void wl_destroy(wl_ctx* c) {
  if (!c) return;
  free_ctx(c);
}

extern "C" int wl_device_bytes(wl_ctx* c, int64_t* out) {
  if (!c || !out) return WL_ERR_ARG;
  *out = c->mem.bytes;
  return WL_OK;
}

// The query runs on a thread of its own, so the caller's current device is never touched: restoring it with
// cudaSetDevice would create a context on a device the caller never used (cudaGetDevice reports 0 on a fresh thread).
// Only the queried device's primary context is initialised -- the device a model is about to be loaded on.
extern "C" int wl_mem_info(int32_t device, int64_t* free_out, int64_t* total_out) {
  if (!free_out || !total_out) return WL_ERR_ARG;
  size_t fr = 0, tot = 0;
  cudaError_t e = cudaSuccess;
  std::thread q([&] {
    e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaMemGetInfo(&fr, &tot);
    if (e != cudaSuccess) cudaGetLastError();
  });
  q.join();
  if (e != cudaSuccess) {
    g_init_error = std::string("wl_mem_info(") + std::to_string(device) + "): " + cudaGetErrorString(e);
    return WL_ERR_CUDA;
  }
  *free_out = (int64_t)fr;
  *total_out = (int64_t)tot;
  return WL_OK;
}

extern "C" const char* wl_last_error(wl_ctx* c) { return c ? c->err.c_str() : g_init_error.c_str(); }
extern "C" int64_t wl_kernel_launches(wl_ctx* c) {
  return c ? gemm_launch_count() + dec_gemm_launch_count() + wgemm_launch_count() + other_launch_count() - c->capture_counted + c->graph_launched : 0;
}
extern "C" float wl_last_device_ms(wl_ctx* c, int32_t which) {
  if (!c) return -1.f;
  if (which == 3) return c->prof_cross_n > 0 ? (float)(c->prof_cross_ms / (double)c->prof_cross_n) : -1.f;   // avg ms per cross-attention launch
  if (which == 4) return (float)c->prof_cross_n;
  if (which >= 0 && which < 10) return c->last_ms[which];   // the calls wl_ctx::last_ms lists
  return -1.f;
}
extern "C" int wl_profile_cross_attn(wl_ctx* c, int32_t enable) {
  API_BEGIN(c)
  if (enable && !c->pev0) {
    WL_CUDA(cudaEventCreate(&c->pev0));
    WL_CUDA(cudaEventCreate(&c->pev1));
  }
  c->prof_cross = enable ? 1 : 0;
  c->prof_cross_ms = 0.0;
  c->prof_cross_n = 0;
  API_END(c)
}

// ------------------------------------------------------------------------------------------ weights
extern "C" int wl_load_tensor(wl_ctx* c, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  API_BEGIN(c)
  WL_CHECK(name && data && shape && ndim >= 1 && ndim <= 3, WL_ERR_ARG, "wl_load_tensor: bad arguments");
  WL_CHECK(!c->finalized, WL_ERR_STATE, "weights already finalized");
  std::string nm(name);
  size_t n = 1;
  std::vector<int64_t> sh(shape, shape + ndim);
  for (auto s : sh) n *= (size_t)s;
  const bool as_f32 = ndim == 1 || nm == "model.encoder.embed_positions.weight" || nm == "mel_filters";
  if (as_f32) {
    float* p = c->mem.alloc<float>(n, false);
    WL_CUDA(cudaMemcpy(p, data, n * sizeof(float), cudaMemcpyHostToDevice));
    c->dev[nm] = p;
  } else {
    // fp32 -> fp16 (and the conv re-layout) on the device: the host only hands over its buffer.  A large-v3 load
    // is 1.5 G values; converting them on one host thread took longer than everything else in wl_init together.
    c->mem.grow(c->stage_f32, c->stage_cap, (long)n);
    WL_CUDA(cudaMemcpyAsync(c->stage_f32, data, n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    __half* p = c->mem.alloc<__half>(n, false);
    if (ndim == 3) cast_weight_f16(c->st, c->stage_f32, p, sh[0], sh[1], sh[2]);   // [co][ci][k] -> [co][k][ci]
    else cast_weight_f16(c->st, c->stage_f32, p, (long)n, 1, 1);
    WL_CUDA(cudaStreamSynchronize(c->st));
    c->dev[nm] = p;
  }
  c->shape[nm] = sh;
  API_END(c)
}

static_assert(WL_DT_F32 == WDT_F32 && WL_DT_F16 == WDT_F16 && WL_DT_BF16 == WDT_BF16 && WL_DT_I8 == WDT_I8,
              "wlb200.h and kernels.cuh disagree on the weight dtypes");

// The bytes go to the device as stored (half the PCIe traffic of wl_load_tensor for an fp16 checkpoint, a quarter
// for int8) and are converted there.  One byte staging buffer holds [overflow count | payload | scales], each part
// 256-byte aligned so the conversion kernels read it 16 bytes at a time.
extern "C" int wl_load_tensor_typed(wl_ctx* c, const char* name, const void* data, int32_t dtype, const int64_t* shape,
                                    int32_t ndim, const void* scale, int32_t scale_dtype) {
  API_BEGIN(c)
  WL_CHECK(name && data && shape && ndim >= 1 && ndim <= 3, WL_ERR_ARG, "wl_load_tensor_typed: bad arguments");
  WL_CHECK(dtype >= WL_DT_F32 && dtype <= WL_DT_I8, WL_ERR_ARG, "wl_load_tensor_typed(%s): unknown dtype %d", name, dtype);
  WL_CHECK(dtype != WL_DT_I8 || (scale && scale_dtype >= WL_DT_F32 && scale_dtype <= WL_DT_BF16), WL_ERR_ARG,
           "wl_load_tensor_typed(%s): int8 needs a float32 / float16 / bfloat16 scale per row", name);
  WL_CHECK(!c->finalized, WL_ERR_STATE, "weights already finalized");
  std::string nm(name);
  size_t n = 1;
  std::vector<int64_t> sh(shape, shape + ndim);
  for (auto s : sh) {
    WL_CHECK(s > 0, WL_ERR_ARG, "wl_load_tensor_typed(%s): empty dimension", name);
    n *= (size_t)s;
  }
  static const size_t esize[4] = {4, 2, 2, 1};
  const size_t rows = (size_t)sh[0], cols = n / rows;
  const size_t pay = esize[dtype] * n, sc = dtype == WL_DT_I8 ? esize[scale_dtype] * rows : 0;
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t off_data = 256, off_scale = off_data + up(pay), total = off_scale + up(sc);
  c->mem.grow(c->stage_bytes, c->stage_bytes_cap, (long)total);
  unsigned char* s = c->stage_bytes;
  int* overflow = (int*)s;
  WL_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), c->st));
  WL_CUDA(cudaMemcpyAsync(s + off_data, data, pay, cudaMemcpyHostToDevice, c->st));
  if (sc) WL_CUDA(cudaMemcpyAsync(s + off_scale, scale, sc, cudaMemcpyHostToDevice, c->st));
  const void* dscale = sc ? (const void*)(s + off_scale) : nullptr;
  const bool as_f32 = ndim == 1 || nm == "model.encoder.embed_positions.weight" || nm == "mel_filters";
  void* p;
  if (as_f32) {
    float* q = c->mem.alloc<float>(n, false);
    convert_weight_f32(c->st, s + off_data, dtype, dscale, scale_dtype, q, (long)n, (long)cols, overflow, c->num_sms);
    p = q;
  } else {
    __half* q = c->mem.alloc<__half>(n, false);
    if (ndim == 3) convert_weight_f16(c->st, s + off_data, dtype, dscale, scale_dtype, q, sh[0], sh[1], sh[2], (long)cols, overflow, c->num_sms);
    else convert_weight_f16(c->st, s + off_data, dtype, dscale, scale_dtype, q, (long)n, 1, 1, (long)cols, overflow, c->num_sms);
    p = q;
  }
  int n_over = 0;
  WL_CUDA(cudaMemcpyAsync(&n_over, overflow, sizeof(int), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaStreamSynchronize(c->st));
  if (n_over) {
    c->mem.release(p);
    WL_CHECK(false, WL_ERR_ARG, "weight '%s': %d finite values exceed the float16 range (|x| > 65504)", name, n_over);
  }
  c->dev[nm] = p;
  c->shape[nm] = sh;
  API_END(c)
}

static void* need(wl_ctx* c, const std::string& nm, std::initializer_list<int64_t> want) {
  auto it = c->dev.find(nm);
  WL_CHECK(it != c->dev.end(), WL_ERR_STATE, "missing weight tensor '%s'", nm.c_str());
  const auto& sh = c->shape[nm];
  std::vector<int64_t> w(want);
  WL_CHECK(sh == w, WL_ERR_ARG, "weight '%s' has the wrong shape", nm.c_str());
  return it->second;
}
static __half* concat_h(wl_ctx* c, std::vector<std::pair<__half*, size_t>> parts) {
  size_t tot = 0;
  for (auto& p : parts) tot += p.second;
  __half* out = c->mem.alloc<__half>(tot, false);
  size_t o = 0;
  for (auto& p : parts) {
    WL_CUDA(cudaMemcpy(out + o, p.first, p.second * sizeof(__half), cudaMemcpyDeviceToDevice));
    o += p.second;
  }
  return out;
}
static float* concat_f(wl_ctx* c, std::vector<std::pair<float*, size_t>> parts) {
  size_t tot = 0;
  for (auto& p : parts) tot += p.second;
  float* out = c->mem.alloc<float>(tot, true);
  size_t o = 0;
  for (auto& p : parts) {
    if (p.first) WL_CUDA(cudaMemcpy(out + o, p.first, p.second * sizeof(float), cudaMemcpyDeviceToDevice));
    o += p.second;
  }
  return out;
}

static void build_mel_tables(wl_ctx* c) {
  std::vector<float> win(400), tw(800);
  const double PI = 3.14159265358979323846;
  for (int i = 0; i < 400; ++i) {
    win[i] = (float)(0.5 - 0.5 * cos(2.0 * PI * i / 400.0));
    tw[2 * i] = (float)cos(2.0 * PI * i / 400.0);
    tw[2 * i + 1] = (float)sin(2.0 * PI * i / 400.0);
  }
  c->mel_window = c->mem.alloc<float>(400);
  c->mel_twiddle = c->mem.alloc<float>(800);
  WL_CUDA(cudaMemcpy(c->mel_window, win.data(), 400 * 4, cudaMemcpyHostToDevice));
  WL_CUDA(cudaMemcpy(c->mel_twiddle, tw.data(), 800 * 4, cudaMemcpyHostToDevice));
  c->mel_filt = (float*)need(c, "mel_filters", {c->n_mels, 201});
  std::vector<float> f((size_t)c->n_mels * 201);
  WL_CUDA(cudaMemcpy(f.data(), c->mel_filt, f.size() * 4, cudaMemcpyDeviceToHost));
  std::vector<int> rg(2 * c->n_mels);
  for (int m = 0; m < c->n_mels; ++m) {
    int lo = 201, hi = 0;
    for (int k = 0; k < 201; ++k)
      if (f[(size_t)m * 201 + k] != 0.f) { lo = std::min(lo, k); hi = std::max(hi, k + 1); }
    if (lo > hi) lo = hi = 0;
    rg[2 * m] = lo; rg[2 * m + 1] = hi;
  }
  c->mel_range = c->mem.alloc<int>(rg.size());
  WL_CUDA(cudaMemcpy(c->mel_range, rg.data(), rg.size() * 4, cudaMemcpyHostToDevice));
  c->mel_gmax = c->mem.alloc<unsigned>(c->Bm);
  c->res_off = c->mem.alloc<long>(c->Bm + 1);
  c->res_ooff = c->mem.alloc<long>(c->Bm + 1);
  c->res_frames = c->mem.alloc<int>(c->Bm);
  c->win_meta = c->mem.alloc<int>(3 * (size_t)c->Bm);
  c->mel_off = c->mem.alloc<long>(c->Bm + 1);
  c->mel_ooff = c->mem.alloc<long>(c->Bm + 1);
}

static void finalize_impl(wl_ctx* c);

// streams per sub-pass of the unfused encoder attention: the fp32 scores of one stream are H x 1500 x 1536 floats
int enc_attn_streams(int d) { return d >= 1024 ? 2 : 4; }

// The weight-load staging buffer is freed first.  A finalize that fails part-way (a missing tensor, an out-of-memory
// workspace) frees every buffer it had allocated before it returns: only the tensors wl_load_tensor uploaded remain,
// until wl_destroy.
extern "C" int wl_finalize_weights(wl_ctx* c) {
  API_BEGIN(c)
  WL_CHECK(!c->finalized, WL_ERR_STATE, "weights already finalized");
  c->mem.release(c->stage_f32);
  c->stage_cap = 0;
  c->mem.release(c->stage_bytes);
  c->stage_bytes_cap = 0;
  const size_t mark = c->mem.list.size();
  try {
    finalize_impl(c);
  } catch (...) {
    c->mem.release_from(mark);
    throw;
  }
  API_END(c)
}

static void finalize_impl(wl_ctx* c) {
  const int64_t d = c->d, ff = 4 * c->d, nm = c->n_mels, V = c->V;
  const size_t dd = (size_t)d * d;
  const std::string E = "model.encoder.", D = "model.decoder.";
  c->w_conv1 = (__half*)need(c, E + "conv1.weight", {d, nm, 3});
  c->b_conv1 = (float*)need(c, E + "conv1.bias", {d});
  c->w_conv2 = (__half*)need(c, E + "conv2.weight", {d, d, 3});
  c->b_conv2 = (float*)need(c, E + "conv2.bias", {d});
  c->pos_enc = (float*)need(c, E + "embed_positions.weight", {S_ENC, d});
  c->lnp_g = (float*)need(c, E + "layer_norm.weight", {d});
  c->lnp_b = (float*)need(c, E + "layer_norm.bias", {d});
  for (int l = 0; l < c->Le; ++l) {
    const std::string p = E + "layers." + std::to_string(l) + ".";
    EncLayer& L = c->enc[l];
    L.w_qk = concat_h(c, {{(__half*)need(c, p + "self_attn.q_proj.weight", {d, d}), dd},
                          {(__half*)need(c, p + "self_attn.k_proj.weight", {d, d}), dd}});
    L.b_qk = concat_f(c, {{(float*)need(c, p + "self_attn.q_proj.bias", {d}), (size_t)d}, {nullptr, (size_t)d}});
    L.w_v = (__half*)need(c, p + "self_attn.v_proj.weight", {d, d});
    L.b_v = (float*)need(c, p + "self_attn.v_proj.bias", {d});
    L.w_o = (__half*)need(c, p + "self_attn.out_proj.weight", {d, d});
    L.b_o = (float*)need(c, p + "self_attn.out_proj.bias", {d});
    L.ln1_g = (float*)need(c, p + "self_attn_layer_norm.weight", {d});
    L.ln1_b = (float*)need(c, p + "self_attn_layer_norm.bias", {d});
    L.w_fc1 = (__half*)need(c, p + "fc1.weight", {ff, d});
    L.b_fc1 = (float*)need(c, p + "fc1.bias", {ff});
    L.w_fc2 = (__half*)need(c, p + "fc2.weight", {d, ff});
    L.b_fc2 = (float*)need(c, p + "fc2.bias", {d});
    L.ln2_g = (float*)need(c, p + "final_layer_norm.weight", {d});
    L.ln2_b = (float*)need(c, p + "final_layer_norm.bias", {d});
  }
  c->emb = (__half*)need(c, D + "embed_tokens.weight", {V, d});
  c->pos_dec = (__half*)need(c, D + "embed_positions.weight", {T_MAX, d});
  c->lnf_g = (float*)need(c, D + "layer_norm.weight", {d});
  c->lnf_b = (float*)need(c, D + "layer_norm.bias", {d});
  for (int l = 0; l < c->Ld; ++l) {
    const std::string p = D + "layers." + std::to_string(l) + ".";
    DecLayer& L = c->dec[l];
    L.w_qkv = concat_h(c, {{(__half*)need(c, p + "self_attn.q_proj.weight", {d, d}), dd},
                           {(__half*)need(c, p + "self_attn.k_proj.weight", {d, d}), dd},
                           {(__half*)need(c, p + "self_attn.v_proj.weight", {d, d}), dd}});
    L.b_qkv = concat_f(c, {{(float*)need(c, p + "self_attn.q_proj.bias", {d}), (size_t)d},
                           {nullptr, (size_t)d},
                           {(float*)need(c, p + "self_attn.v_proj.bias", {d}), (size_t)d}});
    L.w_o = (__half*)need(c, p + "self_attn.out_proj.weight", {d, d});
    L.b_o = (float*)need(c, p + "self_attn.out_proj.bias", {d});
    L.ln1_g = (float*)need(c, p + "self_attn_layer_norm.weight", {d});
    L.ln1_b = (float*)need(c, p + "self_attn_layer_norm.bias", {d});
    L.w_qc = (__half*)need(c, p + "encoder_attn.q_proj.weight", {d, d});
    L.b_qc = (float*)need(c, p + "encoder_attn.q_proj.bias", {d});
    L.w_kc = (__half*)need(c, p + "encoder_attn.k_proj.weight", {d, d});
    L.w_vc = (__half*)need(c, p + "encoder_attn.v_proj.weight", {d, d});
    L.b_vc = (float*)need(c, p + "encoder_attn.v_proj.bias", {d});
    L.w_oc = (__half*)need(c, p + "encoder_attn.out_proj.weight", {d, d});
    L.b_oc = (float*)need(c, p + "encoder_attn.out_proj.bias", {d});
    L.ln2_g = (float*)need(c, p + "encoder_attn_layer_norm.weight", {d});
    L.ln2_b = (float*)need(c, p + "encoder_attn_layer_norm.bias", {d});
    L.w_fc1 = (__half*)need(c, p + "fc1.weight", {ff, d});
    L.b_fc1 = (float*)need(c, p + "fc1.bias", {ff});
    L.w_fc2 = (__half*)need(c, p + "fc2.weight", {d, ff});
    L.b_fc2 = (float*)need(c, p + "fc2.bias", {d});
    L.ln3_g = (float*)need(c, p + "final_layer_norm.weight", {d});
    L.ln3_b = (float*)need(c, p + "final_layer_norm.bias", {d});
  }
  build_mel_tables(c);

  // ---- encoder workspaces (EB streams per pass, AB streams per attention sub-pass)
  const int H = c->H;
  // streams per encoder pass: 16 x 1500 = 24000 rows give the GEMMs many full tile waves on 132 SMs; the workspaces are
  // ~1 GB at large-v3, small next to 80 GB
  static const int enc_batch = [] { const char* e = getenv("WLB200_ENC_BATCH"); return e ? std::max(1, atoi(e)) : 16; }();
  c->EB = std::min(c->Bm, enc_batch);
  c->AB = std::min(c->EB, enc_attn_streams(d));
  const size_t M = (size_t)c->EB * S_ENC;
  c->feat32 = c->mem.alloc<float>((size_t)c->Bm * nm * 3000);  // all streams of a call stay resident (wl_encode_resident)
  c->feat16 = c->mem.alloc<__half>((size_t)c->EB * 3002 * nm + 4096);
  c->conv1o = c->mem.alloc<__half>((size_t)c->EB * 3002 * d + 4096);
  c->x = c->mem.alloc<float>(M * d);
  c->xn = c->mem.alloc<__half>(M * d);
  c->qk = c->mem.alloc<__half>(M * 2 * d);
  c->vt = c->mem.alloc<__half>((size_t)c->EB * d * S_PAD);
  c->scores = c->mem.alloc<float>((size_t)c->AB * H * S_ENC * S_PAD);
  c->probs16 = c->mem.alloc<__half>((size_t)c->AB * H * S_ENC * S_PAD);
  c->attn = c->mem.alloc<__half>(M * d);
  c->hbuf = c->mem.alloc<__half>(M * ff);
  c->enc_slots_dev = c->mem.alloc<int>(c->Bm);
  // ---- slot pool
  c->enc16 = c->mem.alloc<__half>((size_t)c->NS * S_ENC * d, false);
  c->ckv = c->mem.alloc<__half>((size_t)c->Ld * 2 * c->NS * S_ENC * d, false);
  // ---- decoder workspaces
  const size_t R = c->Rm, Rp = (R + 15) / 16 * 16;
  c->dx = c->mem.alloc<float>(R * d);
  // split-K partial sums: up to 16 K ranges of a d-wide output, 4 of the 3d-wide QKV, 3 of the 4d-wide MLP
  c->part1 = c->mem.alloc<float>(R * 16 * (size_t)d + R * 4 * (size_t)ff);
  c->part2 = c->mem.alloc<float>(R * 16 * (size_t)d);
  c->logits = c->mem.alloc<float>(R * c->Vld);
  c->dxn = c->mem.alloc<__half>(Rp * d);
  c->datt = c->mem.alloc<__half>(Rp * d);
  c->dh = c->mem.alloc<__half>(Rp * ff);
  c->cache_row_stride = (long)H * T_MAX * 64;
  c->cache_layer_stride = (long)R * c->cache_row_stride;
  c->kcache = c->mem.alloc<__half>((size_t)c->Ld * c->cache_layer_stride, false);
  c->vcache = c->mem.alloc<__half>((size_t)c->Ld * c->cache_layer_stride, false);
  c->xws.part = c->mem.alloc<float>((size_t)c->Bm * H * 12 * MAX_ROWS_PER_STREAM * 66);
  c->xws.probs = nullptr;
  c->suppress_mask = c->mem.alloc<unsigned>((V + 31) / 32 + 1);
  if (!c->align_heads.empty()) {
    c->align_heads_dev = c->mem.alloc<int>(c->align_heads.size());
    WL_CUDA(cudaMemcpy(c->align_heads_dev, c->align_heads.data(), c->align_heads.size() * 4, cudaMemcpyHostToDevice));
  }
  alloc_decode_state(c, c->ds);
  WL_CUDA(cudaDeviceSynchronize());
  c->finalized = true;
}

// ------------------------------------------------------------------------------------------ K1 mel
static void mel_run(wl_ctx* c) {
  MelTables t{c->mel_window, c->mel_twiddle, c->mel_filt, c->mel_range, c->n_mels};
  WL_CUDA(cudaEventRecord(c->ev0, c->st));
  mel_forward(c->st, c->mel_pcm, c->mel_off, c->mel_out, c->mel_ooff, c->mel_gmax, t, c->mel_last_B, c->mel_last_frames);
  WL_CUDA(cudaEventRecord(c->ev1, c->st));
}

extern "C" int wl_mel(wl_ctx* c, const float* pcm, const int64_t* offsets, int32_t B, float* out, const int64_t* out_offsets) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK(pcm && offsets && out && out_offsets && B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_mel: bad arguments (B=%d, max %d)", B, c->Bm);
  const long total = offsets[B] - offsets[0];
  int max_frames = 0;
  std::vector<long> off(B + 1), ooff(B + 1);
  for (int b = 0; b <= B; ++b) off[b] = offsets[b] - offsets[0];
  for (int b = 0; b < B; ++b) {
    const long n = off[b + 1] - off[b];
    WL_CHECK(n > 0, WL_ERR_ARG, "wl_mel: empty waveform for stream %d", b);
    const int T = (int)(n / 160) + 1;
    max_frames = std::max(max_frames, T);
    WL_CHECK(out_offsets[b + 1] - out_offsets[b] == (long)T * c->n_mels, WL_ERR_ARG, "wl_mel: out_offsets do not match frames");
  }
  for (int b = 0; b <= B; ++b) ooff[b] = out_offsets[b] - out_offsets[0];
  c->mem.grow(c->mel_pcm, c->mel_pcm_cap, total, total + total / 4);
  c->mem.grow(c->mel_out, c->mel_out_cap, ooff[B], ooff[B] + ooff[B] / 4);
  WL_CUDA(cudaMemcpyAsync(c->mel_pcm, pcm + offsets[0], total * sizeof(float), cudaMemcpyHostToDevice, c->st));
  WL_CUDA(cudaMemcpyAsync(c->mel_off, off.data(), (B + 1) * sizeof(long), cudaMemcpyHostToDevice, c->st));
  WL_CUDA(cudaMemcpyAsync(c->mel_ooff, ooff.data(), (B + 1) * sizeof(long), cudaMemcpyHostToDevice, c->st));
  c->mel_last_B = B;
  c->mel_last_frames = max_frames;
  mel_run(c);
  WL_CUDA(cudaMemcpyAsync(out + out_offsets[0], c->mel_out, ooff[B] * sizeof(float), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaStreamSynchronize(c->st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[0], c->ev0, c->ev1));
  API_END(c)
}

// K1 with the result kept on the device: PCM up, log-mel stays in HBM until the next wl_mel_device call; the windows the
// encoder consumes are gathered from it on the device (wl_encode_windows), instead of copying the features to the host,
// zero-padding them there and copying them back (110 MB of PCIe traffic per 32-stream step).
extern "C" int wl_mel_device(wl_ctx* c, const float* pcm, const int64_t* offsets, int32_t B, int32_t* frames_out) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK(pcm && offsets && frames_out && B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_mel_device: bad arguments (B=%d, max %d)", B, c->Bm);
  const long total = offsets[B] - offsets[0];
  int max_frames = 0;
  std::vector<long> off(B + 1), ooff(B + 1, 0);
  c->res_frames_h.assign(B, 0);
  for (int b = 0; b <= B; ++b) off[b] = offsets[b] - offsets[0];
  for (int b = 0; b < B; ++b) {
    const long n = off[b + 1] - off[b];
    WL_CHECK(n > 0, WL_ERR_ARG, "wl_mel_device: empty waveform for stream %d", b);
    const int T = (int)(n / 160) + 1;
    max_frames = std::max(max_frames, T);
    c->res_frames_h[b] = T;
    frames_out[b] = T;
    ooff[b + 1] = ooff[b] + (long)T * c->n_mels;
  }
  c->mem.grow(c->res_pcm, c->res_pcm_cap, total, total + total / 4);
  c->mem.grow(c->res_mel, c->res_mel_cap, ooff[B], ooff[B] + ooff[B] / 4);
  cudaStream_t st = c->st;
  WL_CUDA(cudaMemcpyAsync(c->res_pcm, pcm + offsets[0], total * sizeof(float), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(c->res_off, off.data(), (B + 1) * sizeof(long), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(c->res_ooff, ooff.data(), (B + 1) * sizeof(long), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(c->res_frames, c->res_frames_h.data(), B * sizeof(int), cudaMemcpyHostToDevice, st));
  MelTables t{c->mel_window, c->mel_twiddle, c->mel_filt, c->mel_range, c->n_mels};
  WL_CUDA(cudaEventRecord(c->ev0, st));
  mel_forward(st, c->res_pcm, c->res_off, c->res_mel, c->res_ooff, c->mel_gmax, t, B, max_frames);
  WL_CUDA(cudaEventRecord(c->ev1, st));
  WL_CUDA(cudaStreamSynchronize(st));   // the caller's PCM and the staging vectors above may go away
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[0], c->ev0, c->ev1));
  API_END(c)
}

static void encode_impl(wl_ctx* c, const float* features_host, int B, const int* slots, bool resident);

extern "C" int wl_encode_windows(wl_ctx* c, int32_t B, const int32_t* win_stream, const int32_t* win_seek, const int32_t* win_len,
                                 int32_t* slots_out) {
  API_BEGIN(c)
  WL_CHECK(c->finalized && win_stream && win_seek && win_len && slots_out && B >= 1 && B <= c->Bm, WL_ERR_ARG,
           "wl_encode_windows: bad arguments (B=%d, max %d)", B, c->Bm);
  const int ns = (int)c->res_frames_h.size();
  for (int b = 0; b < B; ++b) {
    WL_CHECK(win_stream[b] >= 0 && win_stream[b] < ns, WL_ERR_ARG, "wl_encode_windows: window %d names stream %d (wl_mel_device holds %d)", b, win_stream[b], ns);
    WL_CHECK(win_seek[b] >= 0 && win_len[b] >= 0 && win_len[b] <= 3000 && win_seek[b] + win_len[b] <= c->res_frames_h[win_stream[b]],
             WL_ERR_ARG, "wl_encode_windows: window %d [%d, +%d) is outside the %d resident frames", b, win_seek[b], win_len[b],
             c->res_frames_h[win_stream[b]]);
  }
  WL_CHECK((int)c->slot_free.size() >= B, WL_ERR_NOMEM, "wl_encode_windows: %d encoder slots requested, %d free", B, (int)c->slot_free.size());
  for (int b = 0; b < B; ++b) {
    slots_out[b] = c->slot_free.back();
    c->slot_free.pop_back();
    c->slot_used[slots_out[b]] = 1;
  }
  try {
    std::vector<int> meta(3 * (size_t)B);
    for (int b = 0; b < B; ++b) { meta[b] = win_stream[b]; meta[B + b] = win_seek[b]; meta[2 * B + b] = win_len[b]; }
    WL_CUDA(cudaMemcpyAsync(c->win_meta, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, c->st));
    gather_windows(c->st, c->res_mel, c->res_ooff, c->res_frames, c->win_meta, c->win_meta + B, c->win_meta + 2 * B, c->feat32, B, c->n_mels);
    WL_CUDA(cudaStreamSynchronize(c->st));   // meta goes out of scope
    encode_impl(c, nullptr, B, slots_out, true);
  } catch (...) {
    for (int b = 0; b < B; ++b) { c->slot_used[slots_out[b]] = 0; c->slot_free.push_back(slots_out[b]); }
    throw;
  }
  API_END(c)
}

extern "C" int wl_mel_resident(wl_ctx* c) {
  API_BEGIN(c)
  WL_CHECK(c->mel_last_B > 0, WL_ERR_STATE, "wl_mel_resident: call wl_mel first");
  mel_run(c);
  WL_CUDA(cudaStreamSynchronize(c->st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[0], c->ev0, c->ev1));
  API_END(c)
}

// ------------------------------------------------------------------------------------------ K2-K7 encoder
GemmOperand opnd(const __half* p, long rows, long k, long ld, int n1, long s1, int n2, long s2) {
  GemmOperand o;
  o.ptr = p; o.rows = rows; o.k = k; o.ld = ld; o.n1 = n1; o.s1 = s1; o.n2 = n2; o.s2 = s2;
  return o;
}

// The conv stem: features [nb][n_mels][3000] f32 -> x [nb][1500][d] f32 (conv1 + GELU, conv2 (stride 2) + GELU + the
// positional table).  feat16 [nb][3002][n_mels] and conv1o [nb][3002][d] are workspaces whose rows 0 and 3001 of every
// stream must be zero (the conv padding): nothing here writes them.
void encoder_stem(wl_ctx* c, cudaStream_t st, int nb, const float* feat_dev, __half* feat16, __half* conv1o, float* x) {
  const int d = c->d, nm = c->n_mels;
  prep_features(st, feat_dev, feat16, nb, nm);
  {  // conv1 + GELU -> conv1o rows 1..3000 (rows 0 / 3001 stay zero)
    GemmEpilogue e;
    e.out = conv1o + d; e.out_f32 = 0; e.ldm = d; e.ldn = 1; e.ob1 = 3002L * d; e.bias = c->b_conv1; e.gelu = 1;
    gemm_tn(st, opnd(feat16, 3000, 3 * nm, nm, nb, 3002L * nm), opnd(c->w_conv1, d, 3 * nm, 3 * nm), 3000, d, 3 * nm, e);
  }
  {  // conv2 (stride 2) + GELU + positional table -> residual stream x (f32)
    GemmEpilogue e;
    e.out = x; e.out_f32 = 1; e.ldm = d; e.ldn = 1; e.ob1 = (long)S_ENC * d; e.bias = c->b_conv2; e.gelu = 1;
    e.resid = c->pos_enc; e.rldm = d; e.rldn = 1; e.rb1 = 0;
    gemm_tn(st, opnd(conv1o, S_ENC, 3 * d, 2 * d, nb, 3002L * d), opnd(c->w_conv2, d, 3 * d, 3 * d), S_ENC, d, 3 * d, e);
  }
}

// Encoder self-attention without the fused kernel (WLB200_FUSED_ATTN=0), AB streams at a time: the scores GEMM into
// scores [AB][H][1500][S_PAD] f32, softmax_rows into probs16 (same shape, fp16, the pad columns written as 0), the P V
// GEMM into attn.  qk [nb][1500][2d], vt [nb][d][S_PAD], attn [nb * 1500][d].
void encoder_attention_unfused(cudaStream_t st, const __half* qk, const __half* vt, __half* attn, float* scores,
                               __half* probs16, int nb, int H, int AB) {
  const int d = H * 64;
  for (int b0 = 0; b0 < nb; b0 += AB) {
    const int ab = std::min(AB, nb - b0);
    const __half* qb = qk + (long)b0 * S_ENC * 2 * d;
    {
      GemmEpilogue e;
      e.out = scores; e.out_f32 = 1; e.ldm = S_PAD; e.ob1 = (long)S_ENC * S_PAD; e.ob2 = (long)H * S_ENC * S_PAD;
      gemm_tn(st, opnd(qb, S_ENC, 64, 2 * d, H, 64, ab, (long)S_ENC * 2 * d),
              opnd(qb + d, S_ENC, 64, 2 * d, H, 64, ab, (long)S_ENC * 2 * d), S_ENC, S_ENC, 64, e);
    }
    softmax_rows(st, scores, probs16, (long)ab * H * S_ENC, S_ENC, S_PAD, S_PAD, 0.125f);
    {
      GemmEpilogue e;
      e.out = attn + (long)b0 * S_ENC * d; e.ldm = d; e.ob1 = 64; e.ob2 = (long)S_ENC * d;
      gemm_tn(st, opnd(probs16, S_ENC, S_PAD, S_PAD, H, (long)S_ENC * S_PAD, ab, (long)H * S_ENC * S_PAD),
              opnd(vt + (long)b0 * d * S_PAD, 64, S_PAD, S_PAD, H, 64L * S_PAD, ab, (long)d * S_PAD), S_ENC, 64, S_PAD, e);
    }
  }
}

static void encoder_pass(wl_ctx* c, int nb, const int* slots_host, const float* feat_dev) {
  const int d = c->d, H = c->H, ff = 4 * c->d;
  const long M = (long)nb * S_ENC;
  cudaStream_t st = c->st;
  encoder_stem(c, st, nb, feat_dev, c->feat16, c->conv1o, c->x);
  for (int l = 0; l < c->Le; ++l) {
    const EncLayer& L = c->enc[l];
    layernorm_rows(st, c->x, L.ln1_g, L.ln1_b, c->xn, nullptr, M, d);
    {
      GemmEpilogue e;
      e.out = c->qk; e.ldm = 2 * d; e.bias = L.b_qk;
      gemm_tn(st, opnd(c->xn, M, d, d), opnd(L.w_qk, 2 * d, d, d), (int)M, 2 * d, d, e);
    }
    {  // V^T[b] = Wv * xn[b]^T  (swap-AB) so that P*V reads V K-major
      GemmEpilogue e;
      e.out = c->vt; e.ldm = S_PAD; e.ldn = 1; e.ob1 = (long)d * S_PAD; e.bias = L.b_v; e.bias_on_m = 1;
      gemm_tn(st, opnd(L.w_v, d, d, d), opnd(c->xn, S_ENC, d, d, nb, (long)S_ENC * d), d, S_ENC, d, e);
    }
    static const bool fused_attn = [] { const char* e = getenv("WLB200_FUSED_ATTN"); return e ? atoi(e) != 0 : true; }();
    if (fused_attn) encoder_attention_fused(st, c->qk, c->vt, c->attn, nb, H, d);
    else encoder_attention_unfused(st, c->qk, c->vt, c->attn, c->scores, c->probs16, nb, H, c->AB);
    {
      GemmEpilogue e;
      e.out = c->x; e.out_f32 = 1; e.ldm = d; e.bias = L.b_o; e.resid = c->x; e.rldm = d;
      gemm_tn(st, opnd(c->attn, M, d, d), opnd(L.w_o, d, d, d), (int)M, d, d, e);
    }
    layernorm_rows(st, c->x, L.ln2_g, L.ln2_b, c->xn, nullptr, M, d);
    {
      GemmEpilogue e;
      e.out = c->hbuf; e.ldm = ff; e.bias = L.b_fc1; e.gelu = 1;
      gemm_tn(st, opnd(c->xn, M, d, d), opnd(L.w_fc1, ff, d, d), (int)M, ff, d, e);
    }
    {
      GemmEpilogue e;
      e.out = c->x; e.out_f32 = 1; e.ldm = d; e.bias = L.b_fc2; e.resid = c->x; e.rldm = d;
      gemm_tn(st, opnd(c->hbuf, M, ff, ff), opnd(L.w_fc2, d, ff, ff), (int)M, d, ff, e);
    }
  }
  layernorm_rows(st, c->x, c->lnp_g, c->lnp_b, c->xn, nullptr, M, d);
  for (int b = 0; b < nb; ++b)
    WL_CUDA(cudaMemcpyAsync(c->enc16 + (long)slots_host[b] * S_ENC * d, c->xn + (long)b * S_ENC * d,
                            (size_t)S_ENC * d * sizeof(__half), cudaMemcpyDeviceToDevice, st));
  // K7: cross-attention K/V of every decoder layer straight into the slot pool ([slot][H][1500][64])
  const long slot_sz = (long)S_ENC * d;
  for (int l = 0; l < c->Ld; ++l) {
    const DecLayer& L = c->dec[l];
    GemmEpilogue e;
    e.mode = GEMM_HEADSPLIT; e.hs_S = S_ENC; e.hs_H = H; e.hs_slot_stride = slot_sz; e.hs_slots = c->enc_slots_dev;
    e.out = c->ckv + ((long)l * 2 + 0) * c->NS * slot_sz;
    gemm_tn(st, opnd(c->xn, M, d, d), opnd(L.w_kc, d, d, d), (int)M, d, d, e);
    e.out = c->ckv + ((long)l * 2 + 1) * c->NS * slot_sz;
    e.bias = L.b_vc;
    gemm_tn(st, opnd(c->xn, M, d, d), opnd(L.w_vc, d, d, d), (int)M, d, d, e);
  }
}

static void encode_impl(wl_ctx* c, const float* features_host, int B, const int* slots, bool resident) {
  const size_t per = (size_t)c->n_mels * 3000;
  float ms_total = 0.f;
  for (int b0 = 0; b0 < B; b0 += c->EB) {
    const int nb = std::min(c->EB, B - b0);
    if (!resident)
      WL_CUDA(cudaMemcpyAsync(c->feat32 + b0 * per, features_host + b0 * per, nb * per * sizeof(float), cudaMemcpyHostToDevice, c->st));
    WL_CUDA(cudaMemcpyAsync(c->enc_slots_dev, slots + b0, nb * sizeof(int), cudaMemcpyHostToDevice, c->st));
    WL_CUDA(cudaEventRecord(c->ev0, c->st));
    encoder_pass(c, nb, slots + b0, c->feat32 + b0 * per);
    WL_CUDA(cudaEventRecord(c->ev1, c->st));
    WL_CUDA(cudaStreamSynchronize(c->st));
    float ms;
    WL_CUDA(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    ms_total += ms;
  }
  c->last_ms[1] = ms_total;
}

extern "C" int wl_encode(wl_ctx* c, const float* features, int32_t B, int32_t* slots_out) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK(features && slots_out && B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_encode: bad arguments (B=%d, max %d)", B, c->Bm);
  WL_CHECK((int)c->slot_free.size() >= B, WL_ERR_NOMEM, "wl_encode: %d encoder slots requested, %d free", B, (int)c->slot_free.size());
  for (int b = 0; b < B; ++b) {
    slots_out[b] = c->slot_free.back();
    c->slot_free.pop_back();
    c->slot_used[slots_out[b]] = 1;
  }
  try {
    encode_impl(c, features, B, slots_out, false);
  } catch (...) {
    for (int b = 0; b < B; ++b) { c->slot_used[slots_out[b]] = 0; c->slot_free.push_back(slots_out[b]); }
    throw;
  }
  API_END(c)
}

extern "C" int wl_encode_resident(wl_ctx* c, int32_t B, const int32_t* slots) {
  API_BEGIN(c)
  WL_CHECK(B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_encode_resident: B must be <= %d", c->Bm);
  for (int b = 0; b < B; ++b) WL_CHECK(slots[b] >= 0 && slots[b] < c->NS && c->slot_used[slots[b]], WL_ERR_ARG, "bad slot");
  encode_impl(c, nullptr, B, slots, true);
  API_END(c)
}

extern "C" int wl_slots_release(wl_ctx* c, const int32_t* slots, int32_t n) {
  API_BEGIN(c)
  for (int i = 0; i < n; ++i) {
    WL_CHECK(slots[i] >= 0 && slots[i] < c->NS && c->slot_used[slots[i]], WL_ERR_ARG, "wl_slots_release: slot %d is not in use", slots[i]);
    c->slot_used[slots[i]] = 0;
    c->slot_free.push_back(slots[i]);
  }
  API_END(c)
}
extern "C" int wl_slots_free_count(wl_ctx* c) { return c ? (int)c->slot_free.size() : -1; }

extern "C" int wl_encoder_output(wl_ctx* c, int32_t slot, float* out) {
  API_BEGIN(c)
  WL_CHECK(out && slot >= 0 && slot < c->NS && c->slot_used[slot], WL_ERR_ARG, "wl_encoder_output: bad slot %d", slot);
  const size_t n = (size_t)S_ENC * c->d;
  std::vector<__half> h(n);
  WL_CUDA(cudaMemcpy(h.data(), c->enc16 + (long)slot * n, n * sizeof(__half), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n; ++i) out[i] = __half2float(h[i]);
  API_END(c)
}

// ------------------------------------------------------------------------------------------ decoder step
namespace wl {
void gather_align_probs(cudaStream_t st, const DecodeState& s, const float* probs, float* buf, const int* heads, int n_heads,
                        int layer, int B, int rows_per_stream, int H);
}

// Decoder rows up to which every linear layer of the decode step is one wgemm launch (one m16 tile: with two, every CTA
// re-reads 82 KB of X from L2, so from 17 rows on the split-K dec_gemm path is used).
constexpr int WGEMM_MAX_ROWS = 16;

static void decode_step(wl_ctx* c, int B, int Kr, const SearchOpts& so, const VocabIds& vi, int nsplit, bool align_mode) {
  const int d = c->d, H = c->H, ff = 4 * c->d, R = B * Kr;
  cudaStream_t st = c->st;
  const DecodeState& s = c->ds;
  const long slot_sz = (long)S_ENC * d;
  PdlScope pdl(true);   // every kernel of the step is launched as a programmatic dependent of its predecessor
  decoder_embed(st, s, c->emb, c->pos_dec, c->dx, R, d);
  // Decode GEMMs are weight-streaming (M = out features, N = rows <= 256): K is split over enough CTAs to fill the
  // SMs; every K range stores its raw fp32 partial sum and the CONSUMER (LayerNorm, attention, GELU) adds the
  // ranges and the bias in a fixed order -- no atomics, bit-reproducible, and no separate reduction kernel.
  // part1 holds activations (qkv, q_cross, fc1), part2 the residual updates (out-proj, fc2) until the next LayerNorm.
  auto part_gemm = [&](const __half* W, int n_out, int K, const __half* X, float* buf, const float* bias,
                       int max_split = 8) -> PartialSrc {
    PartialSrc ps;
    ps.ptr = buf; ps.bias = bias; ps.stride = (long)c->Rm * n_out;
    ps.nsplit = dec_gemm_split_plan(n_out, R, K, max_split);
    dec_gemm(st, W, n_out, K, X, R, buf, n_out, ps.stride, ps.nsplit);
    return ps;
  };
  PartialSrc pending;   // residual update not yet folded into x
  auto cross = [&](int l, const PartialSrc& qc) {
    CrossAttnWorkspace ws = c->xws;
    ws.probs = align_mode ? c->align_probs : nullptr;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    const bool prof = c->prof_cross && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
    if (prof) { ws.ev0 = c->pev0; ws.ev1 = c->pev1; }
    decoder_cross_attn(st, s, qc, c->ckv + ((long)l * 2 + 0) * c->NS * slot_sz, c->ckv + ((long)l * 2 + 1) * c->NS * slot_sz,
                       slot_sz, ws, c->datt, B, Kr, H, d, nsplit);
    if (prof) {   // profiling pass only: serialises the host with the device
      float ms = 0.f;
      WL_CUDA(cudaEventSynchronize(c->pev1));
      WL_CUDA(cudaEventElapsedTime(&ms, c->pev0, c->pev1));
      c->prof_cross_ms += ms;
      c->prof_cross_n += 1;
    }
    if (align_mode)
      gather_align_probs(st, s, c->align_probs, c->align_buf, c->align_heads_dev, (int)c->align_heads.size() / 2, l, B, Kr, H);
  };
  // Small batches (R <= WGEMM_MAX_ROWS decoder rows, e.g. 4 streams per GPU with beam 4): every linear layer is one wgemm
  // launch whose epilogue writes FINAL values (bias, residual, GELU fused), so LayerNorm / attention read one value instead
  // of summing partials and the GELU-cast launch is gone: 12 launches per layer instead of 13, each a fraction of the code.
  const bool small = R <= WGEMM_MAX_ROWS && wgemm_supported(R, d) && wgemm_supported(R, ff);
  auto plain = [](const float* ptr) { PartialSrc ps; ps.ptr = ptr; ps.nsplit = 1; ps.stride = 0; ps.bias = nullptr; return ps; };
  // mode 0: out_f32 = X W^T + bias; 1: out_f32 += X W^T + bias; 2: out_f16 = gelu(X W^T + bias)
  auto lin = [&](const __half* W, int n_out, int K, const __half* X, const float* bias, int mode, float* of32, __half* of16) {
    wgemm(st, W, n_out, K, X, R, bias, mode, of32, of16, 0);
  };
  for (int l = 0; small && l < c->Ld; ++l) {
    const DecLayer& L = c->dec[l];
    layernorm_update_rows(st, c->dx, pending, L.ln1_g, L.ln1_b, c->dxn, R, d);
    lin(L.w_qkv, 3 * d, d, c->dxn, L.b_qkv, 0, c->part1, nullptr);
    decoder_self_attn(st, s, plain(c->part1), c->kcache + (long)l * c->cache_layer_stride, c->vcache + (long)l * c->cache_layer_stride,
                      c->cache_row_stride, c->datt, R, H, d);
    lin(L.w_o, d, d, c->datt, L.b_o, 1, c->dx, nullptr);
    layernorm_update_rows(st, c->dx, PartialSrc(), L.ln2_g, L.ln2_b, c->dxn, R, d);
    lin(L.w_qc, d, d, c->dxn, L.b_qc, 0, c->part1, nullptr);
    cross(l, plain(c->part1));
    lin(L.w_oc, d, d, c->datt, L.b_oc, 1, c->dx, nullptr);
    layernorm_update_rows(st, c->dx, PartialSrc(), L.ln3_g, L.ln3_b, c->dxn, R, d);
    lin(L.w_fc1, ff, d, c->dxn, L.b_fc1, 2, nullptr, c->dh);
    const int ks2 = wgemm_ksplit(ff);
    if (ks2 == 1) {
      lin(L.w_fc2, d, ff, c->dh, L.b_fc2, 1, c->dx, nullptr);
      pending = PartialSrc();
    } else {   // wgemm with K = 4d split over CTAs: the next LayerNorm folds the ranges (+ bias) into x
      wgemm(st, L.w_fc2, d, ff, c->dh, R, nullptr, 3, c->part2, nullptr, (long)c->Rm * d);
      pending.ptr = c->part2; pending.nsplit = ks2; pending.stride = (long)c->Rm * d; pending.bias = L.b_fc2;
    }
  }
  for (int l = 0; !small && l < c->Ld; ++l) {
    const DecLayer& L = c->dec[l];
    layernorm_update_rows(st, c->dx, pending, L.ln1_g, L.ln1_b, c->dxn, R, d);
    const PartialSrc qkv = part_gemm(L.w_qkv, 3 * d, d, c->dxn, c->part1, L.b_qkv);
    decoder_self_attn(st, s, qkv, c->kcache + (long)l * c->cache_layer_stride, c->vcache + (long)l * c->cache_layer_stride,
                      c->cache_row_stride, c->datt, R, H, d);
    pending = part_gemm(L.w_o, d, d, c->datt, c->part2, L.b_o);
    layernorm_update_rows(st, c->dx, pending, L.ln2_g, L.ln2_b, c->dxn, R, d);
    const PartialSrc qc = part_gemm(L.w_qc, d, d, c->dxn, c->part1, L.b_qc, 4);   // cross-attention sums <= 4 ranges
    cross(l, qc);
    pending = part_gemm(L.w_oc, d, d, c->datt, c->part2, L.b_oc);
    layernorm_update_rows(st, c->dx, pending, L.ln3_g, L.ln3_b, c->dxn, R, d);
    const PartialSrc h1 = part_gemm(L.w_fc1, ff, d, c->dxn, c->part1, L.b_fc1);
    gelu_cast(st, h1, c->dh, R, ff);
    pending = part_gemm(L.w_fc2, d, ff, c->dh, c->part2, L.b_fc2);
  }
  layernorm_update_rows(st, c->dx, pending, c->lnf_g, c->lnf_b, c->dxn, R, d);
  dec_gemm(st, c->emb, c->V, d, c->dxn, R, c->logits, c->Vld, 0, 1);
  search_rows(st, s, c->logits, so, vi, R);
  search_streams(st, s, so, vi, B);
}

// ------------------------------------------------------------------------------------------ K8 batched prefill
constexpr int PF_VCHUNK = 128;   // cross-attention groups (8 rows each) per launch

static void prefill_reserve(wl_ctx* c, long rows) {
  wl_ctx::Prefill& f = c->pf;
  if (rows <= f.cap_rows) return;
  const long cap = (rows + 1023) / 1024 * 1024;
  const int d = c->d, ff = 4 * c->d;
  DeviceMem& m = c->mem;
  f.cap_rows = 0;   // until every buffer of the set has its new size
  m.replace(f.tok, cap, true); m.replace(f.pos, cap, true); m.replace(f.active, cap, true); m.replace(f.wrow, cap, true);
  m.replace(f.vslot, cap / 8 + PF_VCHUNK, true); m.replace(f.vdone, cap / 8 + PF_VCHUNK, true);
  if (!f.sel) f.sel = m.alloc<int>(3 * (size_t)c->Rm + 16);
  m.replace(f.src, cap * T_MAX);
  m.replace(f.x, cap * d); m.replace(f.qkv, cap * 3 * d); m.replace(f.qc, cap * d);
  m.replace(f.xn, cap * d); m.replace(f.att, cap * d); m.replace(f.h, cap * ff);
  if (!f.xpart) f.xpart = m.alloc<float>((size_t)PF_VCHUNK * c->H * 12 * MAX_ROWS_PER_STREAM * 66, false);
  f.cap_rows = cap;
}

namespace wl {
void gather_align_rows(cudaStream_t st, const float* probs, const int* row_b, const int* row_pos, const int* row_active, float* buf,
                       const int* heads, int n_heads, int layer, int row0, int n_rows, int H);
void align_postprocess(cudaStream_t st, float* buf, float* mat, const int* Tn, const int* nfn, int B, int nh, int width, int n_start,
                       int max_T, int* path_out, int path_cap, int* path_len);
}

// Row layout of a batched decoder pass: stream b runs positions 0 .. ntok[b]-1 as rows [rowbase[b], rowbase[b] + n8)
struct PfRows {
  std::vector<int> tok, pos, act, wrow, vslot, rowbase, row_b;
  long M = 0;
  int NV = 0;
};

// index (optional, [B]): the decode-state index of list entry b (a decode session admits streams into arbitrary free
// indices; a one-shot call uses b itself) -- selects the hp row and the cache row the positions are written to.
static PfRows pf_rows(int B, int Kr, const int* toks, const int* tok_off /*B+1 or null: hp rows of T_MAX*/, const int* ntok,
                      const int32_t* slots, const int32_t* index = nullptr) {
  PfRows r;
  r.rowbase.assign(B, 0);
  for (int b = 0; b < B; ++b) {
    r.rowbase[b] = (int)r.tok.size();
    const int n = ntok[b], n8 = (n + 7) / 8 * 8;
    const int sb = index ? index[b] : b;
    const int* src = tok_off ? toks + tok_off[b] : toks + (size_t)sb * T_MAX;
    for (int i = 0; i < n8; ++i) {
      r.tok.push_back(i < n ? src[i] : 0);
      r.pos.push_back(i < n ? i : 0);
      r.act.push_back(i < n ? 1 : 0);
      r.wrow.push_back(sb * Kr);
      r.row_b.push_back(b);
    }
    for (int g = 0; g < n8 / 8; ++g) r.vslot.push_back(slots[b]);
  }
  r.M = (long)r.tok.size();
  r.NV = (int)r.vslot.size();
  return r;
}

// The decoder stack over M rows (every prompt / teacher-forced position of every stream at once): uploads the row
// tables, runs embed + Ld layers.  align = true additionally captures the cross-attention probabilities of the
// alignment heads into c->align_buf [B][nh][T_MAX][1500].  On return f.x holds the final residual stream of every row.
static void pf_stack(wl_ctx* c, const PfRows& r, bool align) {
  const int d = c->d, H = c->H, ff = 4 * c->d;
  cudaStream_t st = c->st;
  const long M = r.M;
  const int NV = r.NV;
  prefill_reserve(c, M);
  wl_ctx::Prefill& f = c->pf;
  WL_CUDA(cudaMemcpyAsync(f.tok, r.tok.data(), M * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(f.pos, r.pos.data(), M * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(f.active, r.act.data(), M * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(f.wrow, r.wrow.data(), M * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(f.vslot, r.vslot.data(), NV * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemsetAsync(f.vdone, 0, NV * 4, st));
  const int nh = (int)c->align_heads.size() / 2;
  if (align) {
    c->mem.grow(f.row_b, f.row_b_cap, f.cap_rows, 0, true);
    WL_CUDA(cudaMemcpyAsync(f.row_b, r.row_b.data(), M * 4, cudaMemcpyHostToDevice, st));
    if (!f.aprobs) f.aprobs = c->mem.alloc<float>((size_t)PF_VCHUNK * 8 * H * S_ENC, false);
  }
  prefill_embed(st, f.tok, f.pos, f.active, f.wrow, c->emb, c->pos_dec, f.x, f.src, (int)M, d);
  DecodeState sv = c->ds;
  sv.active = f.active; sv.pos = f.pos; sv.src = f.src; sv.wrow = f.wrow;
  auto plain = [](const float* ptr) { PartialSrc ps; ps.ptr = ptr; ps.nsplit = 1; ps.stride = 0; ps.bias = nullptr; return ps; };
  const long slot_sz = (long)S_ENC * d;
  for (int l = 0; l < c->Ld; ++l) {
    const DecLayer& L = c->dec[l];
    __half* kc = c->kcache + (long)l * c->cache_layer_stride;
    __half* vc = c->vcache + (long)l * c->cache_layer_stride;
    layernorm_rows(st, f.x, L.ln1_g, L.ln1_b, f.xn, nullptr, M, d);
    {
      GemmEpilogue e;
      e.out = f.qkv; e.out_f32 = 1; e.ldm = 3 * d; e.bias = L.b_qkv;
      gemm_tn(st, opnd(f.xn, M, d, d), opnd(L.w_qkv, 3 * d, d, d), (int)M, 3 * d, d, e);
    }
    prefill_kv_write(st, f.qkv, f.pos, f.active, f.wrow, kc, vc, c->cache_row_stride, (int)M, H, d);
    decoder_self_attn(st, sv, plain(f.qkv), kc, vc, c->cache_row_stride, f.att, (int)M, H, d);
    {
      GemmEpilogue e;
      e.out = f.x; e.out_f32 = 1; e.ldm = d; e.bias = L.b_o; e.resid = f.x; e.rldm = d;
      gemm_tn(st, opnd(f.att, M, d, d), opnd(L.w_o, d, d, d), (int)M, d, d, e);
    }
    layernorm_rows(st, f.x, L.ln2_g, L.ln2_b, f.xn, nullptr, M, d);
    {
      GemmEpilogue e;
      e.out = f.qc; e.out_f32 = 1; e.ldm = d; e.bias = L.b_qc;
      gemm_tn(st, opnd(f.xn, M, d, d), opnd(L.w_qc, d, d, d), (int)M, d, d, e);
    }
    bool capture = false;
    if (align)
      for (int i = 0; i < nh; ++i) capture = capture || c->align_heads[2 * i] == l;
    for (int v0 = 0; v0 < NV; v0 += PF_VCHUNK) {   // groups of 8 rows against their stream's encoder K/V
      const int Bv = std::min(PF_VCHUNK, NV - v0);
      DecodeState sx = c->ds;
      sx.done = f.vdone + v0; sx.slot = f.vslot + v0;
      CrossAttnWorkspace ws;
      ws.part = f.xpart; ws.probs = capture ? f.aprobs : nullptr;
      const int nsp = capture ? 1 : cross_attn_pick_nsplit(Bv, H, c->num_sms, MAX_ROWS_PER_STREAM);   // exact probabilities need the whole key range
      decoder_cross_attn(st, sx, plain(f.qc + (long)v0 * 8 * d), c->ckv + ((long)l * 2 + 0) * c->NS * slot_sz,
                         c->ckv + ((long)l * 2 + 1) * c->NS * slot_sz, slot_sz, ws, f.att + (long)v0 * 8 * d, Bv, MAX_ROWS_PER_STREAM, H, d, nsp);
      if (capture)
        gather_align_rows(st, f.aprobs, f.row_b, f.pos, f.active, c->align_buf, c->align_heads_dev, nh, l, v0 * 8, Bv * 8, H);
    }
    {
      GemmEpilogue e;
      e.out = f.x; e.out_f32 = 1; e.ldm = d; e.bias = L.b_oc; e.resid = f.x; e.rldm = d;
      gemm_tn(st, opnd(f.att, M, d, d), opnd(L.w_oc, d, d, d), (int)M, d, d, e);
    }
    layernorm_rows(st, f.x, L.ln3_g, L.ln3_b, f.xn, nullptr, M, d);
    {
      GemmEpilogue e;
      e.out = f.h; e.ldm = ff; e.bias = L.b_fc1; e.gelu = 1;
      gemm_tn(st, opnd(f.xn, M, d, d), opnd(L.w_fc1, ff, d, d), (int)M, ff, d, e);
    }
    {
      GemmEpilogue e;
      e.out = f.x; e.out_f32 = 1; e.ldm = d; e.bias = L.b_fc2; e.resid = f.x; e.rldm = d;
      gemm_tn(st, opnd(f.h, M, ff, ff), opnd(L.w_fc2, d, ff, ff), (int)M, d, ff, e);
    }
  }
  WL_CUDA(cudaStreamSynchronize(st));   // the row tables of `r` were uploaded asynchronously
  f.rows_done += M;
  f.calls += 1;
}

// softmax(logits of row sel[j])[tgt[j]] -> out[oidx[j]] for n selected rows of f.x: final LayerNorm + vocabulary
// projection through the decode step's own kernels, Rm rows at a time
static void pf_row_probs(wl_ctx* c, const std::vector<int>& sel, const std::vector<int>& tgt, const std::vector<int>& oidx, float* out_dev) {
  cudaStream_t st = c->st;
  wl_ctx::Prefill& f = c->pf;
  const int n = (int)sel.size(), d = c->d;
  for (int i0 = 0; i0 < n; i0 += c->Rm) {
    const int m = std::min(c->Rm, n - i0);
    std::vector<int> up(3 * (size_t)m);
    for (int i = 0; i < m; ++i) { up[i] = sel[i0 + i]; up[m + i] = tgt[i0 + i]; up[2 * m + i] = oidx[i0 + i]; }
    WL_CUDA(cudaMemcpyAsync(f.sel, up.data(), up.size() * 4, cudaMemcpyHostToDevice, st));
    gather_rows(st, f.x, f.sel, c->dx, m, d);
    layernorm_update_rows(st, c->dx, PartialSrc(), c->lnf_g, c->lnf_b, c->dxn, m, d);
    dec_gemm(st, c->emb, c->V, d, c->dxn, m, c->logits, c->Vld, 0, 1);
    row_prob(st, c->logits, c->V, c->Vld, f.sel + m, f.sel + 2 * m, out_dev, m);
    WL_CUDA(cudaStreamSynchronize(st));
  }
}

// K8: all prompt positions but the last of every stream through the decoder stack in one pass.  hp = prompts [B][T_MAX]
// (pinned host), P / sot / slots per stream.  Leaves the self-attention cache filled for positions 0 .. P-2 in the
// stream's first decode row (b * Kr) and the no-speech probability of streams whose sot lies inside the prompt.
static void prefill_forward(wl_ctx* c, int B, int Kr, const int* hp, const int* P, const int* sot, const int32_t* slots,
                            const int32_t* index = nullptr) {
  // (with `index`: hp rows and P / sot columns are addressed by state index, list entry b is state index index[b])
  auto at = [&](int b) { return index ? index[b] : b; };
  if (!index) WL_CUDA(cudaMemsetAsync(c->ds.no_speech, 0, B * sizeof(float), c->st));
  else for (int b = 0; b < B; ++b) WL_CUDA(cudaMemsetAsync(c->ds.no_speech + index[b], 0, sizeof(float), c->st));
  std::vector<int> ntok(B);
  for (int b = 0; b < B; ++b) ntok[b] = P[at(b)] - 1;
  const PfRows r = pf_rows(B, Kr, hp, nullptr, ntok.data(), slots, index);
  if (r.M == 0) return;
  pf_stack(c, r, false);
  std::vector<int> sel, tgt, oidx;
  for (int b = 0; b < B; ++b) {
    const int sb = at(b);
    if (sot[sb] >= 0 && sot[sb] < P[sb] - 1) { sel.push_back(r.rowbase[b] + sot[sb]); tgt.push_back(c->cfg.no_speech); oidx.push_back(sb); }
  }
  if (!sel.empty()) pf_row_probs(c, sel, tgt, oidx, c->ds.no_speech);
}

static VocabIds vocab_ids(wl_ctx* c) {
  VocabIds v;
  v.vocab = c->V; v.vocab_ld = c->Vld; v.eot = c->cfg.eot; v.sot = c->cfg.sot; v.no_speech = c->cfg.no_speech;
  v.no_timestamps = c->cfg.no_timestamps; v.ts_begin = c->cfg.timestamp_begin; v.blank = c->cfg.blank;
  return v;
}

// Per-stream metadata of a decode call (rows 0-9 of column b of the [META_ROWS][B] table `meta`; tokens into
// hp_row[T_MAX]; search_meta writes the other rows).  Returns the
// decode steps the stream may need without prefill; *n_new_out = the new tokens it may emit.
static int stream_meta(wl_ctx* c, int b, int slot, const int32_t* prompt, int P, int ml, bool forced, int* hp_row, int* meta, int col,
                       int ncol, int* n_new_out, bool reads_slot = true) {
  WL_CHECK(P >= 1 && P <= T_MAX, WL_ERR_ARG, "stream %d: prompt length %d out of range", b, P);
  WL_CHECK(!reads_slot || (slot >= 0 && slot < c->NS && c->slot_used[slot]), WL_ERR_ARG, "stream %d: bad encoder slot %d", b, slot);
  int sot = -1;
  for (int i = 0; i < P; ++i) {
    const int t = prompt[i];
    WL_CHECK(t >= 0 && t < c->V, WL_ERR_ARG, "stream %d: token id %d out of range", b, t);
    hp_row[i] = t;
    if (t == c->cfg.sot && sot < 0) sot = i;
  }
  int n_new = 0, steps = P;
  if (!forced) {
    WL_CHECK(ml >= 2 && ml <= T_MAX, WL_ERR_ARG, "stream %d: max_length %d out of range", b, ml);
    n_new = std::min(ml / 2, ml - P);
    WL_CHECK(n_new >= 1, WL_ERR_ARG, "stream %d: prompt of %d tokens leaves no room under max_length %d", b, P, ml);
    steps = P - 1 + n_new;
  }
  // end of the sot sequence = CT2's prompt length: sot, then every following id in [sot, no_timestamps]
  // (language, task, notimestamps); the tokens after it are a prefix that counts as sampled text
  int sb = P;
  if (sot >= 0) {
    sb = sot + 1;
    while (sb < P && prompt[sb] >= c->cfg.sot && prompt[sb] <= c->cfg.no_timestamps) ++sb;
  }
  const int npre = P - sb;
  int lts = -1;
  for (int i = sb; i < P; ++i)
    if (prompt[i] >= c->cfg.timestamp_begin) lts = prompt[i];
  meta[0 * ncol + col] = slot;
  meta[1 * ncol + col] = P;
  meta[2 * ncol + col] = sot;
  meta[3 * ncol + col] = sb >= 1 ? prompt[sb - 1] != c->cfg.no_timestamps : 1;
  meta[4 * ncol + col] = n_new;
  meta[5 * ncol + col] = forced ? P : 0;
  meta[6 * ncol + col] = forced ? 0 : npre;
  meta[7 * ncol + col] = npre >= 1 ? prompt[P - 1] : -1;
  meta[8 * ncol + col] = npre >= 2 ? prompt[P - 2] : -1;
  meta[9 * ncol + col] = forced ? -1 : lts;
  if (n_new_out) *n_new_out = n_new;
  return steps;
}

// The search of the stream in column `col` (rows 10-14 of the metadata table): sample = 0 takes the call's / session's
// SearchOpts over `rows` rows; sample = 1 is Gumbel-max sampling at `temperature` over `rows` independent rows, its noise
// that of wl_generate(seed) for the stream at batch position `key`.
static void search_meta(int* meta, int col, int ncol, int sample, float temperature, uint32_t seed, int key, int rows) {
  int tbits;
  memcpy(&tbits, &temperature, 4);
  meta[10 * ncol + col] = sample;
  meta[11 * ncol + col] = tbits;
  meta[12 * ncol + col] = (int)seed;
  meta[13 * ncol + col] = key;
  meta[14 * ncol + col] = rows;
}

// prompts [B][T_MAX] + the [META_ROWS][B] metadata table (pinned host) -> the device state
static void upload_state_tables(wl_ctx* c, const int* hp, const int* meta, int B) {
  const DecodeState& s = c->ds;
  cudaStream_t st = c->st;
  WL_CUDA(cudaMemcpyAsync(s.prompt, hp, (size_t)B * T_MAX * 4, cudaMemcpyHostToDevice, st));
  void* dst[META_ROWS] = {s.slot, s.prompt_len, s.sot_index, s.use_ts, s.n_new, s.force_len, s.pre_n, s.pre_last, s.pre_penult,
                          s.pre_lts, s.smode, s.temp, s.nseed, s.nkey, s.nrows};
  for (int k = 0; k < META_ROWS; ++k) WL_CUDA(cudaMemcpyAsync(dst[k], meta + (size_t)k * B, B * 4, cudaMemcpyHostToDevice, st));
}

// upload prompts & per-stream metadata, every stream with the same search (key = batch position); returns max steps.
// slots == nullptr: the call reads no encoder slot (wl_test_search), every stream gets slot 0.
static int upload_streams(wl_ctx* c, const int32_t* slots, int B, const int32_t* prompts, const int32_t* off, int max_length,
                          bool forced, int sample, float temperature, uint32_t seed, int rows, const int32_t* max_len_ps = nullptr,
                          int* max_new_out = nullptr) {
  ensure_host(c, (size_t)B * (T_MAX + 16), 16);
  int* hp = c->h_int;                      // [B][T_MAX]
  int* meta = c->h_int + (size_t)B * T_MAX;  // [META_ROWS][B]
  int max_steps = 0, max_new = 0;
  for (int b = 0; b < B; ++b) {
    int n_new = 0;
    const int steps = stream_meta(c, b, slots ? slots[b] : 0, prompts + off[b], off[b + 1] - off[b],
                                  max_len_ps ? max_len_ps[b] : max_length, forced, hp + (size_t)b * T_MAX, meta, b, B, &n_new,
                                  slots != nullptr);
    search_meta(meta, b, B, sample, temperature, seed, b, rows);
    max_steps = std::max(max_steps, steps);
    max_new = std::max(max_new, n_new);
  }
  upload_state_tables(c, hp, meta, B);
  if (max_new_out) *max_new_out = max_new;
  return max_steps;
}

// the score CT2 ranks a hypothesis by: cum_logprob / len^length_penalty
static float hyp_score(float cum, int len, float length_penalty) {
  return length_penalty == 0.f ? cum : cum / powf((float)std::max(len, 1), length_penalty);
}

// finished hypotheses of one stream (device order) -> the NH best by cum_logprob / len^length_penalty, like CT2
static void emit_hyps(int NH, float length_penalty, int count, const int* h_len, const float* h_cum, const int* h_tok, int32_t* out_ids,
                      int32_t* out_len, float* out_score) {
  const int cnt = std::min(count, MAX_HYPS);
  std::vector<int> order(cnt);
  std::vector<float> score(cnt);
  for (int i = 0; i < cnt; ++i) {
    order[i] = i;
    score[i] = hyp_score(h_cum[i], h_len[i], length_penalty);
  }
  std::stable_sort(order.begin(), order.end(), [&](int a, int bb) { return score[a] > score[bb]; });
  for (int hh = 0; hh < NH; ++hh) {
    int* dst = out_ids + (size_t)hh * T_MAX;
    if (hh < cnt) {
      const int i = order[hh];
      memcpy(dst, h_tok + (size_t)i * T_MAX, h_len[i] * sizeof(int));
      out_len[hh] = h_len[i];
      out_score[hh] = score[i];
    } else {
      out_len[hh] = -1;
      out_score[hh] = 0.f;
    }
  }
}

// One token step of a generate call: the decoder's (decode_step), or with `script` (wl_test_search) the scripted logits
// followed by the same two search kernels.
static void token_step(wl_ctx* c, int B, int Kr, const SearchOpts& so, const VocabIds& vi, int nsplit, const SearchScript* script) {
  if (!script) {
    decode_step(c, B, Kr, so, vi, nsplit, false);
    return;
  }
  PdlScope pdl(true);
  scripted_logits(c->st, c->ds, so, vi, *script, c->logits, B * Kr);
  search_rows(c->st, c->ds, c->logits, so, vi, B * Kr);
  search_streams(c->st, c->ds, so, vi, B);
}

// The captured token loop for one call shape (cached per context): a conditional WHILE node whose body is the decode
// step + loop_condition, so the whole loop is one launch.  `tag` separates the graphs of the one-shot state ("g") from
// those of the decode session ("s"): the captures bake the state's device pointers in (and a script's parameters).
static cudaGraphExec_t decode_graph(wl_ctx* c, const char* tag, int B, int Kr, int K, const SearchOpts& so, const VocabIds& vi,
                                    int nsplit, long* kernels, const SearchScript* script = nullptr) {
  cudaStream_t st = c->st;
  char key[160];
  snprintf(key, sizeof(key), "%s/%d/%d/%d/%d/%d/%d", tag, B, Kr, K, so.max_cand, so.suppress_blank, so.max_initial_ts);
  if (script) snprintf(key + strlen(key), sizeof(key) - strlen(key), "/script/%u/%d", script->seed, script->pattern);
  GraphEntry& ge = c->graphs[key];
  if (!ge.exec) {
    const long before = gemm_launch_count() + dec_gemm_launch_count() + wgemm_launch_count() + other_launch_count();
    cudaGraph_t g = nullptr, cap = nullptr;
    WL_CUDA(cudaGraphCreate(&g, 0));
    cudaGraphConditionalHandle h;
    WL_CUDA(cudaGraphConditionalHandleCreate(&h, g, 1, cudaGraphCondAssignDefault));
    cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
    np.conditional.handle = h;
    np.conditional.type = cudaGraphCondTypeWhile;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    WL_CUDA(cudaGraphAddNode(&node, g, nullptr, 0, &np));
    cudaGraph_t body = np.conditional.phGraph_out[0];
    WL_CUDA(cudaStreamBeginCaptureToGraph(st, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    try {
      token_step(c, B, Kr, so, vi, nsplit, script);
      loop_condition(st, c->ds, h, B);
    } catch (...) {
      cudaStreamEndCapture(st, &cap);
      cudaGraphDestroy(g);
      throw;
    }
    WL_CUDA(cudaStreamEndCapture(st, &cap));
    ge.kernels = gemm_launch_count() + dec_gemm_launch_count() + wgemm_launch_count() + other_launch_count() - before;
    c->capture_counted += ge.kernels;
    WL_CUDA(cudaGraphInstantiate(&ge.exec, g, 0));
    cudaGraphDestroy(g);
  }
  *kernels = ge.kernels;
  return ge.exec;
}

// round(K * patience) of a beam search, half away from zero like CT2's std::round [recalled, not pinned]; at least 1
static int max_candidates(int K, float patience, const char* who) {
  if (K == 1) return 1;
  const long mc = std::max(1L, lroundf(K * patience));
  WL_CHECK(mc <= MAX_FINISHED, WL_ERR_ARG, "%s: round(beam_size * patience) = %ld exceeds the limit of %d finished hypotheses",
           who, mc, MAX_FINISHED);
  return (int)mc;
}

// wl_generate and wl_test_search.  `script` == nullptr: the decoder computes the logits of every step from the encoder
// slots; otherwise the scripted logits replace the decoder and no slot is read (slots may be null).  Everything else --
// the uploads, decode_init, the captured or host-driven loop, the search kernels, the hypothesis ranking -- is the same
// code for both.  out_hyp_count [B] (optional): hypotheses each stream finished with; out_logits (optional, script only):
// the [B * rows per stream][vocab_ld] logits of the first decode step.
static void generate_run(wl_ctx* c, const int32_t* slots, int32_t B, const int32_t* prompts, const int32_t* prompt_off,
                         const wl_gen_opts* o, const SearchScript* script, int32_t* out_ids, int32_t* out_len, float* out_score,
                         float* out_no_speech, int32_t* out_steps, int32_t* out_hyp_count, float* out_logits) {
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK((slots || script) && prompts && prompt_off && o && out_ids && out_len && out_score, WL_ERR_ARG, "wl_generate: null argument");
  WL_CHECK(B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_generate: B=%d exceeds max_streams=%d", B, c->Bm);
  WL_CHECK(o->beam_size >= 1 && o->num_hypotheses >= 1, WL_ERR_ARG, "wl_generate: beam_size / num_hypotheses must be >= 1");
  const int K = o->beam_size;
  const int Kr = K > 1 ? K : o->num_hypotheses;
  WL_CHECK(Kr <= c->Km, WL_ERR_ARG, "wl_generate: %d rows per stream exceed max_beam=%d", Kr, c->Km);
  WL_CHECK(K == 1 || o->num_hypotheses <= MAX_FINISHED, WL_ERR_ARG, "too many hypotheses");
  WL_CHECK(o->sampling_topk == 0 || o->sampling_topk == 1, WL_ERR_ARG, "sampling_topk must be 0 (full) or 1 (arg-max)");
  WL_CHECK(o->max_length >= 2 && o->max_length <= T_MAX, WL_ERR_ARG, "max_length %d out of range", o->max_length);
  const int R = B * Kr;
  SearchOpts so;
  so.beam = K; so.rows_per_stream = Kr;
  so.max_cand = max_candidates(K, o->patience, "wl_generate");
  so.suppress_blank = o->suppress_blank; so.max_initial_ts = o->max_initial_timestamp_index;
  so.suppress_mask = c->suppress_mask;
  const int sample = (K == 1 && o->sampling_topk == 0 && o->sampling_temperature > 0.f) ? 1 : 0;
  const VocabIds vi = vocab_ids(c);
  cudaStream_t st = c->st;
  // suppress bitmask
  const int nwords = (c->V + 31) / 32 + 1;
  std::vector<unsigned> mask(nwords, 0u);
  for (int i = 0; i < o->n_suppress; ++i) {
    const int t = o->suppress_tokens[i];
    if (t >= 0 && t < c->V) mask[t >> 5] |= 1u << (t & 31);
  }
  int max_new = 0;
  int max_steps = upload_streams(c, script ? nullptr : slots, B, prompts, prompt_off, o->max_length, false, sample,
                                 o->sampling_temperature, o->seed, Kr, o->max_length_per_stream, &max_new);
  // K8: every prompt position but the last goes through the decoder in ONE batched pass (prefill = 2: one decode step per
  // prompt token)
  const bool prefilled = o->prefill == 0 || o->prefill == 1;
  if (prefilled) max_steps = max_new;
  WL_CUDA(cudaMemcpyAsync(c->suppress_mask, mask.data(), nwords * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaEventRecord(c->ev0, st));
  if (prefilled && script) {
    // the batched prefill pass is what writes the no-speech probability of a stream whose sot precedes its last token
    WL_CUDA(cudaMemsetAsync(c->ds.no_speech, 0, B * sizeof(float), st));
    scripted_no_speech(st, c->ds, vi, *script, B);
  } else if (prefilled) {
    // upload_streams staged the prompts in pinned host memory: h_int = [B][T_MAX] tokens, then the per-stream metadata
    WL_CUDA(cudaStreamSynchronize(st));
    const int* hp = c->h_int;
    const int* meta = c->h_int + (size_t)B * T_MAX;
    prefill_forward(c, B, Kr, hp, meta + 1 * B, meta + 2 * B, slots);
  }
  decode_init(st, c->ds, so, vi, B, R, prefilled ? 1 : 0);
  if (script && out_logits) {   // a pure function of the state: the first step below recomputes the same values
    scripted_logits(st, c->ds, so, vi, *script, c->logits, R);
    WL_CUDA(cudaMemcpyAsync(out_logits, c->logits, (size_t)R * c->Vld * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  const int nsplit = cross_attn_pick_nsplit(B, c->H, c->num_sms, Kr);

  // The whole token loop is ONE graph launch: a conditional WHILE node whose body is the captured decode step; the
  // body's last kernel (loop_condition) keeps the loop alive while some stream is still decoding and the step budget
  // lasts.  No host round trip per token, no wasted steps after the last EOT.  Without graphs (use_cuda_graph = 0) the
  // host launches the steps itself and checks for the end every 4 steps.
  cudaGraphExec_t exec = nullptr;
  long graph_kernels = 0;
  if (o->use_cuda_graph) exec = decode_graph(c, script ? "t" : "g", B, Kr, K, so, vi, nsplit, &graph_kernels, script);
  ensure_host(c, (size_t)B * (T_MAX + 16) + (size_t)B * MAX_HYPS * (T_MAX + 2) + 64, (size_t)B * (MAX_HYPS + 2));
  int* h_done = c->h_int;  // reuse (prompts are already on the device: the copies above are stream-ordered)
  WL_CUDA(cudaStreamSynchronize(st));
  if (exec) {
    h_done[0] = max_steps;
    WL_CUDA(cudaMemcpyAsync(c->ds.steps_left, h_done, sizeof(int), cudaMemcpyHostToDevice, st));
    WL_CUDA(cudaGraphLaunch(exec, st));
    WL_CUDA(cudaMemcpyAsync(h_done, c->ds.steps_left, sizeof(int), cudaMemcpyDeviceToHost, st));
    WL_CUDA(cudaStreamSynchronize(st));
    c->graph_launched += graph_kernels * (long)(max_steps - h_done[0]);
  } else {
    int ran = 0;
    const int check_every = 4;
    while (ran < max_steps) {
      const int n = std::min(check_every, max_steps - ran);
      for (int i = 0; i < n; ++i) token_step(c, B, Kr, so, vi, nsplit, script);
      ran += n;
      WL_CUDA(cudaMemcpyAsync(h_done, c->ds.n_done, sizeof(int), cudaMemcpyDeviceToHost, st));
      WL_CUDA(cudaStreamSynchronize(st));
      if (*h_done >= B) break;
    }
  }
  WL_CUDA(cudaEventRecord(c->ev1, st));
  // results
  const DecodeState& s = c->ds;
  int* h_cnt = c->h_int;
  int* h_len = h_cnt + B;
  int* h_steps = h_len + (size_t)B * MAX_HYPS;
  int* h_tok = h_steps + B;
  float* h_cum = c->h_flt;
  float* h_ns = h_cum + (size_t)B * MAX_HYPS;
  WL_CUDA(cudaMemcpyAsync(h_cnt, s.hyp_count, B * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_len, s.hyp_len, (size_t)B * MAX_HYPS * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_steps, s.steps_run, B * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_tok, s.hyp_tok, (size_t)B * MAX_HYPS * T_MAX * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_cum, s.hyp_cum, (size_t)B * MAX_HYPS * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_ns, s.no_speech, B * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[2], c->ev0, c->ev1));
  if (c->tl_dev) {   // dump + reset the in-graph timeline of this call
    std::vector<unsigned long long> h(TL_CAP + 1);
    WL_CUDA(cudaMemcpy(h.data(), c->tl_dev, h.size() * 8, cudaMemcpyDeviceToHost));
    const size_t n = std::min<size_t>((size_t)(h[0] & 0xffffffffu), TL_CAP);
    if (FILE* f = fopen(c->tl_path.c_str(), "wb")) { fwrite(h.data() + 1, 8, n, f); fclose(f); }
    WL_CUDA(cudaMemset(c->tl_dev, 0, 8));
  }
  for (int b = 0; b < B; ++b) {
    emit_hyps(o->num_hypotheses, o->length_penalty, h_cnt[b], h_len + (size_t)b * MAX_HYPS, h_cum + (size_t)b * MAX_HYPS,
              h_tok + (size_t)b * MAX_HYPS * T_MAX, out_ids + (size_t)b * o->num_hypotheses * T_MAX, out_len + (size_t)b * o->num_hypotheses,
              out_score + (size_t)b * o->num_hypotheses);
    if (out_no_speech) out_no_speech[b] = h_ns[b];
    if (out_steps) out_steps[b] = h_steps[b];
    if (out_hyp_count) out_hyp_count[b] = h_cnt[b];
  }
}

extern "C" int wl_generate(wl_ctx* c, const int32_t* slots, int32_t B, const int32_t* prompts, const int32_t* prompt_off,
                           const wl_gen_opts* o, int32_t* out_ids, int32_t* out_len, float* out_score, float* out_no_speech,
                           int32_t* out_steps) {
  API_BEGIN(c)
  WL_CHECK(slots, WL_ERR_ARG, "wl_generate: null argument");
  generate_run(c, slots, B, prompts, prompt_off, o, nullptr, out_ids, out_len, out_score, out_no_speech, out_steps, nullptr, nullptr);
  API_END(c)
}

extern "C" int wl_test_search(wl_ctx* c, int32_t B, const int32_t* prompts, const int32_t* prompt_off, const wl_gen_opts* o,
                              const wl_search_script* script, int32_t* out_ids, int32_t* out_len, float* out_score,
                              float* out_no_speech, int32_t* out_steps, int32_t* out_hyp_count, float* out_logits) {
  API_BEGIN(c)
  WL_CHECK(script, WL_ERR_ARG, "wl_test_search: null script");
  WL_CHECK(script->pattern >= -1 && script->pattern <= 5, WL_ERR_ARG, "wl_test_search: pattern %d out of range", script->pattern);
  SearchScript sc;
  sc.seed = script->seed; sc.pattern = script->pattern;
  generate_run(c, nullptr, B, prompts, prompt_off, o, &sc, out_ids, out_len, out_score, out_no_speech, out_steps, out_hyp_count,
               out_logits);
  API_END(c)
}

// ------------------------------------------------------------------------------------------ N2 decode session
// Step-level continuous batching (replaces the run-to-completion batches of the reference's BatchInferenceWorker,
// whisper_live/batch_inference.py:155-187, :259, :334-339): the decode state has `cap` stream indices; a stream is
// admitted into a free index at any token-step boundary (prompt prefilled in one pass, K8), the device-side loop runs
// for a bounded number of steps or until some stream finishes, and a finished stream is collected -- and its index
// refilled -- while the others keep decoding.  Idle indices carry done = 1: every kernel of the step skips them.
struct SessScope {   // the session's state / cache / suppress mask stand in for the one-shot ones inside a session call
  wl_ctx* c;
  explicit SessScope(wl_ctx* ctx) : c(ctx) { swap(); }
  ~SessScope() { swap(); }
  void swap() {
    std::swap(c->ds, c->sess.ds);
    std::swap(c->kcache, c->sess.kcache);
    std::swap(c->vcache, c->sess.vcache);
    std::swap(c->suppress_mask, c->sess.mask);
  }
};

extern "C" int wl_session_open(wl_ctx* c, const wl_gen_opts* o, int32_t capacity) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "weights not finalized");
  WL_CHECK(o, WL_ERR_ARG, "wl_session_open: null options");
  wl_ctx::Session& ss = c->sess;
  WL_CHECK(!ss.open || ss.live == 0, WL_ERR_STATE, "wl_session_open: %d streams of the open session are still decoding", ss.live);
  WL_CHECK(capacity >= 1 && capacity <= c->Bm, WL_ERR_ARG, "wl_session_open: capacity %d exceeds max_streams=%d", capacity, c->Bm);
  WL_CHECK(o->beam_size >= 1 && o->num_hypotheses >= 1, WL_ERR_ARG, "wl_session_open: beam_size / num_hypotheses must be >= 1");
  const int K = o->beam_size, Kr = K > 1 ? K : o->num_hypotheses;
  WL_CHECK(Kr <= c->Km, WL_ERR_ARG, "wl_session_open: %d rows per stream exceed max_beam=%d", Kr, c->Km);
  WL_CHECK(K == 1 || o->num_hypotheses <= MAX_FINISHED, WL_ERR_ARG, "too many hypotheses");
  // the session's own search is beam or greedy: sampling is chosen per stream at admission (wl_session_admit_ex), where
  // each sampled stream brings the seed and noise key its draws are keyed by
  WL_CHECK(!(K == 1 && o->sampling_topk == 0 && o->sampling_temperature > 0.f), WL_ERR_ARG,
           "wl_session_open: sampling is chosen per stream at admission (wl_session_admit_ex), not for the session");
  if (!ss.allocated) {
    alloc_decode_state(c, ss.ds);
    ss.kcache = c->mem.alloc<__half>((size_t)c->Ld * c->cache_layer_stride, false);
    ss.vcache = c->mem.alloc<__half>((size_t)c->Ld * c->cache_layer_stride, false);
    ss.mask = c->mem.alloc<unsigned>((c->V + 31) / 32 + 1);
    // per-stream logits rules: the captured loop reads them, admission writes them (6.5 KB of mask per index at 51866)
    DecodeState& sd = ss.ds;
    sd.mask_words = (c->V + 31) / 32 + 1;
    sd.r_max_initial = c->mem.alloc<int>(c->Bm); sd.r_suppress_blank = c->mem.alloc<int>(c->Bm);
    sd.r_max_cand = c->mem.alloc<int>(c->Bm); sd.r_length_penalty = c->mem.alloc<float>(c->Bm);
    sd.r_beam = c->mem.alloc<int>(c->Bm);
    sd.r_mask = c->mem.alloc<unsigned>((size_t)c->Bm * sd.mask_words);
    ss.idx_dev = c->mem.alloc<int>(c->Bm);
    ss.peek_dev = c->mem.alloc<int>((size_t)c->Bm * PEEK_STRIDE);
    ss.allocated = true;
  }
  ss.cap = capacity; ss.K = K; ss.Kr = Kr; ss.NH = o->num_hypotheses; ss.length_penalty = o->length_penalty;
  ss.use_graph = o->use_cuda_graph;
  SearchOpts& so = ss.so;
  so.beam = K; so.rows_per_stream = Kr;
  so.max_cand = max_candidates(K, o->patience, "wl_session_open");
  so.suppress_blank = o->suppress_blank; so.max_initial_ts = o->max_initial_timestamp_index;
  so.suppress_mask = ss.mask;
  ss.nsplit = cross_attn_pick_nsplit(capacity, c->H, c->num_sms, Kr);
  const int nwords = (c->V + 31) / 32 + 1;
  std::vector<unsigned> mask(nwords, 0u);
  for (int i = 0; i < o->n_suppress; ++i) {
    const int t = o->suppress_tokens[i];
    if (t >= 0 && t < c->V) mask[t >> 5] |= 1u << (t & 31);
  }
  const int cap = capacity, R = cap * Kr;
  ss.hp.assign((size_t)cap * T_MAX, 0);
  ss.meta.assign((size_t)META_ROWS * cap, 0);
  for (int b = 0; b < cap; ++b) {   // harmless idle values
    ss.meta[1 * cap + b] = 1; ss.meta[2 * cap + b] = -1; ss.meta[4 * cap + b] = 1;
    search_meta(ss.meta.data(), b, cap, 0, 0.f, 0u, b, Kr);
  }
  ss.used.assign(cap, 0);
  ss.finished.assign(cap, 0);
  ss.nh.assign(cap, ss.NH);
  ss.rules.assign((size_t)RULE_ROWS * cap, 0);
  ss.lp.assign(cap, ss.length_penalty);
  ss.script_on = false;
  ss.live = 0;
  cudaStream_t st = c->st;
  const DecodeState& s = ss.ds;
  std::vector<int> ones(cap, 1);
  const int nd = cap, brk0[2] = {0, 0};
  WL_CUDA(cudaMemcpyAsync(ss.mask, mask.data(), nwords * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(s.done, ones.data(), cap * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemsetAsync(s.active, 0, (size_t)R * 4, st));
  WL_CUDA(cudaMemsetAsync(s.hyp_count, 0, (size_t)cap * 4, st));
  WL_CUDA(cudaMemcpyAsync(s.n_done, &nd, 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(s.brk, brk0, 8, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaStreamSynchronize(st));   // the host vectors above go out of scope
  ss.open = true;
  API_END(c)
}

extern "C" int wl_session_admit(wl_ctx* c, int32_t n, const int32_t* index, const int32_t* slots, const int32_t* prompts,
                                const int32_t* prompt_off, const int32_t* max_length) {
  return wl_session_admit_ex(c, n, index, slots, prompts, prompt_off, max_length, nullptr, nullptr);
}

// beam width of a stream admitted with these rules (nullptr: none): its own, or 0 for the session's
static int stream_width(const wl_ctx::Session& ss, const wl_stream_rules* q) {
  return q && q->rules && q->beam_size ? q->beam_size : ss.K;
}

// a stream's own logits rules, checked before anything is staged; every message names the field
static void check_stream_rules(const wl_ctx::Session& ss, int i, const wl_stream_rules& q) {
  WL_CHECK(q.rules == 1, WL_ERR_ARG, "wl_session_admit: stream %d: rules must be 0 or 1, got %d", i, q.rules);
  // a width needs that many rows of the stream's index; a greedy stream runs the session's num_hypotheses rows, as
  // wl_generate(beam_size = 1) does
  WL_CHECK(q.beam_size >= 0 && q.beam_size <= ss.Kr, WL_ERR_ARG,
           "wl_session_admit: stream %d: beam_size %d must be 0 (the session's) or 1 .. %d (rows per stream)", i,
           q.beam_size, ss.Kr);
  WL_CHECK(q.beam_size != 1 || ss.NH <= ss.Kr, WL_ERR_ARG,
           "wl_session_admit: stream %d: beam_size 1 decodes num_hypotheses = %d greedy rows, more than the %d rows per stream",
           i, ss.NH, ss.Kr);
  WL_CHECK(std::isfinite(q.patience) && q.patience > 0.f, WL_ERR_ARG, "wl_session_admit: stream %d: patience %g must be finite and > 0",
           i, (double)q.patience);
  char who[80];
  snprintf(who, sizeof(who), "wl_session_admit: stream %d: patience x beam_size", i);
  max_candidates(stream_width(ss, &q), q.patience, who);
  WL_CHECK(std::isfinite(q.length_penalty), WL_ERR_ARG, "wl_session_admit: stream %d: length_penalty %g is not finite", i,
           (double)q.length_penalty);
  WL_CHECK(q.max_initial_timestamp_index >= 0, WL_ERR_ARG, "wl_session_admit: stream %d: negative max_initial_timestamp_index %d",
           i, q.max_initial_timestamp_index);
  WL_CHECK(q.n_suppress >= 0 && (q.n_suppress == 0 || q.suppress_tokens), WL_ERR_ARG,
           "wl_session_admit: stream %d: suppress_tokens is null for n_suppress %d", i, q.n_suppress);
}

extern "C" int wl_session_admit_ex(wl_ctx* c, int32_t n, const int32_t* index, const int32_t* slots, const int32_t* prompts,
                                   const int32_t* prompt_off, const int32_t* max_length, const wl_stream_search* search,
                                   const wl_stream_rules* rules) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  WL_CHECK(ss.open, WL_ERR_STATE, "wl_session_admit: no open session");
  WL_CHECK(n >= 1 && index && slots && prompts && prompt_off && max_length, WL_ERR_ARG, "wl_session_admit: bad arguments");
  const int cap = ss.cap;
  for (int i = 0; i < n; ++i) {
    WL_CHECK(index[i] >= 0 && index[i] < cap, WL_ERR_ARG, "wl_session_admit: index %d outside the session capacity %d", index[i], cap);
    WL_CHECK(!ss.used[index[i]], WL_ERR_STATE, "wl_session_admit: index %d still holds a stream", index[i]);
    for (int j = 0; j < i; ++j) WL_CHECK(index[j] != index[i], WL_ERR_ARG, "wl_session_admit: index %d listed twice", index[i]);
    if (search && search[i].sample) {
      const wl_stream_search& q = search[i];
      WL_CHECK(q.sample == 1, WL_ERR_ARG, "wl_session_admit: stream %d: sample must be 0 or 1, got %d", i, q.sample);
      WL_CHECK(q.num_hypotheses >= 1 && q.num_hypotheses <= ss.Kr, WL_ERR_ARG,
               "wl_session_admit: stream %d: %d sampled hypotheses outside 1 .. %d rows per stream", i, q.num_hypotheses, ss.Kr);
      WL_CHECK(std::isfinite(q.temperature) && q.temperature > 0.f, WL_ERR_ARG,
               "wl_session_admit: stream %d: sampling temperature %g must be finite and > 0", i, (double)q.temperature);
      WL_CHECK(q.noise_key >= 0, WL_ERR_ARG, "wl_session_admit: stream %d: negative noise key %d", i, q.noise_key);
    }
    if (rules && rules[i].rules) check_stream_rules(ss, i, rules[i]);
  }
  // validate + stage everything before touching the session (a bad prompt must not leave a half-admitted stream)
  std::vector<int> hp = ss.hp, meta = ss.meta, rl = ss.rules;
  const int nwords = ss.ds.mask_words;
  std::vector<unsigned> masks;   // [n][nwords]: the own suppress lists, in admission order (empty rows unused)
  if (rules) masks.assign((size_t)n * nwords, 0u);
  for (int i = 0; i < n; ++i) {
    stream_meta(c, i, slots[i], prompts + prompt_off[i], prompt_off[i + 1] - prompt_off[i], max_length[i], false,
                hp.data() + (size_t)index[i] * T_MAX, meta.data(), index[i], cap, nullptr, !ss.script_on);
    const bool sample = search && search[i].sample;
    const bool own = rules && rules[i].rules;
    const int width = stream_width(ss, rules ? rules + i : nullptr);
    // rows a stream without a beam uses: its samples, or greedy's num_hypotheses (= Kr in a greedy session)
    search_meta(meta.data(), index[i], cap, sample ? 1 : 0, sample ? search[i].temperature : 0.f, sample ? search[i].seed : 0u,
                sample ? search[i].noise_key : index[i], sample ? search[i].num_hypotheses : (width == 1 ? ss.NH : ss.Kr));
    const float lp = own ? rules[i].length_penalty : ss.length_penalty;
    int lbits;
    memcpy(&lbits, &lp, 4);
    const int b = index[i];
    rl[0 * cap + b] = own ? rules[i].max_initial_timestamp_index : ss.so.max_initial_ts;
    rl[1 * cap + b] = own ? (rules[i].suppress_blank ? 1 : 0) : ss.so.suppress_blank;
    rl[2 * cap + b] = own ? max_candidates(width, rules[i].patience, "wl_session_admit") : ss.so.max_cand;
    rl[3 * cap + b] = lbits;
    rl[4 * cap + b] = width;
    if (own)
      for (int k = 0; k < rules[i].n_suppress; ++k) {
        const int t = rules[i].suppress_tokens[k];
        if (t >= 0 && t < c->V) masks[(size_t)i * nwords + (t >> 5)] |= 1u << (t & 31);
      }
  }
  ss.hp.swap(hp);
  ss.meta.swap(meta);
  ss.rules.swap(rl);
  for (int i = 0; i < n; ++i) {
    ss.nh[index[i]] = (search && search[i].sample) ? search[i].num_hypotheses : ss.NH;
    ss.lp[index[i]] = (rules && rules[i].rules) ? rules[i].length_penalty : ss.length_penalty;
  }
  ensure_host(c, (size_t)cap * (T_MAX + 16) + n + (size_t)RULE_ROWS * cap, 16);
  int* php = c->h_int;
  int* pmeta = php + (size_t)cap * T_MAX;
  int* pidx = pmeta + (size_t)META_ROWS * cap;
  int* prules = pidx + n;
  memcpy(php, ss.hp.data(), ss.hp.size() * 4);
  memcpy(pmeta, ss.meta.data(), ss.meta.size() * 4);
  memcpy(pidx, index, (size_t)n * 4);
  memcpy(prules, ss.rules.data(), ss.rules.size() * 4);
  cudaStream_t st = c->st;
  WL_CUDA(cudaEventRecord(c->ev0, st));
  {
    // the rule tables of the session state (written like the others with what the streams in flight already hold) and
    // each admitted index's suppress mask: its own list, or a copy of the session's
    const DecodeState& sd = ss.ds;
    void* dst[RULE_ROWS] = {sd.r_max_initial, sd.r_suppress_blank, sd.r_max_cand, sd.r_length_penalty, sd.r_beam};
    for (int k = 0; k < RULE_ROWS; ++k) WL_CUDA(cudaMemcpyAsync(dst[k], prules + (size_t)k * cap, cap * 4, cudaMemcpyHostToDevice, st));
    for (int i = 0; i < n; ++i) {
      unsigned* m = sd.r_mask + (size_t)index[i] * nwords;
      if (rules && rules[i].rules)
        WL_CUDA(cudaMemcpyAsync(m, masks.data() + (size_t)i * nwords, (size_t)nwords * 4, cudaMemcpyHostToDevice, st));
      else
        WL_CUDA(cudaMemcpyAsync(m, ss.mask, (size_t)nwords * 4, cudaMemcpyDeviceToDevice, st));
    }
  }
  SessScope scope(c);
  // the tables of the streams in flight are rewritten with the values they already hold (nothing runs between two calls)
  upload_state_tables(c, php, pmeta, cap);
  WL_CUDA(cudaMemcpyAsync(ss.idx_dev, pidx, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaStreamSynchronize(st));   // `masks` goes out of scope
  if (ss.script_on)   // scripted logits: no decoder pass; the no-speech probability comes from the script
    scripted_no_speech(st, c->ds, vocab_ids(c), ss.script, n, ss.idx_dev);
  else
    prefill_forward(c, n, ss.Kr, ss.hp.data(), ss.meta.data() + 1 * cap, ss.meta.data() + 2 * cap, slots, index);
  decode_init(st, c->ds, ss.so, vocab_ids(c), n, cap * ss.Kr, 1, ss.idx_dev);
  WL_CUDA(cudaEventRecord(c->ev1, st));
  WL_CUDA(cudaStreamSynchronize(st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[5], c->ev0, c->ev1));
  for (int i = 0; i < n; ++i) { ss.used[index[i]] = 1; ss.finished[index[i]] = 0; }
  ss.live += n;
  ss.admitted += n;
  API_END(c)
}

extern "C" int wl_test_session_script(wl_ctx* c, const wl_search_script* script) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  WL_CHECK(ss.open, WL_ERR_STATE, "wl_test_session_script: no open session");
  WL_CHECK(ss.live == 0, WL_ERR_STATE, "wl_test_session_script: %d streams are still decoding", ss.live);
  if (script) {
    WL_CHECK(script->pattern >= -1 && script->pattern <= 5, WL_ERR_ARG, "wl_test_session_script: pattern %d out of range",
             script->pattern);
    ss.script.seed = script->seed;
    ss.script.pattern = script->pattern;
  }
  ss.script_on = script != nullptr;
  API_END(c)
}

extern "C" int wl_session_run(wl_ctx* c, int32_t max_steps, int32_t break_on_finish, int32_t* done_out, int32_t* steps_ran) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  WL_CHECK(ss.open, WL_ERR_STATE, "wl_session_run: no open session");
  WL_CHECK(max_steps >= 1 && done_out, WL_ERR_ARG, "wl_session_run: bad arguments");
  const int cap = ss.cap;
  int ran = 0;
  c->last_ms[2] = 0.f;
  if (ss.live > 0) {
    SessScope scope(c);
    cudaStream_t st = c->st;
    const VocabIds vi = vocab_ids(c);
    ensure_host(c, (size_t)cap + 16, 16);
    int* h = c->h_int;
    h[0] = max_steps; h[1] = break_on_finish ? 1 : 0; h[2] = cap - ss.live;
    WL_CUDA(cudaMemcpyAsync(c->ds.steps_left, h, 4, cudaMemcpyHostToDevice, st));
    WL_CUDA(cudaMemcpyAsync(c->ds.brk, h + 1, 8, cudaMemcpyHostToDevice, st));
    WL_CUDA(cudaEventRecord(c->ev0, st));
    if (ss.use_graph) {
      long kernels = 0;
      cudaGraphExec_t exec = decode_graph(c, "s", cap, ss.Kr, ss.K, ss.so, vi, ss.nsplit, &kernels, ss.script_on ? &ss.script : nullptr);
      WL_CUDA(cudaGraphLaunch(exec, st));
      WL_CUDA(cudaMemcpyAsync(h + 4, c->ds.steps_left, 4, cudaMemcpyDeviceToHost, st));
      WL_CUDA(cudaMemcpyAsync(h + 8, c->ds.done, (size_t)cap * 4, cudaMemcpyDeviceToHost, st));
      WL_CUDA(cudaEventRecord(c->ev1, st));
      WL_CUDA(cudaStreamSynchronize(st));
      ran = max_steps - h[4];
      c->graph_launched += kernels * (long)ran;
    } else {   // graph-less (profiling / bisecting): the same loop condition evaluated on the host after every step
      for (;;) {
        token_step(c, cap, ss.Kr, ss.so, vi, ss.nsplit, ss.script_on ? &ss.script : nullptr);
        ++ran;
        WL_CUDA(cudaMemcpyAsync(h + 5, c->ds.n_done, 4, cudaMemcpyDeviceToHost, st));
        WL_CUDA(cudaStreamSynchronize(st));
        if (ran >= max_steps || h[5] >= cap || (break_on_finish && h[5] > h[2])) break;
      }
      WL_CUDA(cudaMemcpyAsync(h + 8, c->ds.done, (size_t)cap * 4, cudaMemcpyDeviceToHost, st));
      WL_CUDA(cudaEventRecord(c->ev1, st));
      WL_CUDA(cudaStreamSynchronize(st));
    }
    WL_CUDA(cudaEventElapsedTime(&c->last_ms[2], c->ev0, c->ev1));
    for (int b = 0; b < cap; ++b)
      if (ss.used[b] && !ss.finished[b] && h[8 + b]) { ss.finished[b] = 1; ss.live -= 1; }
    ss.steps += ran;
    ss.runs += 1;
  }
  for (int b = 0; b < cap; ++b) done_out[b] = (ss.used[b] && ss.finished[b]) ? 1 : 0;
  if (steps_ran) *steps_ran = ran;
  API_END(c)
}

extern "C" int wl_session_collect(wl_ctx* c, int32_t index, int32_t* out_ids, int32_t* out_len, float* out_score, float* out_no_speech,
                                  int32_t* out_steps) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  WL_CHECK(ss.open, WL_ERR_STATE, "wl_session_collect: no open session");
  WL_CHECK(index >= 0 && index < ss.cap && out_ids && out_len && out_score, WL_ERR_ARG, "wl_session_collect: bad arguments");
  WL_CHECK(ss.used[index] && ss.finished[index], WL_ERR_STATE, "wl_session_collect: stream index %d has not finished", index);
  const DecodeState& s = ss.ds;
  cudaStream_t st = c->st;
  ensure_host(c, (size_t)MAX_HYPS * (T_MAX + 2) + 16, MAX_HYPS + 2);
  int* h_cnt = c->h_int;
  int* h_steps = h_cnt + 1;
  int* h_len = h_cnt + 8;
  int* h_tok = h_len + MAX_HYPS;
  float* h_cum = c->h_flt;
  float* h_ns = h_cum + MAX_HYPS;
  WL_CUDA(cudaMemcpyAsync(h_cnt, s.hyp_count + index, 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_steps, s.steps_run + index, 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_len, s.hyp_len + (size_t)index * MAX_HYPS, MAX_HYPS * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_tok, s.hyp_tok + (size_t)index * MAX_HYPS * T_MAX, (size_t)MAX_HYPS * T_MAX * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_cum, s.hyp_cum + (size_t)index * MAX_HYPS, MAX_HYPS * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(h_ns, s.no_speech + index, 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  emit_hyps(ss.nh[index], ss.lp[index], h_cnt[0], h_len, h_cum, h_tok, out_ids, out_len, out_score);
  if (out_no_speech) *out_no_speech = h_ns[0];
  if (out_steps) *out_steps = h_steps[0];
  ss.used[index] = 0;
  ss.finished[index] = 0;
  API_END(c)
}

// every listed index must hold a stream (running, or finished and not yet collected); checked before anything launches
static void check_session_indices(const wl_ctx::Session& ss, int n, const int32_t* index, bool distinct, const char* what) {
  WL_CHECK(ss.open, WL_ERR_STATE, "%s: no open session", what);
  WL_CHECK(n >= 1 && n <= ss.cap && index, WL_ERR_ARG, "%s: bad arguments (%d indices, capacity %d)", what, n, ss.cap);
  for (int i = 0; i < n; ++i) {
    WL_CHECK(index[i] >= 0 && index[i] < ss.cap, WL_ERR_ARG, "%s: index %d outside the session capacity %d", what, index[i], ss.cap);
    WL_CHECK(ss.used[index[i]], WL_ERR_STATE, "%s: index %d is idle", what, index[i]);
    if (distinct)
      for (int j = 0; j < i; ++j) WL_CHECK(index[j] != index[i], WL_ERR_ARG, "%s: index %d listed twice", what, index[i]);
  }
}

extern "C" int wl_session_peek(wl_ctx* c, int32_t n, const int32_t* index, int32_t* out_ids, int32_t* out_len, float* out_score,
                               float* out_no_speech, int32_t* out_step, int32_t* out_final) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  check_session_indices(ss, n, index, false, "wl_session_peek");
  WL_CHECK(out_ids && out_len && out_score, WL_ERR_ARG, "wl_session_peek: bad arguments");
  cudaStream_t st = c->st;
  ensure_host(c, (size_t)n * PEEK_STRIDE + n, 16);
  int* h = c->h_int;
  int* hidx = h + (size_t)n * PEEK_STRIDE;
  memcpy(hidx, index, (size_t)n * 4);
  WL_CUDA(cudaMemcpyAsync(ss.idx_dev, hidx, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  session_peek(st, ss.ds, ss.so, ss.length_penalty, ss.idx_dev, ss.peek_dev, n);
  WL_CUDA(cudaMemcpyAsync(h, ss.peek_dev, (size_t)n * PEEK_STRIDE * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    const int* e = h + (size_t)i * PEEK_STRIDE;
    int len = e[0];
    float cum, ns;
    memcpy(&cum, e + 1, 4);
    memcpy(&ns, e + 2, 4);
    int best = e[5];
    if (e[4]) {   // finished: rank its hypotheses with emit_hyps' arithmetic (first of the best scores)
      float bs = 0.f;
      for (int k = 0; k < e[6]; ++k) {
        float ck;
        memcpy(&ck, e + PEEK_TAB + MAX_HYPS + k, 4);
        const float sc = hyp_score(ck, e[PEEK_TAB + k], ss.lp[index[i]]);
        if (k == 0 || sc > bs) { best = k; bs = sc; }
      }
    }
    if (e[4] && best != e[5]) {   // a last-bit near-tie the device's powf ranked the other way: fetch the host's pick
      len = e[PEEK_TAB + best];
      memcpy(&cum, e + PEEK_TAB + MAX_HYPS + best, 4);
      if (len > 0)
        WL_CUDA(cudaMemcpy(out_ids + (size_t)i * T_MAX, ss.ds.hyp_tok + ((size_t)index[i] * MAX_HYPS + best) * T_MAX,
                           (size_t)len * 4, cudaMemcpyDeviceToHost));
    } else if (len > 0) {
      memcpy(out_ids + (size_t)i * T_MAX, e + PEEK_HDR, (size_t)len * 4);
    }
    out_len[i] = len;
    out_score[i] = len < 0 ? 0.f : hyp_score(cum, len, ss.lp[index[i]]);
    if (out_no_speech) out_no_speech[i] = ns;
    if (out_step) out_step[i] = e[3];
    if (out_final) out_final[i] = e[4];
  }
  API_END(c)
}

extern "C" int wl_session_cancel(wl_ctx* c, int32_t n, const int32_t* index) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  check_session_indices(ss, n, index, true, "wl_session_cancel");
  cudaStream_t st = c->st;
  ensure_host(c, (size_t)n, 16);
  memcpy(c->h_int, index, (size_t)n * 4);
  WL_CUDA(cudaMemcpyAsync(ss.idx_dev, c->h_int, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  session_cancel(st, ss.ds, ss.Kr, ss.idx_dev, n);
  WL_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    const int b = index[i];
    if (!ss.finished[b]) ss.live -= 1;
    ss.used[b] = 0;
    ss.finished[b] = 0;
  }
  API_END(c)
}

extern "C" int wl_session_close(wl_ctx* c) {
  API_BEGIN(c)
  wl_ctx::Session& ss = c->sess;
  if (ss.open) {   // streams still in flight are dropped: their indices go idle again
    const int cap = ss.cap;
    std::vector<int> ones(cap, 1);
    const int nd = cap;
    WL_CUDA(cudaMemcpy(ss.ds.done, ones.data(), (size_t)cap * 4, cudaMemcpyHostToDevice));
    WL_CUDA(cudaMemset(ss.ds.active, 0, (size_t)cap * ss.Kr * 4));
    WL_CUDA(cudaMemcpy(ss.ds.n_done, &nd, 4, cudaMemcpyHostToDevice));
    ss.used.assign(cap, 0);
    ss.finished.assign(cap, 0);
    ss.live = 0;
    ss.open = false;
  }
  API_END(c)
}

// teacher-forced driver shared by wl_decode_logits / wl_detect_language / wl_align
static void forced_run(wl_ctx* c, const int32_t* slots, int B, const int32_t* tokens, const int32_t* off, bool align_mode,
                       float* logits_out_dev /* [sumT][V] or null */, const std::vector<long>& row_base) {
  SearchOpts so;
  memset(&so, 0, sizeof(so));
  so.beam = 1; so.rows_per_stream = 1; so.max_cand = 1; so.suppress_mask = c->suppress_mask;
  const VocabIds vi = vocab_ids(c);
  cudaStream_t st = c->st;
  const int max_steps = upload_streams(c, slots, B, tokens, off, T_MAX, true, 0, 0.f, 0u, 1);
  decode_init(st, c->ds, so, vi, B, B);
  const int nsplit = align_mode ? 1 : cross_attn_pick_nsplit(B, c->H, c->num_sms, 1);
  for (int i = 0; i < max_steps; ++i) {
    decode_step(c, B, 1, so, vi, nsplit, align_mode);
    if (logits_out_dev)
      for (int b = 0; b < B; ++b)
        if (i < off[b + 1] - off[b])
          WL_CUDA(cudaMemcpyAsync(logits_out_dev + (row_base[b] + i) * c->V, c->logits + (long)b * c->Vld, (size_t)c->V * 4,
                                  cudaMemcpyDeviceToDevice, st));
  }
  WL_CUDA(cudaStreamSynchronize(st));
}

extern "C" int wl_decode_logits(wl_ctx* c, const int32_t* slots, int32_t B, const int32_t* tokens, const int32_t* tok_off,
                                float* logits_out) {
  API_BEGIN(c)
  WL_CHECK(c->finalized && slots && tokens && tok_off && logits_out && B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_decode_logits: bad arguments");
  std::vector<long> base(B);
  long tot = 0;
  for (int b = 0; b < B; ++b) { base[b] = tot; tot += tok_off[b + 1] - tok_off[b]; }
  Scratch sc(c->st);
  float* dev = sc.alloc<float>((size_t)tot * c->V);
  forced_run(c, slots, B, tokens, tok_off, false, dev, base);
  sc.download(logits_out, dev, (size_t)tot * c->V);
  API_END(c)
}

extern "C" int wl_detect_language(wl_ctx* c, const int32_t* slots, int32_t B, float* probs) {
  API_BEGIN(c)
  WL_CHECK(c->finalized && slots && probs && B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_detect_language: bad arguments");
  WL_CHECK(c->cfg.n_lang > 0, WL_ERR_STATE, "detect_language can only be called on multilingual models");
  std::vector<int32_t> toks(B, c->cfg.sot), off(B + 1);
  std::vector<long> base(B);
  for (int b = 0; b <= B; ++b) off[b] = b;
  forced_run(c, slots, B, toks.data(), off.data(), false, nullptr, base);
  const int nl = c->cfg.n_lang;
  std::vector<float> lg((size_t)B * nl);
  for (int b = 0; b < B; ++b)
    WL_CUDA(cudaMemcpy(lg.data() + (size_t)b * nl, c->logits + (long)b * c->Vld + c->cfg.lang_begin, nl * 4, cudaMemcpyDeviceToHost));
  for (int b = 0; b < B; ++b) {
    float mx = -INFINITY;
    for (int i = 0; i < nl; ++i) mx = std::max(mx, lg[(size_t)b * nl + i]);
    double sum = 0;
    for (int i = 0; i < nl; ++i) sum += exp((double)lg[(size_t)b * nl + i] - mx);
    for (int i = 0; i < nl; ++i) probs[(size_t)b * nl + i] = (float)(exp((double)lg[(size_t)b * nl + i] - mx) / sum);
  }
  API_END(c)
}

// ------------------------------------------------------------------------------------------ K14 align
extern "C" int wl_align(wl_ctx* c, const int32_t* slots, int32_t B, const int32_t* start_seq, int32_t n_start, const int32_t* text,
                        const int32_t* text_off, const int32_t* num_frames, int32_t median_width, int32_t* pairs_out,
                        int32_t cap_pairs, int32_t* pair_off, float* tok_probs) {
  API_BEGIN(c)
  WL_CHECK(c->finalized && slots && start_seq && text && text_off && num_frames && pairs_out && pair_off && tok_probs, WL_ERR_ARG,
           "wl_align: null argument");
  WL_CHECK(B >= 1 && B <= c->Bm, WL_ERR_ARG, "wl_align: B=%d exceeds max_streams", B);
  const int nh = (int)c->align_heads.size() / 2;
  WL_CHECK(nh > 0, WL_ERR_STATE, "wl_align: no alignment heads configured");
  std::vector<int32_t> toks, off(B + 1);
  std::vector<long> base(B, 0);
  int maxT = 0;
  off[0] = 0;
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < n_start; ++i) toks.push_back(start_seq[i]);
    toks.push_back(c->cfg.no_timestamps);
    for (int i = text_off[b]; i < text_off[b + 1]; ++i) toks.push_back(text[i]);
    toks.push_back(c->cfg.eot);
    off[b + 1] = (int)toks.size();
    maxT = std::max(maxT, off[b + 1] - off[b]);
  }
  WL_CHECK(maxT <= T_MAX, WL_ERR_ARG, "wl_align: sequence of %d tokens exceeds %d", maxT, T_MAX);
  const long need_buf = (long)B * nh * T_MAX * S_ENC;
  c->mem.grow(c->align_buf, c->align_buf_cap, need_buf);
  for (int b = 0; b < B; ++b)
    WL_CHECK(slots[b] >= 0 && slots[b] < c->NS && c->slot_used[slots[b]], WL_ERR_ARG, "wl_align: stream %d: bad encoder slot %d", b, slots[b]);
  // ---- teacher-forced pass: every position of every stream at once (the K8 machinery), attention probabilities of
  // the alignment heads captured on the way
  std::vector<int> ntok(B);
  for (int b = 0; b < B; ++b) ntok[b] = off[b + 1] - off[b];
  const PfRows r = pf_rows(B, 1, toks.data(), off.data(), ntok.data(), slots);
  pf_stack(c, r, true);
  wl_ctx::Prefill& f = c->pf;
  cudaStream_t st = c->st;
  // ---- P(text token | prefix): the logits row that predicts it
  const int n_text = text_off[B] - text_off[0];
  if (n_text > 0) {
    c->mem.grow(f.tokp, f.tokp_cap, n_text, n_text + 256, true);
    std::vector<int> sel, tgt, oidx;
    for (int b = 0; b < B; ++b)
      for (int i = 0; i < text_off[b + 1] - text_off[b]; ++i) {
        sel.push_back(r.rowbase[b] + n_start + i);
        tgt.push_back(toks[off[b] + n_start + 1 + i]);
        oidx.push_back(text_off[b] - text_off[0] + i);
      }
    pf_row_probs(c, sel, tgt, oidx, f.tokp);
    WL_CUDA(cudaMemcpy(tok_probs + text_off[0], f.tokp, (size_t)n_text * 4, cudaMemcpyDeviceToHost));
  }
  // ---- standardise / median filter / mean over heads / DTW on the device
  if (!f.mat) {
    f.mat = c->mem.alloc<float>((size_t)c->Bm * T_MAX * S_ENC, false);
    f.aT = c->mem.alloc<int>(c->Bm); f.anf = c->mem.alloc<int>(c->Bm);
    f.path = c->mem.alloc<int>((size_t)c->Bm * (T_MAX + S_ENC + 2) * 2, false);
    f.path_len = c->mem.alloc<int>(c->Bm);
  }
  const int path_cap = T_MAX + S_ENC + 2;
  std::vector<int> hT(B), hnf(B);
  for (int b = 0; b < B; ++b) {
    hT[b] = ntok[b];
    hnf[b] = std::max(1, std::min(num_frames[b] / 2, (int)S_ENC));
  }
  WL_CUDA(cudaMemcpyAsync(f.aT, hT.data(), B * 4, cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(f.anf, hnf.data(), B * 4, cudaMemcpyHostToDevice, st));
  align_postprocess(st, c->align_buf, f.mat, f.aT, f.anf, B, nh, median_width, n_start, maxT, f.path, path_cap, f.path_len);
  std::vector<int> hlen(B), hpath((size_t)B * path_cap * 2);
  WL_CUDA(cudaMemcpyAsync(hlen.data(), f.path_len, B * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaMemcpyAsync(hpath.data(), f.path, hpath.size() * 4, cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  int np_total = 0;
  pair_off[0] = 0;
  for (int b = 0; b < B; ++b) {
    const int len = hlen[b];
    WL_CHECK(np_total + len <= cap_pairs, WL_ERR_ARG, "wl_align: pairs_out capacity %d too small", cap_pairs);
    const int* pp = hpath.data() + (size_t)b * path_cap * 2;
    for (int k = len - 1; k >= 0; --k) {   // the device wrote the path end -> start
      pairs_out[2 * np_total] = pp[2 * k];
      pairs_out[2 * np_total + 1] = pp[2 * k + 1];
      ++np_total;
    }
    pair_off[b + 1] = np_total;
  }
  API_END(c)
}
