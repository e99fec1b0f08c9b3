// Translation context and C ABI (include/wlb200.h, wl_mt_*): M2M100 encoder over the packed source tokens of a call, the
// decoder's cross K/V once per call, then the token loop (decoder step + beam-search step) as one CUDA graph with a
// conditional WHILE node, so no host synchronisation happens per token.
#include <cmath>
#include <cstring>

#include "ctx.cuh"
#include "mt.cuh"

namespace wl {
void gemm_prime();
}

struct MtTensor {
  std::vector<int64_t> shape;
  bool f16 = false;
  void* p = nullptr;
};

struct wl_mt_ctx {
  wl_mt_config cfg;
  int Bc = 0, Km = 0, Ns = 0, Rm = 0, Vld = 0;
  int d = 0, H = 0, ff = 0, Le = 0, Ld = 0, V = 0;
  cudaStream_t st = nullptr;
  std::string err;
  std::map<std::string, MtTensor> w;
  bool finalized = false;
  DeviceMem mem;
  // encoder
  float* ex = nullptr;
  __half *eh = nullptr, *eqkv = nullptr, *eattn = nullptr, *eff = nullptr, *xkv = nullptr;
  int *etok = nullptr, *etpos = nullptr, *eoff = nullptr;
  int2* etiles = nullptr;
  // decoder
  float *dx = nullptr, *dqkv = nullptr, *dq = nullptr, *logits = nullptr;
  __half *dh = nullptr, *dattn = nullptr, *dff = nullptr, *kc = nullptr, *vc = nullptr;
  MtState s;
  std::map<std::string, cudaGraphExec_t> graphs;
};

static std::string g_mt_init_error;

static void mt_free(wl_mt_ctx* c) {
  for (auto& kv : c->graphs) cudaGraphExecDestroy(kv.second);
  c->mem.release_from(0);
  if (c->st) cudaStreamDestroy(c->st);
}

// engine tensor table: name -> shape (fp16 for the matrices, fp32 for biases, LayerNorms and the position table)
static void mt_table(wl_mt_ctx* c) {
  const int64_t d = c->d, ff = c->ff, V = c->V, P = c->cfg.max_positions + 2;
  auto add = [&](const std::string& n, std::vector<int64_t> sh, bool f16) { c->w[n] = MtTensor{sh, f16, nullptr}; };
  add("shared", {V, d}, true);
  add("positions", {P, d}, false);
  auto ln = [&](const std::string& n) { add(n + ".w", {d}, false); add(n + ".b", {d}, false); };
  auto lin = [&](const std::string& n, int64_t o, int64_t i) { add(n + ".w", {o, i}, true); add(n + ".b", {o}, false); };
  for (int l = 0; l < c->Le; ++l) {
    const std::string p = "enc." + std::to_string(l);
    ln(p + ".ln1"); ln(p + ".ln2");
    lin(p + ".qkv", 3 * d, d); lin(p + ".out", d, d); lin(p + ".fc1", ff, d); lin(p + ".fc2", d, ff);
  }
  ln("enc.ln");
  for (int l = 0; l < c->Ld; ++l) {
    const std::string p = "dec." + std::to_string(l);
    ln(p + ".ln1"); ln(p + ".ln2"); ln(p + ".ln3");
    lin(p + ".qkv", 3 * d, d); lin(p + ".out", d, d); lin(p + ".xq", d, d); lin(p + ".xout", d, d);
    lin(p + ".fc1", ff, d); lin(p + ".fc2", d, ff);
  }
  ln("dec.ln");
  lin("dec.xkv", 2 * d * c->Ld, d);
}

template <class T>
static const T* W(wl_mt_ctx* c, const std::string& n) { return (const T*)c->w.at(n).p; }

extern "C" int wl_mt_init(const wl_mt_config* cfg, int32_t device, int32_t capacity_segments, int32_t max_beam, wl_mt_ctx** out) {
  if (!cfg || !out) return WL_ERR_ARG;
  *out = nullptr;
  wl_mt_ctx* c = new wl_mt_ctx();
  try {
    WL_CHECK(cfg->abi_version == WL_ABI_VERSION, WL_ERR_ARG, "ABI version mismatch: header %d, caller %d", WL_ABI_VERSION,
             cfg->abi_version);
    int ndev = 0;
    WL_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0, WL_ERR_CUDA, "no CUDA device available: libwlb200 has no CPU fallback");
    WL_CHECK(device >= 0 && device < ndev, WL_ERR_ARG, "device %d out of range (%d devices)", device, ndev);
    WL_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    WL_CUDA(cudaGetDeviceProperties(&prop, device));
    WL_CHECK(prop.major == 9 && prop.minor == 0, WL_ERR_CUDA, "libwlb200 is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
    c->cfg = *cfg;
    c->mem.device = device;
    c->d = cfg->d_model; c->H = cfg->n_heads; c->ff = cfg->ffn; c->Le = cfg->enc_layers; c->Ld = cfg->dec_layers; c->V = cfg->vocab;
    WL_CHECK(c->H >= 1 && c->d == 64 * c->H && c->d <= 1280, WL_ERR_ARG, "wl_mt_init: d_model %d / heads %d unsupported (head dim 64)", c->d, c->H);
    WL_CHECK(c->ff >= 64 && c->ff % 64 == 0 && c->Le >= 1 && c->Ld >= 1 && c->V >= 16, WL_ERR_ARG, "wl_mt_init: bad shape");
    WL_CHECK(cfg->max_positions >= 1 && cfg->max_positions - 2 <= MT_MAX_SRC && cfg->pad_id >= 0 && cfg->pad_id < cfg->max_positions + 2,
             WL_ERR_ARG, "wl_mt_init: max_positions %d unsupported (sources up to %d tokens)", cfg->max_positions, MT_MAX_SRC);
    WL_CHECK(max_beam >= 1 && max_beam <= MT_MAX_BEAM, WL_ERR_ARG, "wl_mt_init: max_beam %d must be in [1, %d]", max_beam, MT_MAX_BEAM);
    WL_CHECK(capacity_segments >= 1 && cfg->max_src_tokens >= 1, WL_ERR_ARG, "wl_mt_init: bad capacity");
    c->Bc = capacity_segments; c->Km = max_beam; c->Ns = cfg->max_src_tokens; c->Rm = c->Bc * c->Km;
    c->Vld = (c->V + 7) / 8 * 8;
    WL_CUDA(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    c->mem.st = c->st;
    gemm_prime();
    mt_table(c);
    const long d = c->d, Ns = c->Ns, Rm = c->Rm;
    c->ex = c->mem.alloc<float>(Ns * d);
    c->eh = c->mem.alloc<__half>(Ns * d);
    c->eqkv = c->mem.alloc<__half>(Ns * 3 * d);
    c->eattn = c->mem.alloc<__half>(Ns * d);
    c->eff = c->mem.alloc<__half>(Ns * c->ff);
    c->xkv = c->mem.alloc<__half>(Ns * 2 * d * c->Ld);
    c->etok = c->mem.alloc<int>(Ns);
    c->etpos = c->mem.alloc<int>(Ns);
    c->eoff = c->mem.alloc<int>(c->Bc + 1);
    c->etiles = c->mem.alloc<int2>(Ns / 64 + c->Bc);
    c->dx = c->mem.alloc<float>(Rm * d);
    c->dqkv = c->mem.alloc<float>(Rm * 3 * d);
    c->dq = c->mem.alloc<float>(Rm * d);
    c->logits = c->mem.alloc<float>(Rm * c->Vld);
    c->dh = c->mem.alloc<__half>(Rm * d);
    c->dattn = c->mem.alloc<__half>(Rm * d);
    c->dff = c->mem.alloc<__half>(Rm * c->ff);
    c->kc = c->mem.alloc<__half>((long)c->Ld * Rm * d * T_MAX);
    c->vc = c->mem.alloc<__half>((long)c->Ld * Rm * d * T_MAX);
    MtState& s = c->s;
    s.tok_in = c->mem.alloc<int>(Rm);
    s.pos = c->mem.alloc<int>(Rm);
    s.active = c->mem.alloc<int>(Rm);
    s.src = c->mem.alloc<short>(Rm * T_MAX);
    s.hist = c->mem.alloc<int>(Rm * T_MAX);
    s.run_score = c->mem.alloc<float>(Rm);
    s.run_next = c->mem.alloc<float>(Rm);
    s.cand_val = c->mem.alloc<float>(Rm * MT_MAX_CAND);
    s.cand_tok = c->mem.alloc<int>(Rm * MT_MAX_CAND);
    s.fin_score = c->mem.alloc<float>(Rm);
    s.fin_flag = c->mem.alloc<int>(Rm);
    s.fin_len = c->mem.alloc<int>(Rm);
    s.fin_tok = c->mem.alloc<int>((long)c->Bc * MT_MAX_BEAM * T_MAX);
    s.done = c->mem.alloc<int>(c->Bc);
    s.unsat = c->mem.alloc<int>(c->Bc);
    s.steps = c->mem.alloc<int>(c->Bc);
    s.n_done = c->mem.alloc<int>(1);
    s.steps_left = c->mem.alloc<int>(1);
    s.forced_bos = s.forced_eos = -1;
    WL_CUDA(cudaStreamSynchronize(c->st));
  } catch (const wl::Error& e) {
    g_mt_init_error = e.msg;
    mt_free(c);
    delete c;
    return e.code;
  }
  *out = c;
  return WL_OK;
}

extern "C" void wl_mt_destroy(wl_mt_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->mem.device);
  if (c->st) cudaStreamSynchronize(c->st);
  mt_free(c);
  delete c;
}

extern "C" const char* wl_mt_last_error(wl_mt_ctx* c) { return c ? c->err.c_str() : g_mt_init_error.c_str(); }

extern "C" int wl_mt_device_bytes(wl_mt_ctx* c, int64_t* out) {
  API_BEGIN(c)
  WL_CHECK(out, WL_ERR_ARG, "wl_mt_device_bytes: null output");
  *out = c->mem.bytes;
  API_END(c)
}

extern "C" int wl_mt_load_tensor(wl_mt_ctx* c, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  API_BEGIN(c)
  WL_CHECK(name && data && shape && ndim >= 1, WL_ERR_ARG, "wl_mt_load_tensor: bad arguments");
  auto it = c->w.find(name);
  WL_CHECK(it != c->w.end(), WL_ERR_ARG, "wl_mt_load_tensor: unknown tensor '%s'", name);
  MtTensor& t = it->second;
  WL_CHECK(std::vector<int64_t>(shape, shape + ndim) == t.shape, WL_ERR_ARG, "wl_mt_load_tensor: '%s' has the wrong shape", name);
  long n = 1;
  for (int64_t s : t.shape) n *= s;
  if (!t.p) t.p = t.f16 ? (void*)c->mem.alloc<__half>(n) : (void*)c->mem.alloc<float>(n);
  Scratch sc(c->st);
  const float* tmp = sc.upload(data, n);
  if (t.f16) cast_weight_f16(c->st, tmp, (__half*)t.p, n, 1, 1);
  else WL_CUDA(cudaMemcpyAsync(t.p, tmp, n * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
  WL_CUDA(cudaStreamSynchronize(c->st));
  API_END(c)
}

extern "C" int wl_mt_finalize(wl_mt_ctx* c) {
  API_BEGIN(c)
  for (auto& kv : c->w) WL_CHECK(kv.second.p, WL_ERR_STATE, "wl_mt_finalize: missing tensor '%s'", kv.first.c_str());
  c->finalized = true;
  API_END(c)
}

// ---------------------------------------------------------------------------------------------- building blocks
static GemmOperand op(const __half* p, long rows, long k) {
  GemmOperand o;
  o.ptr = p; o.rows = rows; o.k = k; o.ld = k;
  return o;
}

// out = act(X W^T + b) (+ resid); X fp16 [M][K], W fp16 [N][K]
static void linear(wl_mt_ctx* c, const __half* X, long M, const std::string& name, int N, int K, void* out, bool f32,
                   const float* resid = nullptr, bool relu = false, bool bias = true) {
  GemmEpilogue e;
  e.out = out; e.out_f32 = f32 ? 1 : 0; e.ldm = N; e.ldn = 1;
  e.bias = bias ? W<float>(c, name + ".b") : nullptr;
  e.relu = relu ? 1 : 0;
  if (resid) { e.resid = resid; e.rldm = N; e.rldn = 1; }
  gemm_tn(c->st, op(X, M, K), op(W<__half>(c, name + ".w"), N, K), (int)M, N, K, e);
}

static void ln(wl_mt_ctx* c, const float* x, const std::string& name, __half* y, long rows) {
  layernorm_rows(c->st, x, W<float>(c, name + ".w"), W<float>(c, name + ".b"), y, nullptr, rows, c->d);
}

// host tables of a packed source: the sinusoidal row of every token and the 64-query tiles of every segment
static int enc_tables(const int32_t* ids, const int32_t* off, int B, int pad, std::vector<int>& tpos, std::vector<int2>& tiles) {
  const int n = off[B];
  tpos.resize(n);
  tiles.clear();
  for (int b = 0; b < B; ++b) {
    // Hugging Face's create_position_ids_from_input_ids: pad + the running count of non-pad tokens; pad tokens get pad
    int seen = 0;
    for (int i = off[b]; i < off[b + 1]; ++i) {
      const bool is_pad = ids && ids[i] == pad;
      seen += is_pad ? 0 : 1;
      tpos[i] = is_pad ? pad : pad + seen;
    }
    for (int q = 0; q < off[b + 1] - off[b]; q += 64) tiles.push_back(make_int2(b, q));
  }
  return (int)tiles.size();
}

static void check_off(const int32_t* off, int B, int max_len, long max_total, const char* who) {
  WL_CHECK(off && off[0] == 0, WL_ERR_ARG, "%s: offsets must start at 0", who);
  for (int b = 0; b < B; ++b) {
    const int n = off[b + 1] - off[b];
    WL_CHECK(n >= 1 && n <= max_len, WL_ERR_ARG, "%s: segment %d has %d tokens (1 .. %d)", who, b, n, max_len);
  }
  WL_CHECK(off[B] <= max_total, WL_ERR_ARG, "%s: %d tokens in all, the limit is %ld", who, off[B], max_total);
}

static void encode(wl_mt_ctx* c, long n, int n_tiles) {
  const int d = c->d;
  mt_enc_embed(c->st, c->etok, c->etpos, W<__half>(c, "shared"), W<float>(c, "positions"), c->cfg.embed_scale, c->ex, n, d);
  for (int l = 0; l < c->Le; ++l) {
    const std::string p = "enc." + std::to_string(l);
    ln(c, c->ex, p + ".ln1", c->eh, n);
    linear(c, c->eh, n, p + ".qkv", 3 * d, d, c->eqkv, false);
    mt_enc_attn(c->st, c->eqkv, c->eoff, c->etiles, n_tiles, c->eattn, c->H, d);
    linear(c, c->eattn, n, p + ".out", d, d, c->ex, true, c->ex);
    ln(c, c->ex, p + ".ln2", c->eh, n);
    linear(c, c->eh, n, p + ".fc1", c->ff, d, c->eff, false, nullptr, true);
    linear(c, c->eff, n, p + ".fc2", d, c->ff, c->ex, true, c->ex);
  }
  ln(c, c->ex, "enc.ln", c->eh, n);
  linear(c, c->eh, n, "dec.xkv", 2 * d * c->Ld, d, c->xkv, false);
}

// the decoder over R = B * K rows (row r of segment r / K) for the tokens in tok_in at positions pos -> logits
static void dec_forward(wl_mt_ctx* c, int B, int K) {
  const int d = c->d, R = B * K;
  const long row_stride = (long)d * T_MAX;   // one cache row: H heads x T_MAX positions x 64
  mt_dec_embed(c->st, c->s, W<__half>(c, "shared"), W<float>(c, "positions"), c->cfg.embed_scale, c->cfg.pad_id, c->dx, R, d);
  const DecodeState ds = mt_decode_state(c->s);
  for (int l = 0; l < c->Ld; ++l) {
    const std::string p = "dec." + std::to_string(l);
    ln(c, c->dx, p + ".ln1", c->dh, R);
    linear(c, c->dh, R, p + ".qkv", 3 * d, d, c->dqkv, true);
    PartialSrc qkv;
    qkv.ptr = c->dqkv; qkv.nsplit = 1;
    const long layer = (long)l * c->Rm * row_stride;
    decoder_self_attn(c->st, ds, qkv, c->kc + layer, c->vc + layer, row_stride, c->dattn, R, c->H, d);
    linear(c, c->dattn, R, p + ".out", d, d, c->dx, true, c->dx);
    ln(c, c->dx, p + ".ln2", c->dh, R);
    linear(c, c->dh, R, p + ".xq", d, d, c->dq, true);
    mt_cross_attn(c->st, c->s, c->dq, c->xkv, 2L * d * c->Ld, 2 * d * l, 2 * d * l + d, c->eoff, K, c->dattn, R, c->H, d);
    linear(c, c->dattn, R, p + ".xout", d, d, c->dx, true, c->dx);
    ln(c, c->dx, p + ".ln3", c->dh, R);
    linear(c, c->dh, R, p + ".fc1", c->ff, d, c->dff, false, nullptr, true);
    linear(c, c->dff, R, p + ".fc2", d, c->ff, c->dx, true, c->dx);
  }
  ln(c, c->dx, "dec.ln", c->dh, R);
  GemmEpilogue e;
  e.out = c->logits; e.out_f32 = 1; e.ldm = c->Vld; e.ldn = 1;
  gemm_tn(c->st, op(c->dh, R, d), op(W<__half>(c, "shared"), c->V, d), R, c->V, d, e);
}

// one token step: decoder, LM head, beam-search step
static void dec_step(wl_mt_ctx* c, int B, const MtSearch& so) {
  dec_forward(c, B, so.beam);
  mt_search_step(c->st, c->s, so, c->logits, c->Vld, c->V, B);
}

static MtSearch search_opts(wl_mt_ctx* c, const wl_mt_opts* o, int B, const char* who) {
  WL_CHECK(o, WL_ERR_ARG, "%s: null options", who);
  WL_CHECK(o->num_beams >= 1 && o->num_beams <= c->Km, WL_ERR_ARG, "%s: num_beams %d out of range (max_beam %d)", who, o->num_beams, c->Km);
  WL_CHECK(B >= 1 && B <= c->Bc, WL_ERR_ARG, "%s: %d segments, capacity %d", who, B, c->Bc);
  WL_CHECK(o->max_length >= 2 && o->max_length <= T_MAX, WL_ERR_ARG, "%s: max_length %d must be in [2, %d]", who, o->max_length, T_MAX);
  WL_CHECK(o->max_length <= c->cfg.max_positions + 1, WL_ERR_ARG, "%s: max_length %d exceeds the position table (max_positions %d + 1)",
           who, o->max_length, c->cfg.max_positions);
  WL_CHECK(o->early_stopping >= 0 && o->early_stopping <= 2, WL_ERR_ARG, "%s: bad early_stopping", who);
  WL_CHECK(o->eos >= 0 && o->eos < c->V && o->decoder_start >= 0 && o->decoder_start < c->V, WL_ERR_ARG, "%s: bad token ids", who);
  WL_CHECK(o->forced_bos < c->V && o->forced_eos < c->V, WL_ERR_ARG, "%s: bad forced token", who);
  MtSearch so;
  so.beam = o->num_beams; so.max_length = o->max_length; so.length_penalty = o->length_penalty;
  so.early_stopping = o->early_stopping; so.eos = o->eos;
  c->s.forced_bos = o->forced_bos < 0 ? -1 : o->forced_bos;
  c->s.forced_eos = o->forced_eos < 0 ? -1 : o->forced_eos;
  return so;
}

static void collect(wl_mt_ctx* c, int B, const MtSearch& so, int32_t* out_ids, int32_t* out_len, float* out_score, int32_t* out_steps) {
  const int K = so.beam;
  std::vector<int> tok((size_t)B * MT_MAX_BEAM * T_MAX), len((size_t)B * K), steps(B);
  std::vector<float> score((size_t)B * K);
  WL_CUDA(cudaMemcpyAsync(tok.data(), c->s.fin_tok, tok.size() * sizeof(int), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaMemcpyAsync(len.data(), c->s.fin_len, len.size() * sizeof(int), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaMemcpyAsync(score.data(), c->s.fin_score, score.size() * sizeof(float), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaMemcpyAsync(steps.data(), c->s.steps, steps.size() * sizeof(int), cudaMemcpyDeviceToHost, c->st));
  WL_CUDA(cudaStreamSynchronize(c->st));
  for (int b = 0; b < B; ++b) {
    const int n = std::max(0, len[(size_t)b * K] - 1);   // best slot, without the decoder start token
    for (int i = 0; i < so.max_length; ++i) out_ids[(long)b * so.max_length + i] = i < n ? tok[((size_t)b * MT_MAX_BEAM) * T_MAX + 1 + i] : -1;
    out_len[b] = n;
    out_score[b] = score[(size_t)b * K];
    if (out_steps) out_steps[b] = steps[b];
  }
}

static void upload_and_encode(wl_mt_ctx* c, const int32_t* src_ids, const int32_t* src_off, int B, const char* who) {
  check_off(src_off, B, c->cfg.max_positions - 2, c->Ns, who);
  const int n = src_off[B];
  for (int i = 0; i < n; ++i) WL_CHECK(src_ids[i] >= 0 && src_ids[i] < c->V, WL_ERR_ARG, "%s: token id %d out of range", who, src_ids[i]);
  std::vector<int> tpos;
  std::vector<int2> tiles;
  const int n_tiles = enc_tables(src_ids, src_off, B, c->cfg.pad_id, tpos, tiles);
  WL_CUDA(cudaMemcpyAsync(c->etok, src_ids, n * sizeof(int), cudaMemcpyHostToDevice, c->st));
  WL_CUDA(cudaMemcpyAsync(c->etpos, tpos.data(), n * sizeof(int), cudaMemcpyHostToDevice, c->st));
  WL_CUDA(cudaMemcpyAsync(c->eoff, src_off, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, c->st));
  WL_CUDA(cudaMemcpyAsync(c->etiles, tiles.data(), n_tiles * sizeof(int2), cudaMemcpyHostToDevice, c->st));
  encode(c, n, n_tiles);
}

extern "C" int wl_mt_translate(wl_mt_ctx* c, const int32_t* src_ids, const int32_t* src_off, int32_t B, const wl_mt_opts* o,
                               int32_t* out_ids, int32_t* out_len, float* out_score) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "wl_mt_translate: weights not finalized");
  WL_CHECK(src_ids && out_ids && out_len && out_score, WL_ERR_ARG, "wl_mt_translate: bad arguments");
  const MtSearch so = search_opts(c, o, B, "wl_mt_translate");
  upload_and_encode(c, src_ids, src_off, B, "wl_mt_translate");
  const int steps = so.max_length - 1;
  mt_search_init(c->st, c->s, B, so.beam, o->decoder_start, steps);
  if (o->use_cuda_graph) {
    char key[128];
    snprintf(key, sizeof(key), "%d/%d/%d/%g/%d/%d/%d/%d", B, so.beam, so.max_length, so.length_penalty, so.early_stopping, so.eos,
             c->s.forced_bos, c->s.forced_eos);
    cudaGraphExec_t& ex = c->graphs[key];
    if (!ex) {
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
      WL_CUDA(cudaStreamBeginCaptureToGraph(c->st, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
      try {
        dec_step(c, B, so);
        mt_loop_condition(c->st, c->s, h, B);
      } catch (...) {
        cudaStreamEndCapture(c->st, &cap);
        cudaGraphDestroy(g);
        c->graphs.erase(key);
        throw;
      }
      WL_CUDA(cudaStreamEndCapture(c->st, &cap));
      const cudaError_t ie = cudaGraphInstantiate(&ex, g, 0);
      cudaGraphDestroy(g);
      if (ie != cudaSuccess) {
        c->graphs.erase(key);
        WL_CUDA(ie);
      }
    }
    WL_CUDA(cudaGraphLaunch(ex, c->st));
  } else {
    for (int t = 0; t < steps; ++t) {
      dec_step(c, B, so);
      int nd = 0;
      WL_CUDA(cudaMemcpyAsync(&nd, c->s.n_done, sizeof(int), cudaMemcpyDeviceToHost, c->st));
      WL_CUDA(cudaStreamSynchronize(c->st));
      if (nd >= B) break;
    }
  }
  collect(c, B, so, out_ids, out_len, out_score, nullptr);
  API_END(c)
}

// ---------------------------------------------------------------------------------------------- test hooks
extern "C" int wl_test_mt_attn(wl_mt_ctx* c, const uint16_t* qkv_f16, const int32_t* off, int32_t B, int32_t H, uint16_t* out_f16) {
  API_BEGIN(c)
  WL_CHECK(qkv_f16 && out_f16 && B >= 1 && H >= 1 && H <= 20, WL_ERR_ARG, "wl_test_mt_attn: bad arguments");
  check_off(off, B, MT_MAX_SRC, 1L << 30, "wl_test_mt_attn");
  const int d = 64 * H, n = off[B];
  std::vector<int> tpos;
  std::vector<int2> tiles;
  const int n_tiles = enc_tables(nullptr, off, B, 0, tpos, tiles);
  Scratch sc(c->st);
  const __half* qkv = sc.upload(reinterpret_cast<const __half*>(qkv_f16), (size_t)n * 3 * d);
  __half* out = sc.upload(reinterpret_cast<const __half*>(out_f16), (size_t)n * d);
  const int* doff = sc.upload(off, B + 1);
  const int2* dtiles = sc.upload(tiles.data(), n_tiles);
  mt_enc_attn(c->st, qkv, doff, dtiles, n_tiles, out, H, d);
  sc.download(reinterpret_cast<__half*>(out_f16), out, (size_t)n * d);
  API_END(c)
}

extern "C" int wl_test_mt_cross_attn(wl_mt_ctx* c, const float* q, const uint16_t* kv_f16, int32_t ldkv, int32_t koff, int32_t voff,
                                     const int32_t* off, int32_t B, int32_t rows_per_seg, int32_t H, uint16_t* out_f16) {
  API_BEGIN(c)
  WL_CHECK(q && kv_f16 && out_f16 && B >= 1 && rows_per_seg >= 1 && H >= 1 && H <= 20, WL_ERR_ARG, "wl_test_mt_cross_attn: bad arguments");
  const int d = 64 * H, R = B * rows_per_seg;
  WL_CHECK(ldkv % 8 == 0 && koff % 8 == 0 && voff % 8 == 0 && koff + d <= ldkv && voff + d <= ldkv, WL_ERR_ARG,
           "wl_test_mt_cross_attn: bad K/V layout");
  check_off(off, B, MT_MAX_SRC, 1L << 30, "wl_test_mt_cross_attn");
  const int n = off[B];
  Scratch sc(c->st);
  const float* dq = sc.upload(q, (size_t)R * d);
  const __half* kv = sc.upload(reinterpret_cast<const __half*>(kv_f16), (size_t)n * ldkv);
  __half* out = sc.upload(reinterpret_cast<const __half*>(out_f16), (size_t)R * d);
  const int* doff = sc.upload(off, B + 1);
  MtState s;
  memset(&s, 0, sizeof(s));   // no active table: every row
  mt_cross_attn(c->st, s, dq, kv, ldkv, koff, voff, doff, rows_per_seg, out, R, H, d);
  sc.download(reinterpret_cast<__half*>(out_f16), out, (size_t)R * d);
  API_END(c)
}

extern "C" int wl_test_mt_search(wl_mt_ctx* c, const float* logits, int32_t V, int32_t B, const wl_mt_opts* o, int32_t* out_ids,
                                 int32_t* out_len, float* out_score, int32_t* out_steps) {
  API_BEGIN(c)
  WL_CHECK(logits && out_ids && out_len && out_score && out_steps && V >= 16, WL_ERR_ARG, "wl_test_mt_search: bad arguments");
  const MtSearch so = search_opts(c, o, B, "wl_test_mt_search");
  const int R = B * so.beam, steps = so.max_length - 1;
  Scratch sc(c->st);
  const float* dl = sc.upload(logits, (size_t)steps * R * V);
  mt_search_init(c->st, c->s, B, so.beam, o->decoder_start, steps);
  for (int t = 0; t < steps; ++t) mt_search_step(c->st, c->s, so, dl + (size_t)t * R * V, V, V, B);
  collect(c, B, so, out_ids, out_len, out_score, out_steps);
  API_END(c)
}

extern "C" int wl_test_mt_logits(wl_mt_ctx* c, const int32_t* src_ids, const int32_t* src_off, int32_t B, const int32_t* prefix,
                                 int32_t P, float* out_logits) {
  API_BEGIN(c)
  WL_CHECK(c->finalized, WL_ERR_STATE, "wl_test_mt_logits: weights not finalized");
  WL_CHECK(src_ids && prefix && out_logits && B >= 1 && B <= c->Bc && P >= 1 && P <= T_MAX && P <= c->cfg.max_positions,
           WL_ERR_ARG, "wl_test_mt_logits: bad arguments");
  for (long i = 0; i < (long)B * P; ++i)
    WL_CHECK(prefix[i] >= 0 && prefix[i] < c->V, WL_ERR_ARG, "wl_test_mt_logits: token id %d out of range", prefix[i]);
  upload_and_encode(c, src_ids, src_off, B, "wl_test_mt_logits");
  std::vector<int> tok(B), pos(B), on(B, 1);
  std::vector<float> lg((size_t)B * c->Vld);
  WL_CUDA(cudaMemcpyAsync(c->s.active, on.data(), B * sizeof(int), cudaMemcpyHostToDevice, c->st));
  for (int t = 0; t < P; ++t) {
    for (int b = 0; b < B; ++b) { tok[b] = prefix[(long)b * P + t]; pos[b] = t; }
    WL_CUDA(cudaMemcpyAsync(c->s.tok_in, tok.data(), B * sizeof(int), cudaMemcpyHostToDevice, c->st));
    WL_CUDA(cudaMemcpyAsync(c->s.pos, pos.data(), B * sizeof(int), cudaMemcpyHostToDevice, c->st));
    dec_forward(c, B, 1);
    WL_CUDA(cudaMemcpyAsync(lg.data(), c->logits, lg.size() * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    WL_CUDA(cudaStreamSynchronize(c->st));
    for (int b = 0; b < B; ++b)
      memcpy(out_logits + ((long)b * P + t) * c->V, lg.data() + (size_t)b * c->Vld, c->V * sizeof(float));
  }
  API_END(c)
}
