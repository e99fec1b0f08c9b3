// Speaker embeddings on the device (C ABI wl_spk_*): WeSpeaker ResNet34 weights of their own, the Kaldi fbank + CMN
// front end and the network for every segment of a call, and the test hooks of the fbank and of one convolution.
#include <cmath>

#include "ctx.cuh"

struct SpkTensor {
  std::string name;
  int co, ci, k;   // a conv weight [co][ci][k][k]; a bias has k = 0 (shape [co]); seg_1.weight has k = -1 ([co][ci])
};
constexpr int SPK_MEL_BINS = 80, SPK_EMB = 256, SPK_POOL = 2 * 256 * 10;
constexpr long SPK_CHUNK_SAMPLES = 30 * 16000;   // the workspace's first size: max_streams segments of 30 s
static const int SPK_STAGE_C[4] = {32, 64, 128, 256}, SPK_STAGE_N[4] = {3, 4, 6, 3};

static const std::vector<SpkTensor>& spk_tensors() {
  static const std::vector<SpkTensor> t = [] {
    std::vector<SpkTensor> v;
    auto conv = [&](const std::string& n, int co, int ci, int k) {
      v.push_back({n + ".weight", co, ci, k});
      v.push_back({n + ".bias", co, 0, 0});
    };
    conv("spk.conv1", 32, 1, 3);
    int cin = 32;
    for (int L = 0; L < 4; ++L)
      for (int i = 0; i < SPK_STAGE_N[L]; ++i) {
        const std::string b = "spk.layer" + std::to_string(L + 1) + "." + std::to_string(i);
        const int c = SPK_STAGE_C[L];
        conv(b + ".conv1", c, cin, 3);
        conv(b + ".conv2", c, c, 3);
        if (i == 0 && L > 0) conv(b + ".shortcut", c, cin, 1);
        cin = c;
      }
    v.push_back({"spk.seg_1.weight", SPK_EMB, SPK_POOL, -1});
    v.push_back({"spk.seg_1.bias", SPK_EMB, 0, 0});
    return v;
  }();
  return t;
}

static int spk_index(const std::string& name) {
  const auto& T = spk_tensors();
  for (size_t i = 0; i < T.size(); ++i)
    if (T[i].name == name) return (int)i;
  return -1;
}

extern "C" int wl_spk_load_tensor(wl_ctx* c, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  API_BEGIN(c)
  WL_CHECK(name && data && shape && ndim >= 1, WL_ERR_ARG, "wl_spk_load_tensor: bad arguments");
  const int i = spk_index(name);
  WL_CHECK(i >= 0, WL_ERR_ARG, "wl_spk_load_tensor: unknown speaker-embedding tensor '%s'", name);
  const SpkTensor& T = spk_tensors()[i];
  std::vector<int64_t> want;
  if (T.k > 0) want = {T.co, T.ci, T.k, T.k};
  else if (T.k == 0) want = {T.co};
  else want = {T.co, T.ci};
  bool ok = ndim == (int)want.size();
  for (int k = 0; ok && k < ndim; ++k) ok = shape[k] == want[k];
  std::string ws;
  for (size_t k = 0; k < want.size(); ++k) ws += (k ? ", " : "") + std::to_string(want[k]);
  WL_CHECK(ok, WL_ERR_ARG, "wl_spk_load_tensor: '%s' must have shape [%s]", name, ws.c_str());
  auto& s = c->spk;
  if (s.t.empty()) s.t.assign(spk_tensors().size(), nullptr);
  if (T.k > 0 && T.ci > 1) {   // tensor-core conv: fp16 [co][kh * k + kw][ci]
    const int taps = T.k * T.k;
    std::vector<__half> h((size_t)T.co * taps * T.ci);
    for (int co = 0; co < T.co; ++co)
      for (int ci = 0; ci < T.ci; ++ci)
        for (int tap = 0; tap < taps; ++tap)
          h[((size_t)co * taps + tap) * T.ci + ci] = __float2half_rn(data[((size_t)co * T.ci + ci) * taps + tap]);
    if (!s.t[i]) s.t[i] = c->mem.alloc<__half>(h.size(), false);
    WL_CUDA(cudaMemcpyAsync(s.t[i], h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice, c->st));
  } else {
    size_t n = 1;
    for (int k = 0; k < ndim; ++k) n *= (size_t)shape[k];
    std::vector<float> h(data, data + n);
    if (T.k < 0)   // seg_1: [256][5120] -> [5120][256]
      for (int r = 0; r < T.co; ++r)
        for (int k = 0; k < T.ci; ++k) h[(size_t)k * T.co + r] = data[(size_t)r * T.ci + k];
    if (!s.t[i]) s.t[i] = c->mem.alloc<float>(n, false);
    WL_CUDA(cudaMemcpyAsync(s.t[i], h.data(), n * sizeof(float), cudaMemcpyHostToDevice, c->st));
  }
  API_END(c)
}

// Kaldi mel banks [80][257] (20 Hz .. Nyquist, mel = 1127 ln(1 + f / 700)) and each bin's non-zero FFT-bin range
static void spk_mel_tables(std::vector<float>& w, std::vector<int>& range) {
  const int nb = SPK_MEL_BINS, half = 256;
  auto mel = [](double f) { return 1127.0 * std::log(1.0 + f / 700.0); };
  const double lo = mel(20.0), hi = mel(8000.0), delta = (hi - lo) / (nb + 1), width = 16000.0 / 512;
  w.assign((size_t)nb * (half + 1), 0.f);
  range.assign(2 * nb, 0);
  for (int b = 0; b < nb; ++b) {
    const double l = lo + b * delta, ce = lo + (b + 1) * delta, r = lo + (b + 2) * delta;
    int k0 = half, k1 = 0;
    for (int k = 0; k < half; ++k) {
      const double m = mel(width * k);
      const double v = std::max(0.0, std::min((m - l) / (ce - l), (r - m) / (r - ce)));
      w[(size_t)b * (half + 1) + k] = (float)v;
      if (v > 0) { k0 = std::min(k0, k); k1 = k + 1; }
    }
    range[2 * b] = k0 < k1 ? k0 : 0;
    range[2 * b + 1] = k1;
  }
}

// Position offsets of every stage, shared by wl_spk_embed and wl_test_spk_conv: a stream of T frames has H x T positions
// at the stem (H = 80) and ceil-halved H and T after each stride-2 stage.
static void spk_positions(const std::vector<long>& T, int H, std::vector<long>& off) {
  off.assign(T.size() + 1, 0);
  for (size_t b = 0; b < T.size(); ++b) off[b + 1] = off[b] + (long)H * T[b];
}
static std::vector<long> spk_halve(const std::vector<long>& T) {
  std::vector<long> o(T.size());
  for (size_t b = 0; b < T.size(); ++b) o[b] = (T[b] + 1) / 2;
  return o;
}

static SpkConvParams spk_conv_params(const __half* x, const __half* w, const float* bias, const __half* res, __half* out,
                                     const long* in_off, const long* out_off, long M, int B, int H_in, int C_in, int C_out,
                                     int k, int stride, int relu) {
  SpkConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.res = res; p.out = out; p.in_off = in_off; p.out_off = out_off; p.M = M; p.B = B;
  p.H_in = H_in; p.H_out = stride == 2 ? (H_in + 1) / 2 : H_in; p.C_in = C_in; p.C_out = C_out; p.taps = k * k;
  p.stride = stride; p.relu = relu;
  return p;
}

extern "C" int wl_spk_embed(wl_ctx* c, const float* pcm, const int64_t* offsets, int32_t B, float* emb_out) {
  API_BEGIN(c)
  WL_CHECK(pcm && offsets && emb_out && B >= 1, WL_ERR_ARG, "wl_spk_embed: bad arguments (B=%d)", B);
  auto& s = c->spk;
  const auto& TT = spk_tensors();
  for (size_t i = 0; i < TT.size(); ++i)
    WL_CHECK(!s.t.empty() && s.t[i], WL_ERR_STATE, "wl_spk_embed: speaker weights not loaded: '%s' is missing (wl_spk_load_tensor)",
             TT[i].name.c_str());
  std::vector<long> T(B), poff(B + 1);
  for (int b = 0; b <= B; ++b) poff[b] = offsets[b] - offsets[0];
  for (int b = 0; b < B; ++b) {
    const long n = poff[b + 1] - poff[b];
    WL_CHECK(n >= 400, WL_ERR_ARG, "wl_spk_embed: stream %d has %ld samples; the fbank needs at least 400 (one 25 ms frame)", b, n);
    T[b] = 1 + (n - 400) / 160;
  }
  // the tables: pcm offsets, frame offsets, the position offsets of the four stages
  std::vector<long> tab(6 * (size_t)(B + 1)), st_off;
  std::copy(poff.begin(), poff.end(), tab.begin());
  spk_positions(T, 1, st_off);
  std::copy(st_off.begin(), st_off.end(), tab.begin() + (B + 1));
  std::vector<long> Ts = T;
  long elems[4];
  for (int L = 0; L < 4; ++L) {
    if (L > 0) Ts = spk_halve(Ts);
    spk_positions(Ts, SPK_MEL_BINS >> L, st_off);
    std::copy(st_off.begin(), st_off.end(), tab.begin() + (2 + L) * (B + 1));
    elems[L] = st_off[B] * SPK_STAGE_C[L];
  }
  // first size: max_streams segments of 30 s
  long first[4], first_frames = (SPK_CHUNK_SAMPLES - 400) / 160 + 1;
  {
    long t = first_frames;
    for (int L = 0; L < 4; ++L) {
      if (L > 0) t = (t + 1) / 2;
      first[L] = (long)c->Bm * (SPK_MEL_BINS >> L) * t * SPK_STAGE_C[L];
    }
  }
  const long total = poff[B], frames = tab[(B + 1) + B];
  DeviceMem& m = c->mem;
  m.grow(s.pcm, s.pcm_cap, total, (long)c->Bm * SPK_CHUNK_SAMPLES);
  m.grow(s.feat, s.feat_cap, frames * SPK_MEL_BINS, (long)c->Bm * first_frames * SPK_MEL_BINS);
  if (B > s.stream_cap) {
    const long n = std::max(B, c->Bm);
    s.stream_cap = 0;   // until every buffer of the set has its new size
    m.replace(s.mean, (size_t)n * SPK_MEL_BINS);
    m.replace(s.pooled, (size_t)n * SPK_POOL);
    m.replace(s.emb, (size_t)n * SPK_EMB);
    m.replace(s.off, 6 * (size_t)(n + 1));
    s.stream_cap = n;
  }
  // act[0]: stage input / output of stages 1 and 3; act[1]: each block's first conv; act[2]: stages 2 and 4
  m.grow(s.act[0], s.act_cap[0], std::max(elems[0], elems[2]), std::max(first[0], first[2]));
  m.grow(s.act[1], s.act_cap[1], std::max(std::max(elems[0], elems[1]), std::max(elems[2], elems[3])),
         std::max(std::max(first[0], first[1]), std::max(first[2], first[3])));
  m.grow(s.act[2], s.act_cap[2], std::max(elems[1], elems[3]), std::max(first[1], first[3]));
  if (!s.melw) {
    std::vector<float> w;
    std::vector<int> r;
    spk_mel_tables(w, r);
    s.melw = c->mem.alloc<float>(w.size(), false);
    s.mel_range = c->mem.alloc<int>(r.size(), false);
    WL_CUDA(cudaMemcpyAsync(s.melw, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice, c->st));
    WL_CUDA(cudaMemcpyAsync(s.mel_range, r.data(), r.size() * sizeof(int), cudaMemcpyHostToDevice, c->st));
  }
  if (!s.ev[0])
    for (auto& e : s.ev) WL_CUDA(cudaEventCreate(&e));
  cudaStream_t st = c->st;
  const long* d_pcm_off = s.off;
  const long* d_frame_off = s.off + (B + 1);
  auto d_pos = [&](int L) { return s.off + (2 + L) * (B + 1); };
  WL_CUDA(cudaMemcpyAsync(s.pcm, pcm + offsets[0], total * sizeof(float), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(s.off, tab.data(), tab.size() * sizeof(long), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaEventRecord(s.ev[0], st));
  spk_fbank(st, s.pcm, d_pcm_off, d_frame_off, B, frames, s.melw, s.mel_range, s.feat, s.mean);
  WL_CUDA(cudaEventRecord(s.ev[1], st));
  size_t ti = 0;
  auto wgt = [&]() { return s.t[ti++]; };
  {
    const float* w = (const float*)wgt();
    const float* b = (const float*)wgt();
    spk_stem(st, s.feat, s.mean, d_frame_off, B, frames, w, b, s.act[0]);
  }
  __half* cur = s.act[0];
  int cin = 32;
  for (int L = 0; L < 4; ++L) {
    const int C = SPK_STAGE_C[L], H_in = L == 0 ? SPK_MEL_BINS : (SPK_MEL_BINS >> (L - 1)), H = SPK_MEL_BINS >> L;
    const long M = elems[L] / C;
    __half* y = s.act[1];
    for (int i = 0; i < SPK_STAGE_N[L]; ++i) {
      const bool down = i == 0 && L > 0;
      const long* in_off = down ? d_pos(L - 1) : d_pos(L);
      const int hin = down ? H_in : H, stride = down ? 2 : 1;
      const __half* w1 = (const __half*)wgt(); const float* b1 = (const float*)wgt();
      const __half* w2 = (const __half*)wgt(); const float* b2 = (const float*)wgt();
      __half* out = cur;
      if (down) {   // the shortcut goes to the buffer the block's output then replaces in place
        const __half* ws = (const __half*)wgt(); const float* bs = (const float*)wgt();
        out = cur == s.act[0] ? s.act[2] : s.act[0];
        spk_conv(st, spk_conv_params(cur, ws, bs, nullptr, out, in_off, d_pos(L), M, B, hin, cin, C, 1, 2, 0));
      }
      spk_conv(st, spk_conv_params(cur, w1, b1, nullptr, y, in_off, d_pos(L), M, B, hin, cin, C, 3, stride, 1));
      spk_conv(st, spk_conv_params(y, w2, b2, out, out, d_pos(L), d_pos(L), M, B, H, C, C, 3, 1, 1));
      cur = out;
      cin = C;
    }
  }
  {
    const float* w = (const float*)wgt();
    const float* b = (const float*)wgt();
    spk_pool_embed(st, cur, d_pos(3), B, SPK_MEL_BINS >> 3, w, b, s.pooled, s.emb);
  }
  WL_CUDA(cudaEventRecord(s.ev[2], st));
  WL_CUDA(cudaMemcpyAsync(emb_out, s.emb, (size_t)B * SPK_EMB * sizeof(float), cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[8], s.ev[0], s.ev[1]));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[9], s.ev[1], s.ev[2]));
  API_END(c)
}

extern "C" int wl_test_spk_fbank(wl_ctx* c, const float* pcm, const int64_t* offsets, int32_t B, float* feat_out) {
  API_BEGIN(c)
  WL_CHECK(pcm && offsets && feat_out && B >= 1, WL_ERR_ARG, "wl_test_spk_fbank: bad arguments");
  std::vector<long> tab(2 * (size_t)(B + 1), 0);
  for (int b = 0; b <= B; ++b) tab[b] = offsets[b] - offsets[0];
  for (int b = 0; b < B; ++b) {
    const long n = tab[b + 1] - tab[b];
    WL_CHECK(n >= 400, WL_ERR_ARG, "wl_test_spk_fbank: stream %d has %ld samples (< 400)", b, n);
    tab[B + 2 + b] = tab[B + 1 + b] + 1 + (n - 400) / 160;
  }
  const long total = tab[B], frames = tab[2 * B + 1];
  std::vector<float> w;
  std::vector<int> r;
  spk_mel_tables(w, r);
  Scratch sc(c->st);
  const float* dp = sc.upload(pcm + offsets[0], total);
  const float* dw = sc.upload(w.data(), w.size());
  const int* dr = sc.upload(r.data(), r.size());
  const long* doff = sc.upload(tab.data(), tab.size());
  float* df = sc.alloc<float>(frames * SPK_MEL_BINS);
  float* dm = sc.alloc<float>((size_t)B * SPK_MEL_BINS);
  spk_fbank(c->st, dp, doff, doff + B + 1, B, frames, dw, dr, df, dm);
  sc.download(feat_out, df, frames * SPK_MEL_BINS);
  API_END(c)
}

extern "C" int wl_test_spk_conv(wl_ctx* c, const uint16_t* x_f16, const int64_t* frames, int32_t B, int32_t H_in, int32_t C_in,
                                int32_t C_out, int32_t ksize, int32_t stride, const uint16_t* w_f16, const float* bias,
                                const uint16_t* res_f16, int32_t relu, uint16_t* out_f16) {
  API_BEGIN(c)
  WL_CHECK(x_f16 && frames && B >= 1 && w_f16 && bias && out_f16 && (ksize == 1 || ksize == 3), WL_ERR_ARG,
           "wl_test_spk_conv: bad arguments");
  WL_CHECK(spk_conv_supported(C_in, C_out, ksize * ksize, stride), WL_ERR_ARG, "wl_test_spk_conv: unsupported shape");
  std::vector<long> T(frames, frames + B), in_off, out_off;
  for (long t : T) WL_CHECK(t >= 1, WL_ERR_ARG, "wl_test_spk_conv: every stream needs a frame");
  spk_positions(T, H_in, in_off);
  const int H_out = stride == 2 ? (H_in + 1) / 2 : H_in;
  spk_positions(stride == 2 ? spk_halve(T) : T, H_out, out_off);
  const long Min = in_off[B], M = out_off[B];
  const size_t nw = (size_t)C_out * ksize * ksize * C_in;
  std::vector<long> tab(in_off);
  tab.insert(tab.end(), out_off.begin(), out_off.end());
  Scratch sc(c->st);
  const __half* dx = sc.upload(reinterpret_cast<const __half*>(x_f16), Min * C_in);
  const __half* dw = sc.upload(reinterpret_cast<const __half*>(w_f16), nw);
  const float* db = sc.upload(bias, C_out);
  __half* dout = sc.upload(reinterpret_cast<const __half*>(out_f16), M * C_out);
  const long* doff = sc.upload(tab.data(), tab.size());
  const __half* dr = res_f16 ? sc.upload(reinterpret_cast<const __half*>(res_f16), M * C_out) : nullptr;
  spk_conv(c->st, spk_conv_params(dx, dw, db, dr, dout, doff, doff + B + 1, M, B, H_in, C_in, C_out, ksize, stride, relu));
  sc.download(reinterpret_cast<__half*>(out_f16), dout, M * C_out);
  API_END(c)
}
