// Silero VAD on the device (C ABI wl_vad_*): its own weights, independent of the Whisper weights and of finalize, and
// the speech probability of every 512-sample frame of every stream of a call.
#include <cstring>

#include "ctx.cuh"

struct VadTensor {
  const char* name;
  int ndim;
  int64_t shape[3];
  int layout;   // 0 as given, 1 [rows][k] -> [k][rows] (rows = shape[0], k = the rest), 2 conv [co][ci][3] -> [ci][3][co]
};
static const VadTensor VAD_TENSORS[15] = {
    {"vad.stft.basis", 3, {258, 1, 256}, 1},   {"vad.conv0.weight", 3, {128, 129, 3}, 2}, {"vad.conv0.bias", 1, {128}, 0},
    {"vad.conv1.weight", 3, {64, 128, 3}, 2},  {"vad.conv1.bias", 1, {64}, 0},        {"vad.conv2.weight", 3, {64, 64, 3}, 2},
    {"vad.conv2.bias", 1, {64}, 0},            {"vad.conv3.weight", 3, {128, 64, 3}, 2}, {"vad.conv3.bias", 1, {128}, 0},
    {"vad.lstm.weight_ih", 2, {512, 128}, 1},  {"vad.lstm.weight_hh", 2, {512, 128}, 0}, {"vad.lstm.bias_ih", 1, {512}, 0},
    {"vad.lstm.bias_hh", 1, {512}, 0},         {"vad.out.weight", 3, {1, 128, 1}, 0},  {"vad.out.bias", 1, {1}, 0},
};
constexpr long VAD_CHUNK_SAMPLES = 30 * 16000;   // the workspace's first size: max_streams chunks of 30 s

extern "C" int wl_vad_load_tensor(wl_ctx* c, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  API_BEGIN(c)
  WL_CHECK(name && data && shape && ndim >= 1, WL_ERR_ARG, "wl_vad_load_tensor: bad arguments");
  int i = 0;
  while (i < 15 && strcmp(VAD_TENSORS[i].name, name) != 0) ++i;
  WL_CHECK(i < 15, WL_ERR_ARG, "wl_vad_load_tensor: unknown VAD tensor '%s'", name);
  const VadTensor& T = VAD_TENSORS[i];
  bool ok = ndim == T.ndim;
  for (int k = 0; ok && k < ndim; ++k) ok = shape[k] == T.shape[k];
  WL_CHECK(ok, WL_ERR_ARG, "wl_vad_load_tensor: '%s' must have shape [%lld%s%lld%s%lld]", name, (long long)T.shape[0],
           T.ndim > 1 ? ", " : "", (long long)(T.ndim > 1 ? T.shape[1] : 0), T.ndim > 2 ? ", " : "",
           (long long)(T.ndim > 2 ? T.shape[2] : 0));
  size_t n = 1;
  for (int k = 0; k < ndim; ++k) n *= (size_t)shape[k];
  std::vector<float> h(n);
  if (T.layout == 1) {
    const size_t rows = (size_t)shape[0], kk = n / rows;
    for (size_t r = 0; r < rows; ++r)
      for (size_t k = 0; k < kk; ++k) h[k * rows + r] = data[r * kk + k];
  } else if (T.layout == 2) {
    const size_t co_n = (size_t)shape[0], ci_n = (size_t)shape[1];
    for (size_t co = 0; co < co_n; ++co)
      for (size_t ci = 0; ci < ci_n; ++ci)
        for (size_t k = 0; k < 3; ++k) h[(ci * 3 + k) * co_n + co] = data[(co * ci_n + ci) * 3 + k];
  } else {
    std::copy(data, data + n, h.begin());
  }
  if (!c->vad.t[i]) c->vad.t[i] = c->mem.alloc<float>(n, false);
  WL_CUDA(cudaMemcpy(c->vad.t[i], h.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  API_END(c)
}

extern "C" int wl_vad(wl_ctx* c, const float* pcm, const int64_t* offsets, int32_t B, float* probs_out, const int64_t* prob_off) {
  API_BEGIN(c)
  WL_CHECK(pcm && offsets && probs_out && prob_off && B >= 1, WL_ERR_ARG, "wl_vad: bad arguments (B=%d)", B);
  for (int i = 0; i < 15; ++i)
    WL_CHECK(c->vad.t[i], WL_ERR_STATE, "wl_vad: VAD weights not loaded: '%s' is missing (wl_vad_load_tensor)", VAD_TENSORS[i].name);
  std::vector<long> off(2 * (B + 1));
  long* poff = off.data();
  long* foff = off.data() + B + 1;
  for (int b = 0; b <= B; ++b) poff[b] = offsets[b] - offsets[0];
  foff[0] = 0;
  for (int b = 0; b < B; ++b) {
    const long n = poff[b + 1] - poff[b];
    WL_CHECK(n >= 0, WL_ERR_ARG, "wl_vad: offsets decrease at stream %d", b);
    const long frames = n > 0 ? n / 512 + 1 : 0;
    WL_CHECK(prob_off[b + 1] - prob_off[b] == frames, WL_ERR_ARG,
             "wl_vad: prob_off gives stream %d %lld frames; its %ld samples have %ld", b,
             (long long)(prob_off[b + 1] - prob_off[b]), n, frames);
    foff[b + 1] = foff[b] + frames;
  }
  const long total = poff[B], frames = foff[B];
  auto& v = c->vad;
  const long first_frames = (long)c->Bm * (VAD_CHUNK_SAMPLES / 512 + 1);
  c->mem.grow(v.pcm, v.pcm_cap, total, (long)c->Bm * VAD_CHUNK_SAMPLES);
  c->mem.grow(v.gx, v.gx_cap, frames * 512, first_frames * 512);
  c->mem.grow(v.probs, v.frame_cap, frames, first_frames);
  c->mem.grow(v.off, v.off_cap, 2L * (B + 1), 2L * (c->Bm + 1));
  if (!v.ev[0])
    for (auto& e : v.ev) WL_CUDA(cudaEventCreate(&e));
  cudaStream_t st = c->st;
  const VadWeights w{v.t[0], v.t[1], v.t[2], v.t[3], v.t[4], v.t[5], v.t[6], v.t[7], v.t[8], v.t[9], v.t[10], v.t[11],
                     v.t[12], v.t[13], v.t[14]};
  if (total > 0) WL_CUDA(cudaMemcpyAsync(v.pcm, pcm + offsets[0], total * sizeof(float), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaMemcpyAsync(v.off, off.data(), off.size() * sizeof(long), cudaMemcpyHostToDevice, st));
  WL_CUDA(cudaEventRecord(v.ev[0], st));
  vad_front(st, w, v.pcm, v.off, v.off + B + 1, B, frames, v.gx);
  WL_CUDA(cudaEventRecord(v.ev[1], st));
  if (frames > 0) vad_lstm(st, w, v.gx, v.off + B + 1, B, v.probs);
  WL_CUDA(cudaEventRecord(v.ev[2], st));
  if (frames > 0)
    WL_CUDA(cudaMemcpyAsync(probs_out + prob_off[0], v.probs, frames * sizeof(float), cudaMemcpyDeviceToHost, st));
  WL_CUDA(cudaStreamSynchronize(st));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[6], v.ev[0], v.ev[1]));
  WL_CUDA(cudaEventElapsedTime(&c->last_ms[7], v.ev[1], v.ev[2]));
  API_END(c)
}
