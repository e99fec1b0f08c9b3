// Host side of the C ABI, shared by the engine's translation units (engine.cu, vad_engine.cu, spk_engine.cu, hooks.cu,
// mt_engine.cu): the owner of a context's device buffers, per-call scratch buffers, the entry / exit macros of every
// wl_* function and the Whisper context.  No kernel file includes it.
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/wlb200.h"
#include "gemm.cuh"
#include "kernels.cuh"

using namespace wl;

// Every device buffer a context holds and its size: `bytes` is their sum, what wl_device_bytes and wl_mt_device_bytes
// report.  The buffers live on `device`; `st` is the context's stream.
struct DeviceMem {
  int device = 0;
  cudaStream_t st = nullptr;
  std::vector<std::pair<void*, size_t>> list;
  int64_t bytes = 0;

  template <class T>
  T* alloc(size_t n, bool zero = true) {
    void* p = nullptr;
    const size_t nb = std::max<size_t>(n, 1) * sizeof(T);
    cudaError_t e = cudaMalloc(&p, nb);
    if (e != cudaSuccess) {
      cudaGetLastError();   // an out-of-memory cudaMalloc is not sticky: leave no error behind for the next call
      char b[256];
      snprintf(b, sizeof(b), "cudaMalloc of %.1f MB failed: %s", n * sizeof(T) / 1048576.0, cudaGetErrorString(e));
      throw wl::Error{WL_ERR_NOMEM, b};
    }
    list.push_back({p, nb});
    bytes += (int64_t)nb;
    if (zero) {   // complete on return: callers copy into their buffers on the legacy stream as well as on st
      WL_CUDA(cudaMemsetAsync(p, 0, nb, st));
      WL_CUDA(cudaStreamSynchronize(st));
    }
    return (T*)p;
  }

  // A workspace that grows with the calls it serves: when `need` elements exceed `cap`, the buffer is replaced by one of
  // max(need, size) elements, and the one before it is freed.  This relies on no grown buffer being reachable from a
  // captured CUDA graph: a graph bakes in the device pointers it was captured with.
  template <class T>
  void grow(T*& p, long& cap, long need, long size = 0, bool zero = false) {
    if (need <= cap) return;
    cap = 0;
    replace(p, std::max(need, size), zero);
    cap = std::max(need, size);
  }
  // The step of grow for buffers that share one capacity: frees p (when set) and allocates n elements in its place.
  template <class T>
  void replace(T*& p, size_t n, bool zero = false) {
    release(p);
    p = alloc<T>(n, zero);
  }

  // Frees one buffer of the list once the stream's work is done, and clears the pointer.
  template <class T>
  void release(T*& p) {
    if (!p) return;
    if (st) cudaStreamSynchronize(st);
    auto it = std::find_if(list.begin(), list.end(), [&](const std::pair<void*, size_t>& a) { return a.first == (void*)p; });
    if (it != list.end()) {
      cudaFree(it->first);
      bytes -= (int64_t)it->second;
      list.erase(it);
    }
    p = nullptr;
  }

  // Frees the buffers allocated after the first `mark` ones (mark 0: all of them).
  void release_from(size_t mark) {
    if (list.size() > mark && st) cudaStreamSynchronize(st);
    while (list.size() > mark) {
      cudaFree(list.back().first);
      bytes -= (int64_t)list.back().second;
      list.pop_back();
    }
  }
};

// Device buffers of one call (a test hook, wl_decode_logits): outside the context's byte count, freed when the call
// returns, normally or through an exception.  Fills and copies are queued on the context's stream `st`.
struct Scratch {
  cudaStream_t st;
  std::vector<void*> p;
  explicit Scratch(cudaStream_t s) : st(s) {}
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  ~Scratch() {
    cudaStreamSynchronize(st);
    for (void* q : p) cudaFree(q);
  }
  // fill >= 0: every byte of the buffer is set to it
  template <class T>
  T* alloc(size_t n, int fill = -1) {
    void* q = nullptr;
    WL_CUDA(cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T)));
    p.push_back(q);
    if (fill >= 0) WL_CUDA(cudaMemsetAsync(q, fill, n * sizeof(T), st));
    return (T*)q;
  }
  template <class T>
  T* upload(const T* h, size_t n) {
    T* d = alloc<T>(n);
    WL_CUDA(cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, st));
    return d;
  }
  // waits for the stream: the copy is the last thing it runs
  template <class T>
  void download(T* h, const T* d, size_t n) {
    WL_CUDA(cudaMemcpyAsync(h, d, n * sizeof(T), cudaMemcpyDeviceToHost, st));
    WL_CUDA(cudaStreamSynchronize(st));
  }
};

// Entry and exit of every wl_* / wl_mt_* function that takes a context: a wl::Error becomes the return code and the
// context's last error.
#define API_BEGIN(ctx)                                          \
  if (!(ctx)) return WL_ERR_ARG;                                \
  try {                                                         \
    WL_CUDA(cudaSetDevice((ctx)->mem.device));
#define API_END(ctx)                                            \
  }                                                             \
  catch (const wl::Error& e) {                                  \
    (ctx)->err = e.msg;                                         \
    return e.code;                                              \
  }                                                             \
  catch (const std::exception& e) {                             \
    (ctx)->err = e.what();                                      \
    return WL_ERR_STATE;                                        \
  }                                                             \
  return WL_OK;

struct EncLayer {
  __half *w_qk, *w_v, *w_o, *w_fc1, *w_fc2;
  float *b_qk, *b_v, *b_o, *b_fc1, *b_fc2, *ln1_g, *ln1_b, *ln2_g, *ln2_b;
};
struct DecLayer {
  __half *w_qkv, *w_o, *w_qc, *w_kc, *w_vc, *w_oc, *w_fc1, *w_fc2;
  float *b_qkv, *b_o, *b_qc, *b_vc, *b_oc, *b_fc1, *b_fc2;
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *ln3_g, *ln3_b;
};

struct GraphEntry {
  cudaGraphExec_t exec = nullptr;
  long kernels = 0;  // kernel nodes per replay
};

struct wl_ctx {
  wl_config cfg;
  std::vector<int32_t> align_heads;
  std::string err;
  cudaStream_t st = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms[10] = {};   // [0] mel, [1] encode, [2] generate / session run, [5] session admit (prefill),
                            // [6] / [7] VAD front end / recurrence, [8] / [9] speaker embedding front end / network
  // per-kernel profiling of the dominant decode kernel (bench.py roofline): events around every cross-attention launch
  int prof_cross = 0;
  cudaEvent_t pev0 = nullptr, pev1 = nullptr;
  double prof_cross_ms = 0.0;
  long prof_cross_n = 0;
  int num_sms = 132;
  int d, H, Le, Ld, n_mels, V, Vld, Bm, Km, Rm, NS;
  bool finalized = false;
  DeviceMem mem;
  std::map<std::string, void*> dev;                 // raw uploaded tensors (fp16 for ndim>=2, f32 for 1-D)
  std::map<std::string, std::vector<int64_t>> shape;
  long graph_launched = 0;   // kernels executed through graph replays
  long capture_counted = 0;  // launcher calls that were captured, not executed

  // weights
  __half *w_conv1 = nullptr, *w_conv2 = nullptr, *emb = nullptr, *pos_dec = nullptr;
  float *b_conv1, *b_conv2, *pos_enc, *lnp_g, *lnp_b, *lnf_g, *lnf_b;
  std::vector<EncLayer> enc;
  std::vector<DecLayer> dec;
  // mel
  float *mel_window, *mel_twiddle, *mel_filt;
  int* mel_range;
  float* mel_pcm = nullptr;
  float* mel_out = nullptr;
  long *mel_off = nullptr, *mel_ooff = nullptr;
  unsigned* mel_gmax = nullptr;
  long mel_pcm_cap = 0, mel_out_cap = 0;
  int mel_last_B = 0, mel_last_frames = 0;
  // encoder workspaces
  int EB, AB;
  float* feat32;
  __half *feat16, *conv1o, *xn, *qk, *vt, *probs16, *attn, *hbuf;
  float *x, *scores;
  int* enc_slots_dev;
  // slot pool
  __half* enc16;   // [NS][1500][d]
  __half* ckv;     // [Ld][2][NS][H][1500][64]
  std::vector<int> slot_free;
  std::vector<char> slot_used;
  // decoder workspaces
  float *dx, *part1, *part2, *logits;
  __half *dxn, *datt, *dh, *kcache, *vcache;
  long cache_row_stride, cache_layer_stride;
  CrossAttnWorkspace xws;
  float* align_probs = nullptr;   // [R][H][1500]
  float* align_buf = nullptr;     // [B][nh][T_MAX][1500]
  long align_buf_cap = 0;
  int* align_heads_dev = nullptr;
  DecodeState ds;
  unsigned* suppress_mask;
  // pinned host staging
  int* h_int = nullptr;     // generic int staging
  float* h_flt = nullptr;
  size_t h_int_cap = 0, h_flt_cap = 0;
  std::map<std::string, GraphEntry> graphs;
  // WLB200_TIMELINE: in-graph per-kernel timestamps (common.cuh), dumped after every wl_generate
  unsigned long long* tl_dev = nullptr;
  std::string tl_path;
  // resident log-mel of the last wl_mel_device call (features never leave the GPU between mel and encoder)
  float *res_pcm = nullptr, *res_mel = nullptr;
  long res_pcm_cap = 0, res_mel_cap = 0;
  long *res_off = nullptr, *res_ooff = nullptr;
  int *res_frames = nullptr, *win_meta = nullptr;
  std::vector<int> res_frames_h;
  // K8 batched prefill workspaces (allocated on first use, grown on demand)
  struct Prefill {
    long cap_rows = 0;
    int *tok = nullptr, *pos = nullptr, *active = nullptr, *wrow = nullptr, *vslot = nullptr, *vdone = nullptr, *sel = nullptr;
    short* src = nullptr;
    float *x = nullptr, *qkv = nullptr, *qc = nullptr, *xpart = nullptr;
    __half *xn = nullptr, *att = nullptr, *h = nullptr;
    long rows_done = 0, calls = 0;   // statistics
    // K14 (align through the batched pass)
    int* row_b = nullptr;
    long row_b_cap = 0;
    float *aprobs = nullptr, *mat = nullptr, *tokp = nullptr;
    int *aT = nullptr, *anf = nullptr, *path = nullptr, *path_len = nullptr;
    long tokp_cap = 0;
  } pf;
  // Silero VAD: its own weights (wl_vad_load_tensor, independent of the Whisper weights and of finalize) and workspaces
  // grown on demand, at least to max_streams x 30 s on first use
  struct Vad {
    float* t[15] = {};            // device tensors in VAD_TENSORS order, kernel layout
    float *pcm = nullptr, *gx = nullptr, *probs = nullptr;
    long* off = nullptr;          // [2][off_cap]: pcm offsets, frame offsets
    long pcm_cap = 0, gx_cap = 0, frame_cap = 0, off_cap = 0;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  } vad;
  // Speaker embedding: its own weights (wl_spk_load_tensor) and workspaces grown on demand, at least to max_streams x 30 s
  // on first use
  struct Spk {
    std::vector<void*> t;         // device tensors in spk_tensors() order: conv weights fp16 [co][taps][ci] (the stem fp32
                                  // [32][9]), biases fp32, seg_1 fp32 transposed [5120][256]
    float *melw = nullptr, *pcm = nullptr, *feat = nullptr, *mean = nullptr, *pooled = nullptr, *emb = nullptr;
    int* mel_range = nullptr;
    __half *act[3] = {nullptr, nullptr, nullptr};
    long* off = nullptr;          // [6][off_cap]: pcm, frame and the four stages' position offsets
    long pcm_cap = 0, feat_cap = 0, act_cap[3] = {0, 0, 0}, stream_cap = 0;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  } spk;
  float* stage_f32 = nullptr;   // wl_load_tensor staging (freed by wl_finalize_weights)
  long stage_cap = 0;
  unsigned char* stage_bytes = nullptr;   // wl_load_tensor_typed staging: overflow count, payload, scales (freed likewise)
  long stage_bytes_cap = 0;
  // Decode session (N2, step-level continuous batching): a second decode state + self-attention cache whose stream
  // indices are admitted, decoded for a bounded number of token steps and collected independently of each other.
  // One-shot calls (wl_generate / wl_align / wl_detect_language) keep using `ds` / `kcache`, so they may run between two
  // wl_session_run calls without disturbing the streams in flight.
  struct Session {
    bool allocated = false, open = false;
    int cap = 0, K = 1, Kr = 1, NH = 1, nsplit = 1, use_graph = 1;
    float length_penalty = 1.f;
    SearchOpts so;
    DecodeState ds;
    __half *kcache = nullptr, *vcache = nullptr;
    unsigned* mask = nullptr;
    int* idx_dev = nullptr;
    int* peek_dev = nullptr;            // wl_session_peek staging [max_streams][PEEK_STRIDE]
    std::vector<int> hp, meta;          // host shadows: prompts [cap][T_MAX], per-stream metadata [META_ROWS][cap]
    std::vector<char> used, finished;   // index holds an admitted stream / that stream has finished decoding
    std::vector<int> nh;                // hypotheses the index's stream returns: N when it samples, else NH
    std::vector<int> rules;             // host shadow of the per-stream rule rows [RULE_ROWS][cap] (engine.cu)
    std::vector<float> lp;              // length penalty of the index's stream (collect / peek ranking)
    bool script_on = false;             // wl_test_session_script: scripted logits replace the decoder
    SearchScript script{};
    int live = 0;                       // admitted and still decoding
    long steps = 0, runs = 0, admitted = 0;
  } sess;
};

// engine.cu functions the kernel test hooks (hooks.cu) run on their own buffers; internal to the library, like the rest
// of the engine's helpers
namespace wl {
void encoder_attention_fused(cudaStream_t st, const __half* qk, const __half* vt, __half* out, int nb, int H, int d);
}
#define WL_INTERNAL __attribute__((visibility("hidden")))
WL_INTERNAL GemmOperand opnd(const __half* p, long rows, long k, long ld, int n1 = 1, long s1 = 0, int n2 = 1, long s2 = 0);
WL_INTERNAL void encoder_stem(wl_ctx* c, cudaStream_t st, int nb, const float* feat_dev, __half* feat16, __half* conv1o,
                              float* x);
WL_INTERNAL void encoder_attention_unfused(cudaStream_t st, const __half* qk, const __half* vt, __half* attn, float* scores,
                                           __half* probs16, int nb, int H, int AB);
WL_INTERNAL int enc_attn_streams(int d);
