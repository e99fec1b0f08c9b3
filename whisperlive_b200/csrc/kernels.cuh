// Launchers for the non-GEMM kernels of libwlb200 (K1, LN/softmax/prep, K10, K11, K12, K14).
#pragma once
#include "common.cuh"

namespace wl {

constexpr int T_MAX = 448;      // decoder positions
constexpr int S_ENC = 1500;     // encoder positions
constexpr int S_PAD = 1536;     // padded key dimension for materialised attention scores
constexpr int MAX_ROWS_PER_STREAM = 8;
constexpr int MAX_FINISHED = 16;   // largest round(K * patience): a beam search ends once it has this many hypotheses
// Hypothesis table of a stream: a step may close up to K hypotheses while fewer than max_cand exist, so the table
// holds max_cand - 1 + K <= MAX_FINISHED - 1 + MAX_ROWS_PER_STREAM entries (rounded up to 24).
constexpr int MAX_HYPS = MAX_FINISHED + MAX_ROWS_PER_STREAM;
constexpr int MAX_CAND = 16;    // 2 * beam, beam <= 8

// ---------------------------------------------------------------------------- K1 mel
struct MelTables {
  const float* window;      // [400]
  const float* twiddle;     // [400][2]
  const float* filt;        // [n_mels][201]
  const int* filt_range;    // [n_mels][2]
  int n_mels;
};
void mel_forward(cudaStream_t st, const float* pcm, const long* pcm_off, float* out, const long* out_off, unsigned* gmax,
                 const MelTables& t, int B, int max_frames);

// ---------------------------------------------------------------------------- Silero VAD (vad.cu)
// Device copies in the layout wl_vad_load_tensor stores: basis [256][258], conv weights [ci][3][co], w_ih [128][512],
// w_hh [512][128] (PyTorch rows, gate order i, f, g, o), w_out [128].
struct VadWeights {
  const float *basis, *w0, *b0, *w1, *b1, *w2, *b2, *w3, *b3, *w_ih, *w_hh, *b_ih, *b_hh, *w_out, *b_out;
};
// gx [total_frames][512]: the LSTM input projection of every frame (frame_off [B + 1] on the device)
void vad_front(cudaStream_t st, const VadWeights& w, const float* pcm, const long* pcm_off, const long* frame_off, int B,
               long total_frames, float* gx);
// probs [total_frames]: the recurrence over each stream's frames
void vad_lstm(cudaStream_t st, const VadWeights& w, const float* gx, const long* frame_off, int B, float* probs);

// ---------------------------------------------------------------------------- speaker embedding (spk.cu)
// fbank [frames][80] fp32 of every stream's frames (frame_off [B + 1]) and the per-stream bin means [B][80];
// melw [80][257] with the non-zero range of each bin in mel_range [80][2]
void spk_fbank(cudaStream_t st, const float* pcm, const long* pcm_off, const long* frame_off, int B, long frames,
               const float* melw, const int* mel_range, float* feat, float* mean);
// conv3x3 1 -> 32 of the CMN'd fbank (H = 80, positions = frames x 80), folded BN + ReLU, fp16 [position][32]
void spk_stem(cudaStream_t st, const float* feat, const float* mean, const long* frame_off, int B, long frames, const float* w,
              const float* bias, __half* out);
// out[m][n] = act(bias[n] + sum_k x(m, k) w[n][k] (+ res[m][n])): x fp16 [in position][C_in], w fp16 [C_out][taps][C_in]
// (tap = kh * 3 + kw, kh over frequency), positions of stream b at in_off[b] / out_off[b] (device, [B + 1]), time-major
struct SpkConvParams {
  const __half* x;
  const __half* w;
  const float* bias;
  const __half* res;   // nullptr, or [M][C_out] (may be `out`)
  __half* out;
  const long* in_off;
  const long* out_off;
  long M;
  int B, H_in, H_out, C_in, C_out, taps, stride, relu;
};
bool spk_conv_supported(int C_in, int C_out, int taps, int stride);
void spk_conv(cudaStream_t st, const SpkConvParams& p);
// TSTP of x fp16 [position][256] (H frequency rows) -> pooled [B][2 * 256 * H], then emb [B][256] = seg_1 (wt [2*256*H][256])
void spk_pool_embed(cudaStream_t st, const __half* x, const long* pos_off, int B, int H, const float* wt, const float* bias,
                    float* pooled, float* emb);

// A value produced by a split-K GEMM: v(r, c) = bias[c] + sum_s ptr[s * stride + r * ld + c]  (fixed order).
// nsplit == 1 with bias == nullptr is a plain buffer; nsplit == 0 means "nothing pending".
struct PartialSrc {
  const float* ptr = nullptr;
  int nsplit = 0;
  long stride = 0;
  const float* bias = nullptr;
};

// ---------------------------------------------------------------------------- elementwise / normalisation
// features f32 [B][n_mels][3000] -> fp16 [B][3002][n_mels] (rows 0 and 3001 are zero: conv padding)
void prep_features(cudaStream_t st, const float* feats, __half* out, int B, int n_mels);
// weight upload: fp32 [a][b][k] -> fp16 [a][k][b] (conv kernels; b = k = 1 is a plain cast)
void cast_weight_f16(cudaStream_t st, const float* in, __half* out, long a, long b, long k);
// typed weight upload (wl_load_tensor_typed): source element types, the WL_DT_* values of wlb200.h
enum WeightDtype { WDT_F32 = 0, WDT_F16 = 1, WDT_BF16 = 2, WDT_I8 = 3 };
// source of type dt [a][b][k] -> fp16 [a][k][b]; int8 sources are divided by scale[i / cols] (scale of type sdt).
// Finite values that round to +-inf in fp16 are added to *overflow.  `in` must be 16-byte aligned.
void convert_weight_f16(cudaStream_t st, const void* in, int dt, const void* scale, int sdt, __half* out, long a, long b, long k,
                        long cols, int* overflow, int num_sms);
// the same to fp32, no relayout (vectors, the encoder position table, the mel filters)
void convert_weight_f32(cudaStream_t st, const void* in, int dt, const void* scale, int sdt, float* out, long n, long cols,
                        int* overflow, int num_sms);
// window gather from the resident log-mel of wl_mel_device: feat[w][m][t] = t < len[w] ? mel[off[stream[w]] + m * frames[stream[w]] + seek[w] + t] : 0
// (the reference slices features[:, seek : seek + segment_size] and zero-pads to 3000 frames on the host: transcriber_faster_whisper.py:1115-1127)
void gather_windows(cudaStream_t st, const float* mel, const long* mel_off, const int* frames, const int* win_stream, const int* win_seek,
                    const int* win_len, float* feat, int n_windows, int n_mels);
// y = LayerNorm(x) * gamma + beta ; x f32 [rows][d] -> y fp16 [rows][d] (and optionally f32 copy)
void layernorm_rows(cudaStream_t st, const float* x, const float* gamma, const float* beta, __half* y, float* y32,
                    long rows, int d);
// decode step: x[r] += upd(r, :) (residual update pending from a split-K GEMM), then y = LayerNorm(x) as fp16
void layernorm_update_rows(cudaStream_t st, float* x, const PartialSrc& upd, const float* gamma, const float* beta, __half* y,
                           int rows, int d);
// out[r][c] = fp16(gelu(in(r, c))), rows x cols (cols % 4 == 0)
void gelu_cast(cudaStream_t st, const PartialSrc& in, __half* out, int rows, int cols);
// scores f32 [rows][ld_in] (first n valid) -> softmax(scale * s) as fp16 [rows][ld_out], columns >= n zeroed
void softmax_rows(cudaStream_t st, const float* s, __half* p, long rows, int n, int ld_in, int ld_out, float scale);

// ---------------------------------------------------------------------------- decoder state (device resident)
struct DecodeState {
  // per row
  int* tok_in;       // [R]
  int* pos;          // [R] position of tok_in == tokens already cached for the row
  int* active;       // [R]
  float* cum;        // [R]
  int* gen_len;      // [R]
  int* last_ts;      // [R] last generated timestamp token or -1
  int* row_done;     // [R]
  int* hist;         // [R][T_MAX] generated tokens
  short* src;        // [R][T_MAX] physical cache row holding position p of this row's sequence
  int* wrow;         // optional [R]: physical cache row the self-attention kernel WRITES row r's new k/v to (null: r itself;
                     //   the batched prefill runs every prompt position as its own row, all writing to the stream's first row)
  // per-row candidates produced by search_rows
  float* cand_val;   // [R][MAX_CAND]
  int* cand_tok;     // [R][MAX_CAND]
  float* nospeech_row;  // [R] softmax(raw logits)[no_speech] of the row (valid when computed)
  // per stream
  int* slot;         // [B]
  int* prompt;       // [B][T_MAX]
  int* prompt_len;   // [B]
  int* fed;          // [B] index of the prompt token fed at the current step
  int* sot_index;    // [B] or -1
  int* use_ts;       // [B]
  int* pre_n;        // [B] prompt tokens after the sot sequence (a ``prefix``): CT2 treats them as already-sampled text
  int* pre_last;     // [B] last / second-to-last of those tokens (-1 when absent) and the last timestamp among them:
  int* pre_penult;   // [B]   seeds of the timestamp rules' history
  int* pre_lts;      // [B]
  int* n_new;        // [B] max new tokens
  int* step;         // [B] generation steps done
  int* done;         // [B]
  int* n_alive;      // [B]
  float* no_speech;  // [B]
  int* hyp_count;    // [B]
  float* hyp_cum;    // [B][MAX_HYPS]
  int* hyp_len;      // [B][MAX_HYPS]
  int* hyp_tok;      // [B][MAX_HYPS][T_MAX]
  int* steps_run;    // [B] decoder steps executed for the stream (diagnostics)
  int* n_done;       // [1] number of finished streams
  int* steps_left;   // [1] decode steps the device-side loop may still run (conditional WHILE graph)
  // per-stream search (device tables: the captured graph does not depend on which streams sample)
  int* smode;        // [B] 0: the call's / session's search (SearchOpts); 1: Gumbel-max sampling, independent rows
  float* temp;       // [B] sampling temperature
  unsigned* nseed;   // [B] sampling noise seed
  int* nkey;         // [B] noise key: the stream index that goes into the noise hash
  int* nrows;        // [B] rows the stream uses (<= rows_per_stream); rows nrows .. rows_per_stream-1 stay inactive
  // per-stream logits rules (decode sessions only; null in the one-shot state, whose streams take SearchOpts).  Written
  // at admission -- the session's own options for a stream admitted without rules -- and read by the captured loop.
  int* r_max_initial;   // [B] max_initial_timestamp_index
  int* r_suppress_blank;// [B]
  int* r_beam;          // [B] beam width K_b <= rows_per_stream (1: greedy); a beam stream leaves rows K_b .. Kr-1 inactive
  int* r_max_cand;      // [B] round(K_b * patience): finished hypotheses that end a beam stream
  float* r_length_penalty; // [B] (session_peek's ranking)
  unsigned* r_mask;     // [B][mask_words] suppress bitmask
  int mask_words;
  int* brk;         // [2] decode sessions (step-level admission): [0] != 0 -> the device-side loop also ends as soon as a
                     //   stream finishes (so the host can hand its result out and refill the index); [1] = n_done at launch
  // teacher-forced mode (detect_language / align / logits test hook)
  int* force_len;    // [B] 0 = normal search; >0 = feed prompt only, then stop
  float* force_prob; // [B][T_MAX] P(prompt[i+1] | prompt[..i]) in teacher-forced mode
};

// Options shared by every stream of a call / session.  Whether a stream samples, at what temperature and with which
// noise is per stream: DecodeState::smode / temp / nseed / nkey / nrows.
struct SearchOpts {
  int beam;            // K (1 = greedy, or sampling when the stream's smode says so); a session stream's is r_beam
  int rows_per_stream; // Kr
  int max_cand;        // round(K * patience)
  int suppress_blank;
  int max_initial_ts;
  const unsigned* suppress_mask;  // device bitmask over the vocabulary
};

struct VocabIds {
  int vocab, vocab_ld, eot, sot, no_speech, no_timestamps, ts_begin, blank;
};

// x[r] = E[tok_in[r]] + P[pos[r]]  (f32) for active rows; also src[r][pos[r]] = r
void decoder_embed(cudaStream_t st, const DecodeState& s, const __half* emb, const __half* pos_emb, float* x, int R, int d);

// K10: self attention over the KV cache with beam indirection. qkv f32 [R][3d]; out fp16 [R][d].
void decoder_self_attn(cudaStream_t st, const DecodeState& s, const PartialSrc& qkv, __half* kcache, __half* vcache,
                       long cache_row_stride, __half* out, int R, int H, int d);

// K11: cross attention of the rows of each stream over its persistent encoder K/V.
//   q f32 [R][d]; K/V caches [slot][H][1500][64] fp16 (layer base pointers); out fp16 [R][d]
struct CrossAttnWorkspace {
  float* part;     // [B][H][nsplit][MAX_ROWS_PER_STREAM][66]  (m, l, o[64])
  float* probs;    // optional [R][H][1500] f32 attention probabilities (align mode) or nullptr
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // profiling: recorded right before / after the main kernel when set
};
void decoder_cross_attn(cudaStream_t st, const DecodeState& s, const PartialSrc& q, const __half* kc, const __half* vc,
                        long slot_stride, const CrossAttnWorkspace& ws, __half* out, int B, int rows_per_stream, int H,
                        int d, int nsplit);
int cross_attn_pick_nsplit(int B, int H, int num_sms, int rows_per_stream);

// K12: per-row masked log-softmax + top candidates, then per-stream beam / greedy update.
void search_rows(cudaStream_t st, const DecodeState& s, const float* logits, const SearchOpts& o, const VocabIds& v, int R);
void search_streams(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, int B);

// Test only (wl_test_search): the logits of every row as a pure function of the tokens the row has consumed, in place of
// the decoder's (tests/search_script.py restates it).  Inactive rows and the padding columns are NaN.
struct SearchScript {
  uint32_t seed;
  int pattern;   // 0 none, 1 one thread's strided set, 2 one float4 group, 3 vocabulary tail, 4 1/4 grid, 5 dominant; -1 mixed
};
void scripted_logits(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, const SearchScript& sc,
                     float* logits, int R);
// no_speech[b] = softmax(scripted logits of prompt[0 .. sot])[no_speech] for every stream whose sot precedes its last
// prompt token (what the batched prefill writes in production).  index != null (device, B entries): only those stream
// indices of a decode session; a listed index without such a sot gets 0.
void scripted_no_speech(cudaStream_t st, const DecodeState& s, const VocabIds& v, const SearchScript& sc, int B,
                        const int* index = nullptr);

// Last node of the loop body of the conditional WHILE graph: keep iterating while some stream is still decoding and the
// step budget is not used up (one thread; it runs after search_streams, so n_done is final for this step).
void loop_condition(cudaStream_t st, const DecodeState& s, cudaGraphConditionalHandle h, int B);

// initialise the state for a generate call (prompts already uploaded).  prefilled = 1: positions 0 .. P-2 of every prompt
// are already in the self-attention cache (K8 batched prefill): start at the last prompt token.
// index != null (device, B entries): initialise only those state indices of a running decode session -- their `done`
// flag was 1 and is counted in n_done, which drops by one per admitted stream instead of being reset.
void decode_init(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, int B, int R, int prefilled = 0,
                 const int* index = nullptr);

// Decode sessions, between two runs (never while the loop graph is in flight).  session_peek: the interim hypothesis of
// the n stream indices index[n] -> out [n][PEEK_STRIDE] ints: [0] token count (-1: finished without a hypothesis),
// [1] cum_logprob and [2] no-speech probability (float bits), [3] generation steps, [4] 1 = finished, [PEEK_HDR ..] the
// tokens; a finished stream also gives [5] the hypothesis slot reported, [6] its hypothesis count and at [PEEK_TAB ..]
// the lengths, then the cum_logprobs (float bits), of its MAX_HYPS hypothesis slots.
// session_cancel: the n listed indices go idle (done, rows inactive, n_done counts them).
constexpr int PEEK_TAB = 8;
constexpr int PEEK_HDR = PEEK_TAB + 2 * MAX_HYPS;
constexpr int PEEK_STRIDE = PEEK_HDR + T_MAX;
void session_peek(cudaStream_t st, const DecodeState& s, const SearchOpts& o, float length_penalty, const int* index, int* out,
                  int n);
void session_cancel(cudaStream_t st, const DecodeState& s, int Kr, const int* index, int n);

// ---------------------------------------------------------------------------- K8 batched prefill helpers (prefill.cu)
void prefill_embed(cudaStream_t st, const int* tok, const int* pos, const int* active, const int* wrow, const __half* emb,
                   const __half* pos_emb, float* x, short* src, int M, int d);
void prefill_kv_write(cudaStream_t st, const float* qkv, const int* pos, const int* active, const int* wrow, __half* kc, __half* vc,
                      long row_stride, int M, int H, int d);
void gather_rows(cudaStream_t st, const float* x, const int* rows, float* dst, int n, int d);
void row_prob(cudaStream_t st, const float* logits, int vocab, int vocab_ld, const int* target, const int* out_index, float* out, int n);

}  // namespace wl
