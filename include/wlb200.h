/* libwlb200 -- C ABI of the H100-native Whisper hot path behind WhisperLive's transcriber.
 *
 * Every entry point replaces one call the reference makes into its native engine
 * (ctranslate2.models.Whisper + faster_whisper.FeatureExtractor; neither is in the reference tree,
 * the citations are the reference-side CALL SITES, /root/reference/whisper_live/...):
 *
 *   wl_init / wl_load_tensor / wl_finalize_weights
 *        <- ctranslate2.models.Whisper(model_path, device, device_index, compute_type, ...)
 *           transcriber/transcriber_faster_whisper.py:634-643 (model load; backend/faster_whisper_backend.py:173-178)
 *   wl_mel               <- FeatureExtractor.__call__      transcriber_faster_whisper.py:862, :1759; batch_inference.py:258
 *   wl_encode            <- Whisper.encode                 transcriber_faster_whisper.py:1339-1348; batch_inference.py:271
 *   wl_generate          <- Whisper.generate               transcriber_faster_whisper.py:1394-1407; batch_inference.py:355
 *   wl_detect_language   <- Whisper.detect_language        transcriber_faster_whisper.py:1140, :1771; batch_inference.py:283
 *   wl_align             <- Whisper.align                  transcriber_faster_whisper.py:1657-1663
 *   wl_slots_release     <- StorageView lifetime           transcriber_faster_whisper.py:1055, :1820-1823
 *   wl_vad               <- faster_whisper.vad.get_speech_timestamps (the Silero model call) transcriber_faster_whisper.py:830-838
 *   wl_spk_embed         <- SpeakerDiarizer._compute_embedding (pyannote Inference)  diarization.py:100-118
 *   wl_mt_translate      <- ServeClientTranslation.translate_text (M2M100 generate)  backend/translation_backend.py:73-100
 *
 * Conventions: plain pointers and sizes only; the caller owns every host buffer; the library owns
 * device memory, streams, CUDA graphs.  Every function returns 0 or a negative WL_ERR_* code and
 * never throws / aborts; wl_last_error() returns the message of the last failure on that context.
 * A context is driven by one thread at a time (the scheduler thread); ctypes releases the GIL.
 */
#ifndef WLB200_H
#define WLB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WL_ABI_VERSION 14

typedef struct wl_ctx wl_ctx;

typedef struct wl_config {
  int32_t abi_version;   /* WL_ABI_VERSION */
  int32_t device;        /* CUDA ordinal */
  /* architecture */
  int32_t d_model, n_heads, enc_layers, dec_layers, n_mels, vocab;
  /* vocabulary ids the engine needs (ctranslate2 reads them from the model vocabulary) */
  int32_t eot, sot, no_speech, no_timestamps, timestamp_begin, blank;
  int32_t lang_begin, n_lang; /* language token ids are [lang_begin, lang_begin + n_lang) */
  /* capacity */
  int32_t max_streams;   /* streams per encode/generate call */
  int32_t max_beam;      /* decoder rows per stream (beam_size or num_hypotheses), <= 8 */
  int32_t enc_slots;     /* encoder-output / cross-KV slots in the pool (>= max_streams) */
  /* word alignment heads: pairs (layer, head) */
  int32_t n_align_heads;
  const int32_t* align_heads;
} wl_config;

typedef struct wl_gen_opts {
  int32_t beam_size;                 /* 1 = greedy / sampling */
  float patience;                    /* beam search ends with round(beam_size * patience) <= 16 hypotheses (more is an error) */
  int32_t num_hypotheses;
  float length_penalty;
  int32_t max_length;                /* CT2 max_length (448) */
  int32_t suppress_blank;
  int32_t max_initial_timestamp_index;
  int32_t sampling_topk;             /* 1 = arg-max, 0 = sample from the full distribution */
  float sampling_temperature;
  uint32_t seed;
  const int32_t* suppress_tokens;
  int32_t n_suppress;
  int32_t use_cuda_graph;            /* 1: capture the decoder step once per call shape */
  const int32_t* max_length_per_stream; /* optional [B]: overrides max_length per stream (ragged max_new_tokens) */
  int32_t prefill;                   /* K8: 0 = library default (batched prefill of the prompt), 1 = on, 2 = off (one decode
                                        step per prompt token; the parity tests compare the two) */
} wl_gen_opts;

/* A wl_init that fails frees whatever it had created; so does a wl_finalize_weights that fails (the tensors
 * wl_load_tensor uploaded stay until wl_destroy).  A failed load leaves no device memory behind but the context's. */
int wl_init(const wl_config* cfg, wl_ctx** out);
void wl_destroy(wl_ctx* ctx);
const char* wl_last_error(wl_ctx* ctx);   /* ctx may be NULL: last wl_init / wl_mem_info failure */

/* Device memory the context holds right now, in bytes, counted where the library allocates it: weights (the uploaded
 * tensors and their fused copies), the encoder workspaces and slot pool, the self-attention caches, both decode
 * states, an open session, the log-mel / prefill / align / VAD workspaces at their current grown size, the VAD weights,
 * the speaker-embedding weights and workspace, and the weight-load staging buffer while a load runs.  Not counted: buffers a call frees before it returns, CUDA graph executables and
 * the CUDA context of the process. */
int wl_device_bytes(wl_ctx* ctx, int64_t* out);
/* Free and total device memory of CUDA ordinal `device` (cudaMemGetInfo); needs no context, so a load can be checked
 * before it starts.  The query runs on its own thread: the calling thread's current device is untouched, and no
 * device other than `device` gets a CUDA context. */
int wl_mem_info(int32_t device, int64_t* free_bytes, int64_t* total_bytes);

/* Weights: float32 host tensors under HF WhisperForConditionalGeneration names
 * ("model.encoder.conv1.weight", ...), plus "mel_filters" [n_mels, 201]. */
int wl_load_tensor(wl_ctx* ctx, const char* name, const float* data, const int64_t* shape, int32_t ndim);
/* The same upload from the bytes as a checkpoint stores them (ABI 12): data is `dtype` (WL_DT_*).  For WL_DT_I8,
 * scale holds one value per leading-dimension row, of type scale_dtype (F32, F16 or BF16), and the weight is
 * (float)q / scale[row]; scale is ignored otherwise.  The device keeps exactly what wl_load_tensor keeps for the same
 * values (fp32 vectors, encoder position table and mel filters; fp16 with the conv re-layout for the rest), rounded
 * with __float2half_rn.  A finite value that would become +-inf in fp16 fails the call with WL_ERR_ARG, naming the
 * tensor and the count; nothing of that tensor stays on the device. */
#define WL_DT_F32 0
#define WL_DT_F16 1
#define WL_DT_BF16 2
#define WL_DT_I8 3
int wl_load_tensor_typed(wl_ctx* ctx, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim,
                         const void* scale, int32_t scale_dtype);
int wl_finalize_weights(wl_ctx* ctx);

/* K1. pcm: B waveforms concatenated, offsets[B+1] in samples.  out: per stream [n_mels, n_b/160 + 1]
 * float32 row-major, concatenated at out_offsets[B+1] (in floats).  Host pointers. */
int wl_mel(wl_ctx* ctx, const float* pcm, const int64_t* offsets, int32_t B, float* out, const int64_t* out_offsets);

/* K2-K7. features: host [B, n_mels, 3000] float32.  slots_out[B] receives pool slots that hold the
 * encoder output and the cross-attention K/V of each stream until released. */
int wl_encode(wl_ctx* ctx, const float* features, int32_t B, int32_t* slots_out);
int wl_slots_release(wl_ctx* ctx, const int32_t* slots, int32_t n);
int wl_slots_free_count(wl_ctx* ctx);
/* encoder output of one slot as float32 [1500, d_model] (host) */
int wl_encoder_output(wl_ctx* ctx, int32_t slot, float* out);

/* K8-K13. prompts: B token lists concatenated, prompt_off[B+1].  Outputs (host):
 *   out_ids   [B, num_hypotheses, 448] int32      out_len  [B, num_hypotheses]
 *   out_score [B, num_hypotheses] (cum_logprob / len^length_penalty)
 *   out_no_speech [B]                              out_steps [B] decoder steps executed */
int wl_generate(wl_ctx* ctx, const int32_t* slots, int32_t B, const int32_t* prompts, const int32_t* prompt_off,
                const wl_gen_opts* opts, int32_t* out_ids, int32_t* out_len, float* out_score, float* out_no_speech,
                int32_t* out_steps);

/* N2. Decode session: step-level continuous batching -- replaces the run-to-completion batches of the reference's
 * BatchInferenceWorker._process_multi (whisper_live/batch_inference.py:155-187; its gaps :259, :334-339).
 *   wl_session_open    fixes the search options (wl_generate's beam or greedy search; sampling is chosen per stream at
 *                      admission) and the number of stream indices (<= max_streams); every index starts idle.
 *                      Re-opening is allowed once nothing is decoding.
 *   wl_session_admit   puts n streams into idle indices: prompts prefilled in one batched pass (K8), search state
 *                      initialised; the streams already decoding are untouched.  max_length[n] like wl_generate's.
 *   wl_session_admit_ex the same with a search per stream (search[n], or NULL = wl_session_admit): sample = 1 decodes
 *                      the stream by Gumbel-max sampling over the full distribution, num_hypotheses independent rows
 *                      (1 .. the session's rows per stream: beam_size, or num_hypotheses when beam_size = 1), with the
 *                      draws of wl_generate(seed) for the stream at batch position noise_key.  The result does not
 *                      depend on which other streams share the loop, and admitting it captures no new graph.  A bad
 *                      spec (num_hypotheses out of range, temperature <= 0 or not finite, negative key) fails the
 *                      whole call before anything is staged: every index stays free.  sample = 0 is the session's own
 *                      search (the other fields are ignored).
 *                      rules[n] (ABI 13; NULL, or rules = 0 for a stream: the session's options) gives a stream its own
 *                      logits rules -- suppress list, suppress_blank, max_initial_timestamp_index -- and its own
 *                      length_penalty and patience (the finished hypotheses that end a beam stream; the ranking of
 *                      wl_session_collect and wl_session_peek), and (ABI 14) its own beam_size: 1 .. the session's rows
 *                      per stream.  A stream of width 1 is wl_generate's greedy search over the session's num_hypotheses
 *                      rows; a wider one a beam search over its first beam_size rows, the others staying inactive.  They
 *                      live in per-index device tables the captured loop reads: admitting a stream with its own rules or
 *                      width captures no new graph, and its result does not depend on the other streams.  A width above
 *                      the rows per stream, round(beam_size * patience) above 16, or any other bad field fails the call
 *                      before anything is staged, with the field named.
 *   wl_session_run     runs the device-side token loop over every admitted stream for at most max_steps steps; with
 *                      break_on_finish it also returns as soon as some stream has finished.  done_out[capacity]: 1 for
 *                      indices whose stream is finished and not yet collected.  steps_ran: token steps executed.
 *   wl_session_collect hypotheses of one finished index (outputs like one stream of wl_generate at the stream's own
 *                      search and width); the index goes idle.
 *                      out_ids / out_len / out_score hold the index's own hypothesis count: the sampled stream's
 *                      num_hypotheses, else the session's.
 *   wl_session_peek    the interim hypothesis of n indices (index[n]), for text before a stream finishes: out_ids
 *                      [n][448], out_len / out_score / out_no_speech / out_step / out_final [n] (the last three may be
 *                      NULL).  A stream still decoding reports its leading row -- row 0 for the session's own search
 *                      (beam search keeps its best live beam there), the alive row with the highest cum_logprob (lowest
 *                      row on ties) for a sampled stream -- as the tokens generated so far (the layout of
 *                      wl_session_collect), score cum_logprob / len^length_penalty, step = generation steps done, final = 0.
 *                      A finished, uncollected index reports the hypothesis wl_session_collect returns first, final = 1,
 *                      and stays collectable (ranked with collect's own arithmetic).  One kernel, one device-to-host copy,
 *                      one stream synchronise -- plus one small copy in the rare case of a finished index whose last-bit
 *                      near-tie the device ranked the other way (length_penalty other than 0 or 1); legal between
 *                      two wl_session_run calls.  A beam stream's interim hypothesis need not be a prefix of its final one.
 *   wl_session_cancel  n distinct indices go idle at once: a running stream stops decoding, a finished one's result is
 *                      discarded; each index can be admitted again right away.  The streams in flight are untouched.
 *   Both fail before anything is launched, with no index changed, when an index is idle or out of range.
 *   wl_session_close   drops whatever is still in flight.
 * The session has its own decode state and self-attention cache: wl_generate / wl_align / wl_detect_language /
 * wl_encode may be called between two wl_session_run calls (temperature-fallback retries, word alignment of a finished
 * window, the encoder pass of a stream about to be admitted). */
int wl_session_open(wl_ctx* ctx, const wl_gen_opts* opts, int32_t capacity);
int wl_session_admit(wl_ctx* ctx, int32_t n, const int32_t* index, const int32_t* slots, const int32_t* prompts,
                     const int32_t* prompt_off, const int32_t* max_length);
typedef struct wl_stream_search {
  int32_t sample;            /* 0: the session's search options; 1: Gumbel-max sampling over the full distribution */
  int32_t num_hypotheses;    /* sampling: 1 .. the session's rows per stream */
  float temperature;         /* sampling: > 0, finite */
  uint32_t seed;             /* sampling noise = that of wl_generate(seed) ... */
  int32_t noise_key;         /* ... for the stream at batch position noise_key (>= 0) */
} wl_stream_search;
typedef struct wl_stream_rules {
  int32_t rules;             /* 0: the session's options (the other fields are ignored); 1: the fields below */
  int32_t beam_size;         /* 0: the session's; else 1 (greedy) .. the session's rows per stream (its beam_size, or its
                                num_hypotheses when its beam_size is 1) */
  float patience;            /* beam search ends with round(beam_size * patience) <= 16 hypotheses (this stream's width) */
  float length_penalty;
  int32_t suppress_blank;
  int32_t max_initial_timestamp_index;
  const int32_t* suppress_tokens;   /* ids outside the vocabulary are ignored, as in wl_gen_opts */
  int32_t n_suppress;
} wl_stream_rules;
int wl_session_admit_ex(wl_ctx* ctx, int32_t n, const int32_t* index, const int32_t* slots, const int32_t* prompts,
                        const int32_t* prompt_off, const int32_t* max_length, const wl_stream_search* search,
                        const wl_stream_rules* rules);
int wl_session_run(wl_ctx* ctx, int32_t max_steps, int32_t break_on_finish, int32_t* done_out, int32_t* steps_ran);
int wl_session_collect(wl_ctx* ctx, int32_t index, int32_t* out_ids, int32_t* out_len, float* out_score, float* out_no_speech,
                       int32_t* out_steps);
int wl_session_peek(wl_ctx* ctx, int32_t n, const int32_t* index, int32_t* out_ids, int32_t* out_len, float* out_score,
                    float* out_no_speech, int32_t* out_step, int32_t* out_final);
int wl_session_cancel(wl_ctx* ctx, int32_t n, const int32_t* index);
int wl_session_close(wl_ctx* ctx);

/* K13. probs [B, n_lang] softmax over the language tokens after feeding <|startoftranscript|>. */
int wl_detect_language(wl_ctx* ctx, const int32_t* slots, int32_t B, float* probs);

/* K14. Teacher-forced pass over start_seq + <|notimestamps|> + text + <|endoftext|> per stream.
 *   text/text_off[B+1]; num_frames[B]; pairs_out [cap_pairs][2] (text_idx, time_idx) concatenated at
 *   pair_off[B+1] (written); tok_probs concatenated like text. */
int wl_align(wl_ctx* ctx, const int32_t* slots, int32_t B, const int32_t* start_seq, int32_t n_start, const int32_t* text,
             const int32_t* text_off, const int32_t* num_frames, int32_t median_width, int32_t* pairs_out,
             int32_t cap_pairs, int32_t* pair_off, float* tok_probs);

/* Diagnostics / parity hooks (used by tests and bench.py, not by the reference-facing path) */
/* teacher-forced logits: tokens concatenated at tok_off[B+1]; logits_out [sum T, vocab] float32 */
int wl_decode_logits(wl_ctx* ctx, const int32_t* slots, int32_t B, const int32_t* tokens, const int32_t* tok_off,
                     float* logits_out);
/* C[z] = A[z] (MxK) * B[z]^T (NxK) (+bias[n]) on the wgmma path (use_simt=0) or the CUDA-core checker.  opts:
 *   bits 0-1 output: 0 fp32; 1 fp32 plus the fp32 residual read from c and updated in place; 2 fp16;
 *            3 fp16 head-split layout (cross-KV cache) of M / hs rows per stream into slots in reverse stream order,
 *            c = [slot][N / 64][hs][64] with the 16-byte pieces of a row XOR-swizzled by (s & 7), hs = opts >> 8
 *   bit 2: A is one matrix shared by the batch (a holds M x K); bit 3: the same for B
 *   bits 4-5 kernel: 0 as gemm_tn picks it, 1 the classic kernel, 2 the ping-pong kernel (N tiles of 128 only)
 *   bit 6: bias indexed by m with the row-major store (always so with transposed_store) */
int wl_test_gemm(wl_ctx* ctx, const uint16_t* a_f16, const uint16_t* b_f16, const float* bias, float* c, int32_t M, int32_t N,
                 int32_t K, int32_t batch, int32_t transposed_store, int32_t gelu, int32_t use_simt, int32_t opts);
/* the GEMM kernel gemm_tn picks for this shape on this device: 1 classic, 2 ping-pong */
int wl_gemm_variant(wl_ctx* ctx, int32_t M, int32_t N, int32_t K, int32_t batch, int32_t* variant_out);
/* test hook of the small-batch decode GEMM (csrc/wgemm.cu, R <= 32): out[R][n_out] = X[R][K] W[n_out][K]^T with the fused
 * epilogue `mode` -- 0: + bias; 1: out += acc + bias (residual in place); 2: gelu(acc + bias) through fp16;
 * 3: split-K partial sums (K > 1280), summed by the hook */
int wl_test_wgemm(wl_ctx* ctx, const uint16_t* w_f16, const uint16_t* x_f16, const float* bias, float* out, int32_t R,
                  int32_t n_out, int32_t K, int32_t mode);
/* Test hooks of the decode-step kernels of the default path for more than 16 decoder rows.  Each launches the kernels
 * exactly as the decode step does, but without programmatic dependent launch, on device copies of the host inputs.
 *
 * Split-K decode GEMM (csrc/dec_gemm.cu): out [nsplit][R][n_out] = the raw fp32 partial sum of W[n_out][K] X[R][K]^T
 * over each K range (ranges of ceil(k-blocks / nsplit) 64-wide k-blocks, the last one shorter).  nsplit = 0 takes the
 * engine's plan, dec_gemm_split_plan(n_out, R, K, 8).  The split used is written to nsplit_out; a split that cannot be
 * formed (an empty K range) is an error.  out = NULL only resolves and reports the split. */
int wl_test_dec_gemm(wl_ctx* ctx, const uint16_t* w_f16, const uint16_t* x_f16, float* out, int32_t R, int32_t n_out,
                     int32_t K, int32_t nsplit, int32_t* nsplit_out);
/* K11 cross attention + the combine kernel.  q = q_bias + the q_nsplit (1..4) fp32 partials q_part [q_nsplit][R][H*64],
 * R = B * rows_per_stream; q_bias may be NULL.  k_pool / v_pool: fp16 [n_slots][H][1500][64] in the pool layout, i.e.
 * the 16-byte piece p of key s stored at piece p ^ (s & 7) (wl_test_gemm opts 3).  Stream b reads slot[b] and is
 * skipped when done[b] != 0.  nsplit: key ranges per (stream, head), one of 1, 2, 3, 4, 6, 12, or 0 for the engine's
 * choice (cross_attn_pick_nsplit); the value used goes to nsplit_out.  out [R][H*64]: the fp16 output as float, the
 * buffer filled with `sentinel` before the launch.  probs (nsplit 1 only, or NULL): [R][H][1500] attention
 * probabilities, 0 for the rows of done streams. */
int wl_test_cross_attn(wl_ctx* ctx, const float* q_part, const float* q_bias, int32_t q_nsplit, const uint16_t* k_pool,
                       const uint16_t* v_pool, int32_t n_slots, const int32_t* slot, const int32_t* done, int32_t B,
                       int32_t rows_per_stream, int32_t H, int32_t nsplit, int32_t* nsplit_out, float sentinel, float* out,
                       float* probs);
/* K10 self attention.  qkv = qkv_bias + the nsplit (1..8) partials qkv_part [nsplit][R][3*H*64]; nsplit 1 with
 * qkv_bias NULL is the plain form.  Caches fp16 [n_rows][H][448][64], updated in place (the new k / v of row r at
 * position pos[r] of cache row wrow[r], or of row r when wrow is NULL).  src [R][448]: cache row holding position p of
 * row r.  Rows with active[r] == 0 are skipped.  out [R][H*64]: the fp16 output as float, filled with `sentinel`
 * before the launch. */
int wl_test_self_attn(wl_ctx* ctx, const float* qkv_part, const float* qkv_bias, int32_t nsplit, uint16_t* k_cache,
                      uint16_t* v_cache, int32_t n_rows, const int16_t* src, const int32_t* pos, const int32_t* active,
                      const int32_t* wrow, int32_t R, int32_t H, float sentinel, float* out);
/* The consumers that fold split-K partials (part [nsplit][rows][cols], bias [cols] or NULL).  mode 0,
 * layernorm_update_rows: x [rows][cols] += bias + the nsplit (0..8) partials in place, y = LayerNorm(x) * gamma + beta.
 * mode 1, gelu_cast: y = gelu(bias + the nsplit (1..8) partials); x, gamma, beta unused.  y: the fp16 result as float. */
int wl_test_fold(wl_ctx* ctx, int32_t mode, float* x, const float* part, int32_t nsplit, const float* bias,
                 const float* gamma, const float* beta, float* y, int32_t rows, int32_t cols);
/* Test hooks of the encoder-pass kernels.  Each runs the code the encoder pass runs, on device copies of the inputs.
 *
 * Encoder self-attention of nb streams, H heads (d = 64 H).  qk: fp16 [nb][1500][2d], Q | K as the QK GEMM writes it;
 * vt: fp16 [nb][d][1536], V transposed per head, the 36 pad columns taken as given.  out: fp16 [nb * 1500 + 128][d],
 * uploaded as the caller filled it and copied back whole (128 guard rows after the last stream).  path 0: the fused
 * flash-attention kernel; path 1: the unfused scores GEMM + softmax_rows + P V GEMM in sub-passes of ab streams
 * (ab = 0: the engine's rule, 2 streams for d >= 1024, else 4). */
int wl_test_enc_attn(wl_ctx* ctx, const uint16_t* qk_f16, const uint16_t* vt_f16, uint16_t* out_f16, int32_t nb, int32_t H,
                     int32_t path, int32_t ab);
/* The conv stem with the loaded conv weights, biases and positional table: feats [nb][n_mels][3000] f32 -> x_out
 * [nb][1500][d] f32, the residual stream after conv2 + GELU + positions. */
int wl_test_enc_stem(wl_ctx* ctx, const float* feats_f32, float* x_out_f32, int32_t nb);
/* A tensor uploaded by wl_load_tensor / wl_load_tensor_typed as the device holds it, before wl_finalize_weights: fp32
 * (vectors, encoder position table, mel filters) or fp16 bits after the conv re-layout, into out. */
int wl_test_read_weight(wl_ctx* ctx, const char* name, void* out);
/* layernorm_rows over x [rows][d] (d a multiple of 4, at most 1280).  y16_as_f32 (the fp16 output as float) and y32
 * (the fp32 output), either may be NULL: [rows + 8][d], uploaded as the caller filled them (y16 rounded to fp16) and
 * copied back whole, so the 8 guard rows after the last one show what the kernel wrote past it. */
int wl_test_layernorm(wl_ctx* ctx, const float* x_f32, const float* gamma, const float* beta, float* y16_as_f32, float* y32,
                      int32_t rows, int32_t d);
/* Search on scripted logits: wl_generate with the decoder replaced.  Each step's logits are a pure function of the
 * tokens a row has consumed (tests/search_script.py restates the function); no encoder slot is read.  Everything else
 * -- prompt upload, decode_init, the captured or host-driven loop, the search kernels, the hypothesis ranking -- is
 * wl_generate's own code.  opts->prefill = 1: the stream starts at its last prompt token (the no-speech probability is
 * then written from the scripted logits at the sot position); 2: the prompt is fed token by token.  Outputs as
 * wl_generate, plus out_hyp_count [B] (hypotheses each stream finished with) and, when not NULL, out_logits
 * [B * rows per stream][(vocab + 3) / 4 * 4]: the logits of the first decode step. */
typedef struct wl_search_script {
  uint32_t seed;
  int32_t pattern;   /* 0 none, 1 one selection thread's strided set, 2 one float4 group, 3 the vocabulary's last tokens,
                        4 a grid of 1/4, 5 one or two dominant tokens; -1 chosen per step */
} wl_search_script;
int wl_test_search(wl_ctx* ctx, int32_t B, const int32_t* prompts, const int32_t* prompt_off, const wl_gen_opts* opts,
                   const wl_search_script* script, int32_t* out_ids, int32_t* out_len, float* out_score, float* out_no_speech,
                   int32_t* out_steps, int32_t* out_hyp_count, float* out_logits);
/* Test hook: with script != NULL, the open decode session's streams are decoded on the scripted logits of
 * wl_test_search instead of the decoder, from the next admission on (slots are not read; the stream starts at its last
 * prompt token, as with opts->prefill = 1); NULL goes back to the decoder.  Only while no stream is decoding;
 * wl_session_open resets it. */
int wl_test_session_script(wl_ctx* ctx, const wl_search_script* script);
/* device-resident timing of the GEMM kernel: C = A(MxK) * B(NxK)^T, `iters` launches between CUDA events;
 * bn = 0 picks the tile like the engine does. ms_out = average milliseconds per launch. */
int wl_bench_gemm(wl_ctx* ctx, int32_t M, int32_t N, int32_t K, int32_t batch, int32_t iters, int32_t flags,
                  float* ms_out); /* flags: 1 transposed store, 2 bias, 4 GELU, 8 fp32 output + fp32 residual,
                                   16 bias indexed by m, 32 A shared by the batch, 64 output row pitch padded to 64 */
/* launches of library kernels since wl_init (gpu_launches accounting in bench.py) */
int64_t wl_kernel_launches(wl_ctx* ctx);
/* time (ms, CUDA events on the library stream) of the last wl_mel / wl_encode / wl_generate device work;
 * which = 3: average ms per cross-attention kernel launch since wl_profile_cross_attn(ctx, 1), 4: launches timed;
 * 2 also holds the last wl_session_run, 5 the last wl_session_admit */
float wl_last_device_ms(wl_ctx* ctx, int32_t which /*0 mel, 1 encode, 2 generate, 3/4 cross-attention profile,
                                                      6 / 7 the last wl_vad's front end / recurrence,
                                                      8 / 9 the last wl_spk_embed's fbank + CMN / network*/);
/* enable = 1: wl_generate calls made WITHOUT a CUDA graph bracket every cross-attention launch (K11, the dominant
 * decode kernel) with CUDA events on the library stream -- bench.py's live roofline measurement.  Resets the sums. */
int wl_profile_cross_attn(wl_ctx* ctx, int32_t enable);
/* K1 with the features kept in HBM (replaces FeatureExtractor + pad_or_trim + the feature upload of encode inside
 * B200WhisperModel.transcribe_batch; reference call sites transcriber_faster_whisper.py:862, :1115-1127, :1348):
 * wl_mel_device computes the log-mel of B waveforms (frames_out[b] = len/160 + 1, like wl_mel) and keeps it resident
 * until the next wl_mel_device call; wl_encode_windows encodes B windows cut from it -- window w is frames
 * [seek, seek + len) of stream win_stream[w], zero-padded to 3000 on the device -- into fresh encoder slots. */
int wl_mel_device(wl_ctx* ctx, const float* pcm, const int64_t* offsets, int32_t B, int32_t* frames_out);
int wl_encode_windows(wl_ctx* ctx, int32_t B, const int32_t* win_stream, const int32_t* win_seek, const int32_t* win_len,
                      int32_t* slots_out);
/* resident-input variants for bench.py `value`: inputs already uploaded by the previous call of the
 * host variant are reused (no H2D, no D2H) */
int wl_mel_resident(wl_ctx* ctx);
int wl_encode_resident(wl_ctx* ctx, int32_t B, const int32_t* slots);

/* Silero VAD (16 kHz), fp32.  wl_vad_load_tensor takes a float32 host tensor under one of the fixed names
 *   vad.stft.basis [258, 1, 256]     vad.conv0.weight [128, 129, 3]  vad.conv0.bias [128]
 *   vad.conv1.weight [64, 128, 3]    vad.conv1.bias [64]             vad.conv2.weight [64, 64, 3]   vad.conv2.bias [64]
 *   vad.conv3.weight [128, 64, 3]    vad.conv3.bias [128]
 *   vad.lstm.weight_ih / vad.lstm.weight_hh [512, 128], vad.lstm.bias_ih / vad.lstm.bias_hh [512]  (gate order i, f, g, o)
 *   vad.out.weight [1, 128, 1]       vad.out.bias [1]
 * and rejects any other name or shape; it may be called before or after wl_finalize_weights (loading a name again
 * replaces it).  wl_vad: pcm holds B waveforms concatenated at offsets[B+1] (samples); a waveform of n > 0 samples has
 * n / 512 + 1 frames (the audio padded to the next multiple of 512, a whole frame of zeros when n already is one), one of
 * 0 samples has none.  probs_out receives the speech probability of every frame, stream b's at
 * [prob_off[b], prob_off[b+1]); prob_off must match the frame counts.  One upload, one download; host pointers.  Fails
 * when any VAD tensor is missing. */
int wl_vad_load_tensor(wl_ctx* ctx, const char* name, const float* data, const int64_t* shape, int32_t ndim);
int wl_vad(wl_ctx* ctx, const float* pcm, const int64_t* offsets, int32_t B, float* probs_out, const int64_t* prob_off);

/* Speaker embedding: the wespeaker ResNet34 of pyannote's wespeaker-voxceleb-resnet34-LM over Kaldi fbank (the protocol
 * whisperlive_b200/speaker.py names).  wl_spk_load_tensor takes a float32 host tensor, BatchNorm already folded into each
 * conv, under one of the fixed names
 *   spk.conv1.weight [32, 1, 3, 3]                      spk.conv1.bias [32]
 *   spk.layerL.i.conv1.weight / .conv2.weight [C, C_in, 3, 3] (.conv1.bias / .conv2.bias [C])
 *   spk.layerL.0.shortcut.weight [C, C_in, 1, 1]        spk.layerL.0.shortcut.bias [C]        (L = 2, 3, 4)
 *     L = 1..4 with C = 32, 64, 128, 256 and i < 3, 4, 6, 3; C_in = C except for the first conv / shortcut of a stage
 *   spk.seg_1.weight [256, 5120]                        spk.seg_1.bias [256]
 * and rejects any other name or shape; it may be called before or after wl_finalize_weights (loading a name again
 * replaces it).  wl_spk_embed: pcm holds B waveforms in [-1, 1] concatenated at offsets[B+1] (samples, 16 kHz), each at
 * least 400 samples (one fbank frame; checked before anything is launched); emb_out [B][256] receives the embeddings.
 * A segment of fewer than 8 frames pools over one time step, whose unbiased variance is 0/0: its std half is NaN, as in
 * PyTorch.  One upload of the samples and the offset tables, one download; fp16 activations, fp32 accumulation; a
 * stream's embedding does not depend on the other streams of the call.  Fails when any tensor is missing. */
int wl_spk_load_tensor(wl_ctx* ctx, const char* name, const float* data, const int64_t* shape, int32_t ndim);
int wl_spk_embed(wl_ctx* ctx, const float* pcm, const int64_t* offsets, int32_t B, float* emb_out);
/* Test hook: wl_spk_embed's fbank launch over B waveforms (offsets[B+1], each >= 400 samples): feat_out [frames][80], the
 * log mel energies before CMN, streams concatenated (stream b has 1 + (n_b - 400) / 160 frames). */
int wl_test_spk_fbank(wl_ctx* ctx, const float* pcm, const int64_t* offsets, int32_t B, float* feat_out);
/* Test hook: the launch wl_spk_embed makes for one convolution, on device copies of the inputs.  x fp16 [positions][C_in]
 * with B streams of frames[b] time steps x H_in frequency rows, time-major per stream; w fp16 [C_out][ksize * ksize][C_in]
 * (tap = kh * ksize + kw, kh over frequency); bias fp32 [C_out]; res fp16 [out positions][C_out] or NULL; relu 0/1;
 * out fp16 [out positions][C_out] (uploaded as given, copied back whole).  ksize 3 pads by one, ksize 1 not; stride 2
 * gives ceil(H_in / 2) x ceil(frames / 2) outputs per stream. */
int wl_test_spk_conv(wl_ctx* ctx, const uint16_t* x_f16, const int64_t* frames, int32_t B, int32_t H_in, int32_t C_in,
                     int32_t C_out, int32_t ksize, int32_t stride, const uint16_t* w_f16, const float* bias,
                     const uint16_t* res_f16, int32_t relu, uint16_t* out_f16);

/* Translation: an M2M100 encoder-decoder (SMaLL-100) with Hugging Face's beam search, in a context of its own (one per
 * process, shared by every connection; it belongs to no Whisper model).  wl_mt_load_tensor takes float32 host tensors
 * under the engine's names (whisperlive_b200/translation.py maps the checkpoint onto them):
 *   shared [vocab, d] (token embedding and LM head)     positions [max_positions + 2, d] (sinusoidal table, pad row zero;
 *   a source token's row is pad + its count of non-pad tokens so far, a decoder token's pad + 1 + its position)
 *   enc.L.{ln1,ln2}.{w,b} [d]   enc.L.qkv.w [3d, d]  enc.L.qkv.b [3d]  enc.L.out.{w [d, d], b [d]}
 *   enc.L.fc1.{w [ffn, d], b [ffn]}  enc.L.fc2.{w [d, ffn], b [d]}  enc.ln.{w,b} [d]
 *   dec.L.{ln1,ln2,ln3}.{w,b}, dec.L.qkv.*, dec.L.out.*, dec.L.xq.{w [d, d], b}, dec.L.xout.*, dec.L.fc1.*, dec.L.fc2.*,
 *   dec.ln.{w,b}, dec.xkv.w [dec_layers * 2d, d] and dec.xkv.b [dec_layers * 2d] (layer L's cross K then V)
 * wl_mt_translate: B segments of source ids packed at src_off[B+1] (each 1 .. max_positions - 2 tokens, at most
 * max_src_tokens in all, B <= capacity_segments; opts->max_length <= max_positions + 1); out_ids [B][opts->max_length] receives the best hypothesis of each
 * segment without the decoder start token (EOS included when it ended on one), out_len its length, out_score its
 * length-normalised score (beam search) or cumulative log-probability (greedy).  One upload, one download; the token
 * loop is one CUDA graph whose loop ends on the device.  A segment's result does not depend on the other segments. */
typedef struct wl_mt_ctx wl_mt_ctx;

typedef struct wl_mt_config {
  int32_t abi_version;   /* WL_ABI_VERSION */
  int32_t d_model, n_heads, enc_layers, dec_layers, ffn, vocab, max_positions;
  int32_t pad_id;        /* padding_idx: the zero row of the position table */
  float embed_scale;     /* sqrt(d_model) with scale_embedding, else 1 */
  int32_t max_src_tokens;/* packed source tokens per call */
} wl_mt_config;

typedef struct wl_mt_opts {
  int32_t num_beams;     /* 1 = greedy, <= max_beam */
  int32_t max_length;    /* decoder start token included, <= 448 */
  float length_penalty;
  int32_t early_stopping;/* 0 False, 1 True, 2 "never" */
  int32_t decoder_start, eos, forced_bos, forced_eos; /* -1: no forced token */
  int32_t use_cuda_graph;
} wl_mt_opts;

int wl_mt_init(const wl_mt_config* config, int32_t device, int32_t capacity_segments, int32_t max_beam, wl_mt_ctx** out);
void wl_mt_destroy(wl_mt_ctx* ctx);
const char* wl_mt_last_error(wl_mt_ctx* ctx);
int wl_mt_load_tensor(wl_mt_ctx* ctx, const char* name, const float* data, const int64_t* shape, int32_t ndim);
int wl_mt_finalize(wl_mt_ctx* ctx);
int wl_mt_device_bytes(wl_mt_ctx* ctx, int64_t* out);
int wl_mt_translate(wl_mt_ctx* ctx, const int32_t* src_ids, const int32_t* src_off, int32_t B, const wl_mt_opts* opts,
                    int32_t* out_ids, int32_t* out_len, float* out_score);
/* Test hook: the encoder self-attention launch.  qkv fp16 [n][3 * 64 H] (q | k | v) of B segments at off[B+1] ->
 * out fp16 [n][64 H] (uploaded as given, copied back whole). */
int wl_test_mt_attn(wl_mt_ctx* ctx, const uint16_t* qkv_f16, const int32_t* off, int32_t B, int32_t H, uint16_t* out_f16);
/* Test hook: the decoder cross-attention launch.  q fp32 [R][64 H], kv fp16 [n][ldkv] with K at column koff and V at
 * voff, B segments at off[B+1], row r of segment r / rows_per_seg -> out fp16 [R][64 H] (uploaded, copied back whole). */
int wl_test_mt_cross_attn(wl_mt_ctx* ctx, const float* q, const uint16_t* kv_f16, int32_t ldkv, int32_t koff, int32_t voff,
                          const int32_t* off, int32_t B, int32_t rows_per_seg, int32_t H, uint16_t* out_f16);
/* Test hook: teacher-forced logits.  The encoder of wl_mt_translate over B segments, then the decoder (one row per
 * segment) fed prefix [B][P] token by token (position t at step t) -> out_logits [B][P][vocab], the logits after each
 * prefix token. */
int wl_test_mt_logits(wl_mt_ctx* ctx, const int32_t* src_ids, const int32_t* src_off, int32_t B, const int32_t* prefix,
                      int32_t P, float* out_logits);
/* Test hook: wl_mt_translate's search launches on scripted logits [opts->max_length - 1][B * num_beams][V] (step t's
 * logits of row r at [t][r]) in place of the decoder's.  Outputs as wl_mt_translate's; out_steps [B]: the running length
 * (cur_len) at which each segment stopped. */
int wl_test_mt_search(wl_mt_ctx* ctx, const float* logits, int32_t V, int32_t B, const wl_mt_opts* opts, int32_t* out_ids,
                      int32_t* out_len, float* out_score, int32_t* out_steps);

#ifdef __cplusplus
}
#endif
#endif /* WLB200_H */
