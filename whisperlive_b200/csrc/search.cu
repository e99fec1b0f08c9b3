// K12: logits processors + log-softmax + candidate selection (search_rows), and the per-stream
// search state machine: prompt feeding, CT2-style beam search, greedy / Gumbel-max sampling
// (search_streams).  Everything stays on the device; the host only polls a finished-stream counter.
// Semantics: oracle/search.py (restated CTranslate2 behaviour; reference call site
// transcriber_faster_whisper.py:1394-1407).
#include "kernels.cuh"

namespace wl {

struct MaskCtx {
  const unsigned* suppress;
  int first, suppress_blank, use_ts, last_is_ts, penult_is_ts, has_ts, ts_cutoff, max_initial;
  int eot, no_timestamps, ts_begin, blank;
};

// The logits rules of stream b: its own (a decode session's state carries them per stream) or the call's.
__device__ __forceinline__ void stream_rules(const DecodeState& s, const SearchOpts& o, int b, MaskCtx& c, int glen) {
  const bool own = s.r_mask != nullptr;
  c.suppress = own ? s.r_mask + (long)b * s.mask_words : o.suppress_mask;
  c.suppress_blank = (own ? s.r_suppress_blank[b] : o.suppress_blank) && glen == 0;
  c.max_initial = own ? s.r_max_initial[b] : o.max_initial_ts;
}

// The beam width of stream b: its own (a decode session's state carries it per stream, <= rows_per_stream) or the call's.
__device__ __forceinline__ int stream_beam(const DecodeState& s, const SearchOpts& o, int b) {
  return s.r_beam ? s.r_beam[b] : o.beam;
}

// the rule-based part of the logits processors (everything but the user's suppress list)
__device__ __forceinline__ bool rule_masked(int t, const MaskCtx& c) {
  if (c.suppress_blank && (t == c.blank || t == c.eot)) return true;
  if (c.use_ts) {
    if (t == c.no_timestamps) return true;
    if (c.first) {
      if (t < c.ts_begin || t > c.ts_begin + c.max_initial) return true;
    } else {
      if (c.last_is_ts) {
        if (c.penult_is_ts) {
          if (t >= c.ts_begin) return true;
        } else if (t < c.eot) {
          return true;
        }
      }
      if (c.has_ts && t >= c.ts_begin && t < c.ts_cutoff) return true;
    }
  }
  return false;
}

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) { m = m2; s = s2; return; }
  if (m2 > m) { s = s * __expf(m - m2) + s2; m = m2; }
  else s += s2 * __expf(m2 - m);
}

constexpr int SR_THREADS = 1024;
constexpr int SR_WARPS = SR_THREADS / 32;

// block-wide (max, sum-of-exp) merge; red holds 2 x SR_WARPS floats
__device__ void block_lse(float& m, float& s, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, m2, s2);
  }
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { red[w] = m; red[SR_WARPS + w] = s; }
  __syncthreads();
  m = red[0]; s = red[SR_WARPS];
  for (int i = 1; i < SR_WARPS; ++i) lse_merge(m, s, red[i], red[SR_WARPS + i]);
  __syncthreads();
}
// block-wide max / sum of two values at once
__device__ void block_max2(float& a, float& b, float* red) {
  a = warp_max(a); b = warp_max(b);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[w] = a; red[SR_WARPS + w] = b; }
  __syncthreads();
  a = warp_max(red[threadIdx.x & 31]); b = warp_max(red[SR_WARPS + (threadIdx.x & 31)]);
  __syncthreads();
}
__device__ void block_sum2(float& a, float& b, float* red) {
  a = warp_sum(a); b = warp_sum(b);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[w] = a; red[SR_WARPS + w] = b; }
  __syncthreads();
  // fixed order: every thread adds the 32 warp sums in the same sequence
  float x = 0.f, y = 0.f;
#pragma unroll
  for (int i = 0; i < SR_WARPS; ++i) { x += red[i]; y += red[SR_WARPS + i]; }
  a = x; b = y;
  __syncthreads();
}

// One 1024-thread CTA per decoder row.  The row of logits (<= 53248 floats, 207 KB for the 51866-token vocabulary)
// is read from HBM/L2 exactly once: it is masked on the way in (suppress list + timestamp rules -> -inf) and kept in
// shared memory; the softmax statistics, the key computation and the candidate rounds all run on the resident copy.
// Candidates: each thread remembers the best of its own 4-token groups; a round is one block arg-max over those
// (ties -> lower token id) after which only the winning thread looks for its next-best entry.
__global__ void __launch_bounds__(SR_THREADS) search_rows_kernel(DecodeState s, const float* __restrict__ logits, SearchOpts o,
                                                                 VocabIds v) {
  extern __shared__ float4 sr_smem[];   // [n4] masked logits, later selection keys
  const int r = blockIdx.x, tid = threadIdx.x;
  const int b = r / o.rows_per_stream;
  pdl_trigger();
  tl_stamp(TL_SROWS, 0);
  if (!s.active[r] || s.done[b]) return;   // per-step state, complete before this step started
  __shared__ float red[2 * SR_WARPS];
  __shared__ float wkey[SR_WARPS];
  __shared__ int wtok[SR_WARPS], wtid[SR_WARPS];
  __shared__ int win_tid;

  const float* lg = logits + (long)r * v.vocab_ld;
  const int fed = s.fed[b], P = s.prompt_len[b];
  pdl_wait();   // logits come from the vocabulary GEMM right before this kernel
  tl_stamp(TL_SROWS, 1);
  if (fed == s.sot_index[b] && r == b * o.rows_per_stream) {
    float m = -INFINITY, sm = 0.f;
    for (int t = tid; t < v.vocab; t += SR_THREADS) lse_merge(m, sm, lg[t], 1.f);
    block_lse(m, sm, red);
    if (tid == 0) s.nospeech_row[r] = __expf(lg[v.no_speech] - m) / sm;
  }
  if (s.force_len[b] > 0) {
    // teacher-forced pass: probability of the NEXT forced token under the raw distribution (K14 text_token_probs)
    if (fed + 1 < P && r == b * o.rows_per_stream) {
      float m = -INFINITY, sm = 0.f;
      for (int t = tid; t < v.vocab; t += SR_THREADS) lse_merge(m, sm, lg[t], 1.f);
      block_lse(m, sm, red);
      if (tid == 0) s.force_prob[(long)b * T_MAX + fed] = __expf(lg[s.prompt[(long)b * T_MAX + fed + 1]] - m) / sm;
    }
    return;
  }
  if (fed < P - 1) return;

  const int glen = s.gen_len[r];
  const int* hist = s.hist + (long)r * T_MAX;
  // CTranslate2 ends the "prompt" at the sot sequence (sot, language, task, notimestamps): whatever follows -- the
  // ``prefix`` of transcriber_faster_whisper.py:1505-1511, incl. its leading <|0.00|> -- counts as sampled text for the
  // timestamp rules.  Blank suppression is keyed to the first GENERATED step.
  const int npre = s.pre_n[b], nhist = glen + npre;
  MaskCtx c;
  stream_rules(s, o, b, c, glen);
  c.first = nhist == 0;
  c.use_ts = s.use_ts[b];
  c.eot = v.eot; c.no_timestamps = v.no_timestamps; c.ts_begin = v.ts_begin; c.blank = v.blank;
  const int last = glen > 0 ? hist[glen - 1] : s.pre_last[b];
  const int penult = glen > 1 ? hist[glen - 2] : (glen == 1 ? s.pre_last[b] : s.pre_penult[b]);
  c.last_is_ts = nhist > 0 && last >= v.ts_begin;
  c.penult_is_ts = nhist < 2 || penult >= v.ts_begin;
  const int lts = s.last_ts[r];
  c.has_ts = lts >= 0;
  c.ts_cutoff = (c.last_is_ts && !c.penult_is_ts) ? lts : lts + 1;

  // load + mask (processors a-d) -> shared memory; thread-local maxima of the text and the timestamp part
  const float4* lg4 = reinterpret_cast<const float4*>(lg);
  const int n4 = v.vocab_ld >> 2;
  float mt = -INFINITY, mz = -INFINITY;
  for (int i4 = tid; i4 < n4; i4 += SR_THREADS) {
    const int t = 4 * i4;
    const float4 q = lg4[i4];
    const unsigned bits = t < v.vocab ? (c.suppress[t >> 5] >> (t & 31)) : 0xFu;   // 4 | 32: the 4 tokens share a word
    float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const bool masked = t + e >= v.vocab || ((bits >> e) & 1u) || rule_masked(t + e, c);
      x[e] = masked ? -INFINITY : x[e];
      if (t + e < v.ts_begin) mt = fmaxf(mt, x[e]);
      else mz = fmaxf(mz, x[e]);
    }
    sr_smem[i4] = make_float4(x[0], x[1], x[2], x[3]);
  }
  block_max2(mt, mz, red);
  // softmax statistics of the two parts (exp of -inf is 0: masked entries drop out)
  float st = 0.f, sz = 0.f;
  {
    const float mt0 = mt == -INFINITY ? 0.f : mt, mz0 = mz == -INFINITY ? 0.f : mz;
    for (int i4 = tid; i4 < n4; i4 += SR_THREADS) {
      const int t = 4 * i4;
      const float4 q = sr_smem[i4];
      const float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (t + e < v.ts_begin) st += __expf(x[e] - mt0);
        else sz += __expf(x[e] - mz0);
      }
    }
  }
  block_sum2(st, sz, red);
  const float lse_text = st > 0.f ? mt + logf(st) : -INFINITY;
  const float lse_ts = sz > 0.f ? mz + logf(sz) : -INFINITY;
  const bool text_off = c.use_ts && !c.first && lse_ts > mt;  // rule e: mass on timestamps beats the best text token
  float lse;
  if (text_off || lse_text == -INFINITY) lse = lse_ts;
  else if (lse_ts == -INFINITY) lse = lse_text;
  else {
    const float hi = fmaxf(lse_text, lse_ts), lo = fminf(lse_text, lse_ts);
    lse = hi + log1pf(expf(lo - hi));
  }

  // selection keys in place: log-prob (beam / greedy) or log-prob / T + Gumbel noise (sampling); rule e drops text.
  // The noise of row j of a sampling stream is keyed by (seed, noise key, j, step) -- wl_generate: key = batch position.
  // Only the stream's own 2 K_b candidates: the rounds are sequential, so they are the first 2 K_b entries of the list
  // the session's width would give, and a narrower stream's row runs fewer rounds instead of the session's 2 K.
  const bool sampling = s.smode[b] != 0;
  const int K = stream_beam(s, o, b);
  const int NC = (!sampling && K > 1) ? 2 * K : 1;
  const float temperature = s.temp[b];
  uint32_t gkey = 0;
  if (sampling)
    gkey = hash_u32((s.nseed[b] * 0x9E3779B1u) ^ hash_u32((uint32_t)((s.nkey[b] * 64 + (r - b * o.rows_per_stream)) * 65537 + s.step[b])));
  float bk = -INFINITY;        // this thread's best remaining entry
  int bt = 0x7fffffff;
  for (int i4 = tid; i4 < n4; i4 += SR_THREADS) {
    const int t = 4 * i4;
    const float4 q = sr_smem[i4];
    float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float key = -INFINITY;
      if (x[e] > -INFINITY && !(text_off && t + e < v.ts_begin)) {
        const float lp = x[e] - lse;
        key = lp;
        if (sampling) {
          const double u = ((double)hash_u32((uint32_t)(t + e) ^ gkey) + 0.5) / 4294967296.0;
          key = __fdiv_rn(lp, temperature) + (float)(-log(-log(u)));
        }
        if (key > bk) { bk = key; bt = t + e; }   // ascending token order: strict > keeps the lowest id among equals
      }
      x[e] = key;
    }
    sr_smem[i4] = make_float4(x[0], x[1], x[2], x[3]);
  }
  const float* keys = reinterpret_cast<const float*>(sr_smem);
  for (int round = 0; round < NC; ++round) {
    float k = bk;
    int t = bt, who = tid;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float k2 = __shfl_xor_sync(0xffffffffu, k, off);
      const int t2 = __shfl_xor_sync(0xffffffffu, t, off), w2 = __shfl_xor_sync(0xffffffffu, who, off);
      if (k2 > k || (k2 == k && t2 < t)) { k = k2; t = t2; who = w2; }
    }
    if ((tid & 31) == 0) { wkey[tid >> 5] = k; wtok[tid >> 5] = t; wtid[tid >> 5] = who; }
    __syncthreads();
    if (tid < 32) {
      k = wkey[tid]; t = wtok[tid]; who = wtid[tid];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float k2 = __shfl_xor_sync(0xffffffffu, k, off);
        const int t2 = __shfl_xor_sync(0xffffffffu, t, off), w2 = __shfl_xor_sync(0xffffffffu, who, off);
        if (k2 > k || (k2 == k && t2 < t)) { k = k2; t = t2; who = w2; }
      }
      if (tid == 0) {
        const bool none = t == 0x7fffffff;
        win_tid = none ? -1 : who;
        s.cand_val[(long)r * MAX_CAND + round] = none ? -INFINITY : lg[t] - lse;
        s.cand_tok[(long)r * MAX_CAND + round] = none ? -1 : t;
      }
    }
    __syncthreads();
    if (tid == win_tid) {
      // next-best entry of this thread: strictly after (bk, bt) in (key descending, token ascending) order
      const float pk = bk;
      const int pt = bt;
      bk = -INFINITY; bt = 0x7fffffff;
      for (int i4 = tid; i4 < n4; i4 += SR_THREADS) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int tt = 4 * i4 + e;
          const float key = keys[tt];
          if (key > -INFINITY && (key < pk || (key == pk && tt > pt)) && key > bk) { bk = key; bt = tt; }
        }
      }
    }
  }
}

void search_rows(cudaStream_t st, const DecodeState& s, const float* logits, const SearchOpts& o, const VocabIds& v, int R) {
  const size_t smem = (size_t)(v.vocab_ld >> 2) * sizeof(float4);
  WL_CHECK(v.vocab_ld % 4 == 0 && smem <= 216 * 1024, WL_ERR_ARG, "search_rows: vocabulary row of %d floats does not fit in shared memory", v.vocab_ld);
  launch_kernel(search_rows_kernel, dim3(R), dim3(SR_THREADS), smem, st, s, logits, o, v);
  note_launch(1);
}

void search_tl_bind(unsigned long long* p) { tl_bind_tu(p); }
void search_prime() {
  WL_CUDA(cudaFuncSetAttribute(search_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
}

// ============================================================================ per-stream state machine
__device__ void finish_stream(DecodeState& s, int b, int Kr) {
  s.done[b] = 1;
  for (int j = 0; j < Kr; ++j) s.active[b * Kr + j] = 0;
  atomicAdd(s.n_done, 1);
}

__global__ void __launch_bounds__(128) search_streams_kernel(DecodeState s, SearchOpts o, VocabIds v) {
  const int b = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  tl_stamp(TL_SSTREAMS, 0);
  pdl_wait();
  tl_stamp(TL_SSTREAMS, 1);
  if (s.done[b]) return;
  const int Kr = o.rows_per_stream, row0 = b * Kr;
  const int P = s.prompt_len[b], fed = s.fed[b];
  // greedy / sampling: every row is an independent hypothesis, over the stream's own N <= Kr rows (a sampling or
  // width-1 stream of a beam session included); otherwise a beam of the stream's own width K <= Kr
  const int K = stream_beam(s, o, b);
  const bool independent = K == 1 || s.smode[b] != 0;
  const int N = s.nrows[b];
  __shared__ int sh_hist[MAX_ROWS_PER_STREAM][T_MAX];
  __shared__ short sh_src[MAX_ROWS_PER_STREAM][T_MAX];
  __shared__ int new_parent[MAX_ROWS_PER_STREAM], new_tok[MAX_ROWS_PER_STREAM];
  __shared__ float new_cum[MAX_ROWS_PER_STREAM];
  __shared__ int hyp_parent[MAX_ROWS_PER_STREAM], hyp_extra[MAX_ROWS_PER_STREAM], hyp_slot[MAX_ROWS_PER_STREAM];
  __shared__ int n_newalive, n_newhyp, finished;

  if (tid == 0) {
    s.steps_run[b] += 1;
    // the probability at the sot position: when sot is the last prompt token, fed stays there for the whole search and
    // only the first decode step's row is that position
    if (fed == s.sot_index[b] && (fed < P - 1 || s.step[b] == 0)) s.no_speech[b] = s.nospeech_row[row0];
  }
  // ---- teacher-forced feeding only (detect_language / align / logits hook)
  if (s.force_len[b] > 0) {
    if (tid == 0) {
      if (fed + 1 < P) {
        s.tok_in[row0] = s.prompt[(long)b * T_MAX + fed + 1];
        s.pos[row0] = fed + 1;
        s.fed[b] = fed + 1;
      } else {
        finish_stream(s, b, Kr);
      }
    }
    return;
  }
  // ---- prompt feeding
  if (fed < P - 1) {
    const int nf = fed + 1;
    if (tid == 0) {
      s.tok_in[row0] = s.prompt[(long)b * T_MAX + nf];
      s.pos[row0] = nf;
      s.fed[b] = nf;
    }
    if (nf == P - 1 && independent && N > 1) {
      // independent sampling rows all start from the prompt cache of row 0
      for (int j = 1; j < N; ++j) {
        for (int p = tid; p < nf; p += 128) s.src[(long)(row0 + j) * T_MAX + p] = s.src[(long)row0 * T_MAX + p];
        if (tid == 0) {
          s.tok_in[row0 + j] = s.prompt[(long)b * T_MAX + nf];
          s.pos[row0 + j] = nf;
          s.active[row0 + j] = 1;
        }
      }
    }
    return;
  }
  const int step = s.step[b];
  const bool last_step = step + 1 >= s.n_new[b];

  // ---- greedy / sampling: every row is an independent hypothesis
  if (independent) {
    if (tid < N && !s.row_done[row0 + tid]) {
      const int r = row0 + tid;
      const int tok = s.cand_tok[(long)r * MAX_CAND];
      const float val = s.cand_val[(long)r * MAX_CAND];
      int len = s.gen_len[r];
      bool fin = false;
      if (tok < 0) fin = true;
      else {
        s.cum[r] += val;
        if (tok == v.eot) fin = true;
        else {
          s.hist[(long)r * T_MAX + len] = tok;
          s.gen_len[r] = ++len;
          if (tok >= v.ts_begin) s.last_ts[r] = tok;
          if (last_step) fin = true;
        }
      }
      if (fin) { s.row_done[r] = 1; s.active[r] = 0; }
      else { s.tok_in[r] = tok; s.pos[r] += 1; }
    }
    __syncthreads();
    if (tid == 0) {
      s.step[b] = step + 1;
      bool all = true;
      for (int j = 0; j < N; ++j) all = all && s.row_done[row0 + j];
      finished = all ? 1 : 0;
      if (all) {
        s.hyp_count[b] = N;
        for (int j = 0; j < N; ++j) {
          s.hyp_cum[b * MAX_HYPS + j] = s.cum[row0 + j];
          s.hyp_len[b * MAX_HYPS + j] = s.gen_len[row0 + j];
        }
        finish_stream(s, b, Kr);
      }
    }
    __syncthreads();
    if (finished) {
      for (int j = 0; j < N; ++j)
        for (int p = tid; p < s.gen_len[row0 + j]; p += 128)
          s.hyp_tok[((long)b * MAX_HYPS + j) * T_MAX + p] = s.hist[(long)(row0 + j) * T_MAX + p];
    }
    return;
  }

  // ---- beam search (CT2 walk, see oracle/search.py) over rows 0 .. K-1; rows K .. Kr-1 stay inactive
  const int n_alive = s.n_alive[b];
  const int pos_old = s.pos[row0];
  const int len_old = s.gen_len[row0];
  for (int j = 0; j < n_alive; ++j) {
    for (int p = tid; p < len_old; p += 128) sh_hist[j][p] = s.hist[(long)(row0 + j) * T_MAX + p];
    for (int p = tid; p <= pos_old; p += 128) sh_src[j][p] = s.src[(long)(row0 + j) * T_MAX + p];
  }
  // candidate lists and cumulative scores of the alive rows -> shared memory with one parallel load: the merge below is
  // one thread walking <= 8 x 16 entries, which as a chain of dependent global loads would sit on the token step's
  // critical path
  __shared__ float sh_cval[MAX_ROWS_PER_STREAM][MAX_CAND];
  __shared__ int sh_ctok[MAX_ROWS_PER_STREAM][MAX_CAND];
  __shared__ float sh_cum[MAX_ROWS_PER_STREAM];
  for (int i = tid; i < n_alive * MAX_CAND; i += 128) {
    const int j = i / MAX_CAND, k = i % MAX_CAND;
    sh_cval[j][k] = s.cand_val[(long)(row0 + j) * MAX_CAND + k];
    sh_ctok[j][k] = s.cand_tok[(long)(row0 + j) * MAX_CAND + k];
  }
  if (tid < n_alive) sh_cum[tid] = s.cum[row0 + tid];
  __syncthreads();
  if (tid == 0) {
    // merged top-2K over the alive rows (each row's list is sorted): (total desc, row asc, list order)
    int idx[MAX_ROWS_PER_STREAM];
    for (int j = 0; j < MAX_ROWS_PER_STREAM; ++j) idx[j] = 0;
    int cb[MAX_CAND], ct[MAX_CAND];
    float cs[MAX_CAND];
    int nc = 0;
    const int NC = 2 * K;
    for (int k = 0; k < NC; ++k) {
      int bj = -1;
      float bs = -INFINITY;
      for (int j = 0; j < n_alive; ++j) {
        if (idx[j] >= NC) continue;
        const float cv = sh_cval[j][idx[j]];
        if (cv == -INFINITY) continue;
        const float tot = sh_cum[j] + cv;
        if (tot > bs) { bs = tot; bj = j; }
      }
      if (bj < 0) break;
      cb[nc] = bj; ct[nc] = sh_ctok[bj][idx[bj]]; cs[nc] = bs;
      ++idx[bj]; ++nc;
    }
    int na = 0, nh = 0, hc = s.hyp_count[b];
    int secondary = K;
    for (int k = 0; k < K && k < nc; ++k) {
      int beam = cb[k], tok = ct[k];
      float sc = cs[k];
      if (tok == v.eot || last_step) {
        if (hc + nh < MAX_HYPS) {
          hyp_parent[nh] = beam;
          hyp_extra[nh] = tok == v.eot ? -1 : tok;
          hyp_slot[nh] = hc + nh;
          s.hyp_cum[b * MAX_HYPS + hc + nh] = sc;
          s.hyp_len[b * MAX_HYPS + hc + nh] = len_old + (tok == v.eot ? 0 : 1);
          ++nh;
        }
        if (last_step) continue;
        bool found = false;
        while (secondary < nc) {
          const int b2 = cb[secondary], t2 = ct[secondary];
          const float s2 = cs[secondary];
          ++secondary;
          if (t2 != v.eot) { beam = b2; tok = t2; sc = s2; found = true; break; }
        }
        if (!found) continue;
      }
      new_parent[na] = beam; new_tok[na] = tok; new_cum[na] = sc;
      ++na;
    }
    s.hyp_count[b] = hc + nh;
    s.step[b] = step + 1;
    n_newalive = na; n_newhyp = nh;
    const int max_cand = s.r_max_cand ? s.r_max_cand[b] : o.max_cand;
    finished = (hc + nh >= max_cand || last_step || na == 0) ? 1 : 0;
  }
  __syncthreads();
  for (int i = 0; i < n_newhyp; ++i) {
    int* dst = s.hyp_tok + ((long)b * MAX_HYPS + hyp_slot[i]) * T_MAX;
    for (int p = tid; p < len_old; p += 128) dst[p] = sh_hist[hyp_parent[i]][p];
    if (tid == 0 && hyp_extra[i] >= 0) dst[len_old] = hyp_extra[i];
  }
  if (finished) {
    if (tid == 0) finish_stream(s, b, Kr);
    return;
  }
  for (int j = 0; j < n_newalive; ++j) {
    const int r = row0 + j, pj = new_parent[j];
    for (int p = tid; p < len_old; p += 128) s.hist[(long)r * T_MAX + p] = sh_hist[pj][p];
    for (int p = tid; p <= pos_old; p += 128) s.src[(long)r * T_MAX + p] = sh_src[pj][p];
  }
  __syncthreads();
  if (tid < Kr) {
    const int r = row0 + tid;
    if (tid < n_newalive) {
      const int tok = new_tok[tid];
      const int plts = s.last_ts[row0 + new_parent[tid]];
      s.hist[(long)r * T_MAX + len_old] = tok;
      s.gen_len[r] = len_old + 1;
      s.cum[r] = new_cum[tid];
      s.tok_in[r] = tok;
      s.pos[r] = pos_old + 1;
      s.active[r] = 1;
      // last_ts of the parent must be read before any row overwrites it: stage through registers + barrier
      new_tok[tid] = tok >= v.ts_begin ? tok : plts;
    } else {
      s.active[r] = 0;
    }
  }
  __syncthreads();
  if (tid < n_newalive) s.last_ts[row0 + tid] = new_tok[tid];
  if (tid == 0) s.n_alive[b] = n_newalive;
}

void search_streams(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, int B) {
  launch_kernel(search_streams_kernel, dim3(B), dim3(128), 0, st, s, o, v);
  note_launch(1);
}

// ============================================================================ scripted logits (wl_test_search only)
// A row's logits are a pure function of the tokens it has consumed: prompt[0 .. fed] while the prompt is fed, then the
// whole prompt and the row's generated tokens.  Every value is an exact fp32 number (a multiple of 2^-11), so
// tests/search_script.py reproduces them bit for bit.  h = lowbias32(FNV-1a(seed, tokens)) picks, per step:
//   base(t)   = ((lowbias32(h ^ t * 0x9E3779B1) >> 20) - 2048) / 256, a 1/256 grid over [-8, 8)
//   + a timestamp bias and an EOT bias from 4-entry tables (bits 0-1 / 2-3), + 10 on no_speech after sot (bit 4);
//   a pattern (SearchScript::pattern, or bits 5.. of h when it is -1) that puts the top candidates where the selection
//   code is fragile; and, on a row that searches, 60 + base / 8 on every token some rule must mask at this step, so a
//   missed mask changes the arg-max.
__constant__ float SCRIPT_TS_BIAS[4] = {-8.f, -5.f, -2.f, 2.f};
__constant__ float SCRIPT_EOT_BIAS[4] = {-8.f, -2.f, 2.f, 8.f};

struct ScriptRow {
  uint32_t h, g;
  int pattern, after_sot, search;
  MaskCtx c;   // the rules of this step (search != 0)
};

// h of the first n tokens of `prompt` followed by the first glen of `gen`
__device__ uint32_t script_hash(uint32_t seed, const int* prompt, int n, const int* gen, int glen) {
  uint32_t h = (2166136261u ^ seed) * 16777619u;
  for (int i = 0; i < n; ++i) h = (h ^ (uint32_t)prompt[i]) * 16777619u;
  for (int i = 0; i < glen; ++i) h = (h ^ (uint32_t)gen[i]) * 16777619u;
  return hash_u32(h);
}

__device__ void script_row_setup(ScriptRow& w, uint32_t h, int last, const SearchScript& sc) {
  w.h = h;
  w.g = hash_u32(h ^ 0x5BD1E995u);
  w.pattern = sc.pattern >= 0 ? sc.pattern : (int)((h >> 5) % 6u);
  w.after_sot = last;
}

__device__ __forceinline__ float script_quarter(float x) { return floorf(x * 4.f) * 0.25f; }

__device__ float script_logit(int t, const ScriptRow& w, const VocabIds& v) {
  const float base = (float)((int)(hash_u32(w.h ^ ((uint32_t)t * 0x9E3779B1u)) >> 20) - 2048) * (1.f / 256.f);
  if (w.search) {
    const bool sup = (w.c.suppress[t >> 5] >> (t & 31)) & 1u;
    const bool ts_masked = w.c.use_ts && t >= v.ts_begin &&
                           (w.c.first ? t > v.ts_begin + w.c.max_initial : (w.c.has_ts && t < w.c.ts_cutoff));
    if (sup || ts_masked || (w.c.use_ts && t == v.no_timestamps) || (w.c.suppress_blank && (t == v.blank || t == v.eot)))
      return 60.f + base * 0.125f;
  }
  float x = base;
  if (t >= v.ts_begin) x += SCRIPT_TS_BIAS[w.h & 3u];
  else if (t == v.eot) x += SCRIPT_EOT_BIAS[(w.h >> 2) & 3u];
  else if (t == v.no_speech && w.after_sot && ((w.h >> 4) & 1u)) x += 10.f;
  switch (w.pattern) {
    case 1: if (((t % 4096) >> 2) == (int)(w.g % 1024u)) x = 8.f + script_quarter(base); break;
    case 2: if ((t >> 2) == (int)(w.g % (uint32_t)(v.vocab >> 2))) x = 8.f + script_quarter(base); break;
    case 3: if (t >= v.vocab - 8) x = 8.f + script_quarter(base); break;
    case 4: x = script_quarter(x); break;
    case 5: {
      const int d = (int)(w.g % (uint32_t)v.eot), d2 = (d + 1 + (int)((w.g >> 24) & 63u)) % v.eot;
      if (t == d || (((w.h >> 7) & 1u) && t == d2)) x = 48.f;
      break;
    }
    default: break;
  }
  return x;
}

__global__ void __launch_bounds__(256) scripted_logits_kernel(DecodeState s, SearchOpts o, VocabIds v, SearchScript sc,
                                                              float* __restrict__ logits) {
  const int r = blockIdx.x, b = r / o.rows_per_stream, tid = threadIdx.x;
  float* out = logits + (long)r * v.vocab_ld;
  __shared__ ScriptRow w;
  // wait first: the state comes from the previous step's search_streams, and search_rows (launched as soon as every
  // CTA here has triggered) reads its per-step flags before its own wait
  pdl_wait();
  pdl_trigger();
  if (!s.active[r] || s.done[b]) {
    for (int t = tid; t < v.vocab_ld; t += blockDim.x) out[t] = __int_as_float(0x7fc00000);
    return;
  }
  if (tid == 0) {
    const int fed = s.fed[b], P = s.prompt_len[b];
    const int* prompt = s.prompt + (long)b * T_MAX;
    const int glen = fed >= P - 1 ? s.gen_len[r] : 0;
    const int* hist = s.hist + (long)r * T_MAX;
    const int last = glen > 0 ? hist[glen - 1] : prompt[fed];
    script_row_setup(w, script_hash(sc.seed, prompt, fed + 1, hist, glen), last == v.sot, sc);
    w.search = fed >= P - 1;
    // the rules of search_rows_kernel for this row
    MaskCtx& c = w.c;
    const int npre = s.pre_n[b], nhist = glen + npre;
    stream_rules(s, o, b, c, glen);
    c.first = nhist == 0;
    c.use_ts = s.use_ts[b];
    const int penult = glen > 1 ? hist[glen - 2] : (glen == 1 ? s.pre_last[b] : s.pre_penult[b]);
    const int plast = glen > 0 ? last : s.pre_last[b];
    c.last_is_ts = nhist > 0 && plast >= v.ts_begin;
    c.penult_is_ts = nhist < 2 || penult >= v.ts_begin;
    const int lts = s.last_ts[r];
    c.has_ts = lts >= 0;
    c.ts_cutoff = (c.last_is_ts && !c.penult_is_ts) ? lts : lts + 1;
  }
  __syncthreads();
  for (int t = tid; t < v.vocab_ld; t += blockDim.x) out[t] = t < v.vocab ? script_logit(t, w, v) : __int_as_float(0x7fc00000);
}

void scripted_logits(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, const SearchScript& sc,
                     float* logits, int R) {
  launch_kernel(scripted_logits_kernel, dim3(R), dim3(256), 0, st, s, o, v, sc, logits);
  note_launch(1);
}

__global__ void __launch_bounds__(256) scripted_no_speech_kernel(DecodeState s, VocabIds v, SearchScript sc,
                                                                 const int* __restrict__ index) {
  const int b = index ? index[blockIdx.x] : blockIdx.x, tid = threadIdx.x;
  const int sot = s.sot_index[b];
  if (sot < 0 || sot >= s.prompt_len[b] - 1) {
    if (index && tid == 0) s.no_speech[b] = 0.f;   // a session index: clear what its previous stream left
    return;
  }
  __shared__ ScriptRow w;
  __shared__ float red[2 * 8];
  if (tid == 0) {
    script_row_setup(w, script_hash(sc.seed, s.prompt + (long)b * T_MAX, sot + 1, nullptr, 0), 1, sc);
    w.search = 0;
  }
  __syncthreads();
  float m = -INFINITY, sm = 0.f;
  for (int t = tid; t < v.vocab; t += blockDim.x) lse_merge(m, sm, script_logit(t, w, v), 1.f);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) lse_merge(m, sm, __shfl_xor_sync(0xffffffffu, m, off), __shfl_xor_sync(0xffffffffu, sm, off));
  if ((tid & 31) == 0) { red[tid >> 5] = m; red[8 + (tid >> 5)] = sm; }
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i < 8; ++i) lse_merge(m, sm, red[i], red[8 + i]);
    s.no_speech[b] = __expf(script_logit(v.no_speech, w, v) - m) / sm;
  }
}

void scripted_no_speech(cudaStream_t st, const DecodeState& s, const VocabIds& v, const SearchScript& sc, int B,
                        const int* index) {
  scripted_no_speech_kernel<<<B, 256, 0, st>>>(s, v, sc, index);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ============================================================================ device-terminated decode loop
__global__ void loop_condition_kernel(DecodeState s, cudaGraphConditionalHandle h, int B) {
  pdl_trigger();
  pdl_wait();
  if (threadIdx.x == 0) {
    const int left = *s.steps_left - 1, nd = *s.n_done;
    *s.steps_left = left;
    bool go = left > 0 && nd < B;
    if (s.brk[0] != 0 && nd > s.brk[1]) go = false;   // decode session: a stream finished in this step -> back to the host
    cudaGraphSetConditional(h, go ? 1u : 0u);
  }
}
void loop_condition(cudaStream_t st, const DecodeState& s, cudaGraphConditionalHandle h, int B) {
  PdlScope no_pdl(false);   // a full dependency: every search_streams block has updated n_done
  launch_kernel(loop_condition_kernel, dim3(1), dim3(32), 0, st, s, h, B);
  note_launch(1);
}

// ============================================================================ init
__global__ void decode_init_kernel(DecodeState s, SearchOpts o, VocabIds v, int prefilled, const int* __restrict__ index) {
  const int b = index ? index[blockIdx.x] : blockIdx.x, tid = threadIdx.x;
  const int Kr = o.rows_per_stream, row0 = b * Kr;
  const int P = s.prompt_len[b];
  // token-by-token feeding starts at prompt position 0; after the batched prefill (positions 0 .. P-2 cached in the
  // stream's first row) the first decode step feeds the LAST prompt token
  const int fed0 = (prefilled && s.force_len[b] == 0) ? P - 1 : 0;
  // independent sampling rows all continue from the prompt cache of row 0 (what search_streams does when the feeding
  // reaches the last prompt token); a stream that uses N < Kr rows leaves rows N .. Kr-1 inactive for its whole life
  const bool fan_out = (stream_beam(s, o, b) == 1 || s.smode[b] != 0) && s.force_len[b] == 0 && fed0 == P - 1;
  const int N = fan_out ? s.nrows[b] : 1;
  if (tid < Kr) {
    const int r = row0 + tid;
    const bool on = tid < N;
    s.tok_in[r] = s.prompt[(long)b * T_MAX + fed0];
    s.pos[r] = fed0;
    s.active[r] = on ? 1 : 0;
    s.cum[r] = 0.f;
    s.gen_len[r] = 0;
    s.last_ts[r] = s.pre_lts[b];
    s.row_done[r] = 0;
    s.nospeech_row[r] = 0.f;
  }
  for (int j = 0; j < N; ++j)
    for (int p = tid; p < fed0; p += blockDim.x) s.src[(long)(row0 + j) * T_MAX + p] = (short)row0;
  if (tid == 0) {
    s.fed[b] = fed0;
    s.step[b] = 0;
    s.done[b] = 0;
    s.n_alive[b] = 1;
    if (!prefilled) s.no_speech[b] = 0.f;   // the prefill pass zeroes it and, with sot inside the prompt, has already written it
    s.hyp_count[b] = 0;
    s.steps_run[b] = fed0;
    if (index) atomicSub(s.n_done, 1);   // session admission: the index was idle (done = 1, counted)
    else if (b == 0) *s.n_done = 0;
  }
}

void decode_init(cudaStream_t st, const DecodeState& s, const SearchOpts& o, const VocabIds& v, int B, int R, int prefilled,
                 const int* index) {
  decode_init_kernel<<<B, 32, 0, st>>>(s, o, v, prefilled, index);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ============================================================================ decode sessions between two runs
// One block per listed stream index.  A stream still decoding reports its leading row: row 0 (beam search keeps the best
// live beam there; greedy), or for a sampling stream the alive row with the highest cum (lowest row on ties).  A finished
// stream reports the hypothesis wl_session_collect would put first: the best cum / len^length_penalty, lowest slot on
// ties (emit_hyps' stable sort), and its whole hypothesis table, so the host can rank it with the host's own powf (the
// device's may differ in the last bit for a penalty other than 0 or 1).  The penalty is the stream's own when the state
// carries per-stream rules.  Reads the decode state only.
__global__ void __launch_bounds__(128) session_peek_kernel(DecodeState s, SearchOpts o, float session_length_penalty,
                                                           const int* __restrict__ index, int* __restrict__ out) {
  const int b = index[blockIdx.x], tid = threadIdx.x;
  const int Kr = o.rows_per_stream, row0 = b * Kr;
  int* dst = out + (long)blockIdx.x * PEEK_STRIDE;
  __shared__ const int* sh_tok;
  __shared__ int sh_len;
  if (tid == 0) {
    const int fin = s.done[b];
    int len;
    float cum;
    const int* tok;
    if (fin) {
      const float length_penalty = s.r_length_penalty ? s.r_length_penalty[b] : session_length_penalty;
      const int cnt = min(s.hyp_count[b], MAX_HYPS);
      int best = -1;
      float bs = 0.f;
      for (int i = 0; i < cnt; ++i) {
        const float c = s.hyp_cum[b * MAX_HYPS + i];
        const int hl = s.hyp_len[b * MAX_HYPS + i];
        const float l = (float)max(hl, 1);
        // the host's powf(l, 1) is exactly l: divide directly so the default penalty ranks exactly like emit_hyps
        const float sc = length_penalty == 0.f ? c : (length_penalty == 1.f ? c / l : c / powf(l, length_penalty));
        if (best < 0 || sc > bs) { best = i; bs = sc; }
        dst[PEEK_TAB + i] = hl;
        dst[PEEK_TAB + MAX_HYPS + i] = __float_as_int(c);
      }
      dst[5] = best;
      dst[6] = cnt;
      len = best < 0 ? -1 : s.hyp_len[b * MAX_HYPS + best];
      cum = best < 0 ? 0.f : s.hyp_cum[b * MAX_HYPS + best];
      tok = s.hyp_tok + ((long)b * MAX_HYPS + max(best, 0)) * T_MAX;
    } else {
      int r = row0;
      if (s.smode[b] != 0)
        for (int j = 1; j < s.nrows[b]; ++j) {
          const int q = row0 + j;
          if (!s.row_done[q] && (s.row_done[r] || s.cum[q] > s.cum[r])) r = q;
        }
      len = s.gen_len[r];
      cum = s.cum[r];
      tok = s.hist + (long)r * T_MAX;
    }
    dst[0] = len;
    dst[1] = __float_as_int(cum);
    dst[2] = __float_as_int(s.no_speech[b]);
    dst[3] = s.step[b];
    dst[4] = fin;
    sh_tok = tok;
    sh_len = len;
  }
  __syncthreads();
  for (int p = tid; p < sh_len; p += blockDim.x) dst[PEEK_HDR + p] = sh_tok[p];
}

void session_peek(cudaStream_t st, const DecodeState& s, const SearchOpts& o, float length_penalty, const int* index, int* out,
                  int n) {
  session_peek_kernel<<<n, 128, 0, st>>>(s, o, length_penalty, index, out);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// The listed indices go idle: done, rows inactive.  A stream still decoding is counted into n_done here, the way
// finish_stream counts a stream that ends (decode_init's admission takes it out again); a finished one already is.
__global__ void session_cancel_kernel(DecodeState s, int Kr, const int* __restrict__ index) {
  const int b = index[blockIdx.x], j = threadIdx.x;
  if (j < Kr) s.active[b * Kr + j] = 0;
  if (j == 0 && !s.done[b]) {
    s.done[b] = 1;
    atomicAdd(s.n_done, 1);
  }
}

void session_cancel(cudaStream_t st, const DecodeState& s, int Kr, const int* index, int n) {
  session_cancel_kernel<<<n, 32, 0, st>>>(s, Kr, index);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

}  // namespace wl
