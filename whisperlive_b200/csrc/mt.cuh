// Translation (M2M100 / SMaLL-100) kernels of libwlb200 (mt.cu); the context and the C ABI are in mt_engine.cu.
#pragma once
#include "kernels.cuh"

namespace wl {

constexpr int MT_MAX_BEAM = 8;
constexpr int MT_MAX_CAND = 2 * MT_MAX_BEAM;   // Hugging Face keeps the top 2K continuations of a step
constexpr int MT_MAX_SRC = 1024;               // source tokens of one segment (max_position_embeddings - 2 at most)

// Device state of a translate call: rows r = segment * K + beam.
struct MtState {
  // per row
  int* tok_in;       // token the next decoder step feeds
  int* pos;          // its position (tokens already cached); pos + 1 = cur_len of the running sequence
  int* active;
  short* src;        // [R][T_MAX] physical cache row holding position p (beam indirection)
  int* hist;         // [R][T_MAX] running sequence, decoder start token first
  float* run_score;  // cumulative log-probability of the running beam
  float* run_next;
  float* cand_val;   // [R][MT_MAX_CAND] log-probabilities of the row's best continuations
  int* cand_tok;     // [R][MT_MAX_CAND]
  float* fin_score;  // [B][K] finished table, best first (rows indexing: b * K + slot)
  int* fin_flag;
  int* fin_len;      // tokens, decoder start included
  int* fin_tok;      // [B][MT_MAX_BEAM][T_MAX]
  // per segment
  int* done;
  int* unsat;        // Hugging Face's is_early_stop_heuristic_unsatisfied
  int* steps;        // cur_len when the segment stopped
  int* n_done;       // [1]
  int* steps_left;   // [1]
  int forced_bos, forced_eos;   // -1: none
};

struct MtSearch {
  int beam;            // K; 1 = greedy
  int max_length;      // decoder start token included
  float length_penalty;
  int early_stopping;  // 0 False, 1 True, 2 "never"
  int eos;
};

// the view of MtState the shared decoder self-attention kernel reads (active, pos, src; writes to the row itself)
inline DecodeState mt_decode_state(const MtState& s) {
  DecodeState d;
  memset(&d, 0, sizeof(d));
  d.tok_in = s.tok_in;
  d.pos = s.pos;
  d.active = s.active;
  d.src = s.src;
  return d;
}

void mt_enc_embed(cudaStream_t st, const int* tok, const int* tpos, const __half* emb, const float* pos_tab, float scale, float* x,
                  long n, int d);
void mt_dec_embed(cudaStream_t st, const MtState& s, const __half* emb, const float* pos_tab, float scale, int pad, float* x, int R,
                  int d);
// qkv fp16 [n][3d] (q | k | v, heads of 64) -> out fp16 [n][d]; tiles [n_tiles] = (segment, first query) of 64-query tiles
void mt_enc_attn(cudaStream_t st, const __half* qkv, const int* off, const int2* tiles, int n_tiles, __half* out, int H, int d);
// q f32 [R][d] -> out fp16 [R][d] over kv fp16 [n_src][ldkv] (K at column koff, V at voff) of the row's segment
void mt_cross_attn(cudaStream_t st, const MtState& s, const float* q, const __half* kv, long ldkv, int koff, int voff, const int* off,
                   int rows_per_seg, __half* out, int R, int H, int d);
void mt_search_init(cudaStream_t st, const MtState& s, int B, int K, int start, int steps);
// logits f32 [R][ld] (V valid): the per-row candidates, then the per-segment beam step
void mt_search_step(cudaStream_t st, const MtState& s, const MtSearch& o, const float* logits, long ld, int V, int B);
void mt_loop_condition(cudaStream_t st, const MtState& s, cudaGraphConditionalHandle h, int B);

}  // namespace wl
