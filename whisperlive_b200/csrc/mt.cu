// Translation kernels (M2M100 / SMaLL-100, sm_90a): embeddings, the ragged encoder self-attention on the tensor cores,
// the ragged decoder cross-attention and Hugging Face's beam-search step.  All segments of a call share one packed
// token axis (src_off [B + 1]); nothing a CTA reads or writes belongs to another segment, so a segment's result does not
// depend on which segments share the call.
#include <mma.h>

#include "mt.cuh"

namespace wl {

// ============================================================================ embeddings
// x[i] = E[tok[i]] * scale + P[tpos[i]]  (fp32), tpos = the sinusoidal row (position + 2, or the zero pad row)
__global__ void mt_enc_embed_kernel(const int* __restrict__ tok, const int* __restrict__ tpos, const __half* __restrict__ emb,
                                    const float* __restrict__ pos_tab, float scale, float* __restrict__ x, int d) {
  const long i = blockIdx.x;
  const long t = tok[i], p = tpos[i];
  for (int c = threadIdx.x; c < d; c += blockDim.x) x[i * d + c] = __half2float(emb[t * d + c]) * scale + pos_tab[p * d + c];
}

void mt_enc_embed(cudaStream_t st, const int* tok, const int* tpos, const __half* emb, const float* pos_tab, float scale, float* x,
                  long n, int d) {
  launch_kernel(mt_enc_embed_kernel, dim3((unsigned)n), dim3(128), 0, st, tok, tpos, emb, pos_tab, scale, x, d);
  note_launch(1);
}

// decoder row r (active): x[r] = E[tok_in[r]] * scale + P[pos + pad + 1] (P[pad] for the pad token); src[r][pos] = r
__global__ void mt_dec_embed_kernel(MtState s, const __half* __restrict__ emb, const float* __restrict__ pos_tab, float scale,
                                    int pad, float* __restrict__ x, int d) {
  const int r = blockIdx.x;
  if (!s.active[r]) return;
  const long t = s.tok_in[r];
  const int pos = s.pos[r];
  const long p = t == pad ? pad : pos + pad + 1;   // Hugging Face: past length + padding_idx + 1
  for (int c = threadIdx.x; c < d; c += blockDim.x) x[(long)r * d + c] = __half2float(emb[t * d + c]) * scale + pos_tab[p * d + c];
  if (threadIdx.x == 0) s.src[(long)r * T_MAX + pos] = (short)r;
}

void mt_dec_embed(cudaStream_t st, const MtState& s, const __half* emb, const float* pos_tab, float scale, int pad, float* x, int R,
                  int d) {
  PdlScope no_pdl(false);
  launch_kernel(mt_dec_embed_kernel, dim3(R), dim3(128), 0, st, s, emb, pos_tab, scale, pad, x, d);
  note_launch(1);
}

// ============================================================================ encoder self-attention (ragged, non-causal)
// One CTA per (64-query tile of a segment, head), 4 warps, each warp 16 query rows.  S = Q K^T and O += P V on the tensor
// cores (wmma m16n16k16, fp16 in, fp32 accumulate) over 64-key tiles of the segment's own keys; an online softmax in fp32
// between them.  Keys at or beyond the segment's length are masked; query rows beyond it are computed and not stored.
constexpr int EA_T = 64, EA_LD = 72, EA_LDF = 68;
constexpr int EA_SMEM = 4 * EA_T * EA_LD * 2 + 2 * EA_T * EA_LDF * 4 + 2 * EA_T * 4;

__global__ void __launch_bounds__(128) mt_enc_attn_kernel(const __half* __restrict__ qkv, const int* __restrict__ off,
                                                          const int2* __restrict__ tiles, __half* __restrict__ out, int d) {
  using namespace nvcuda;
  extern __shared__ __align__(128) unsigned char ea_smem[];
  __half* sq = reinterpret_cast<__half*>(ea_smem);
  __half* sk = sq + EA_T * EA_LD;
  __half* sv = sk + EA_T * EA_LD;
  __half* sp = sv + EA_T * EA_LD;
  float* ss = reinterpret_cast<float*>(sp + EA_T * EA_LD);
  float* so = ss + EA_T * EA_LDF;
  float* sm = so + EA_T * EA_LDF;
  float* sl = sm + EA_T;
  const int2 tile = tiles[blockIdx.x];
  const int h = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long base = off[tile.x];
  const int L = (int)(off[tile.x + 1] - base), q0 = tile.y;
  const long ld = 3L * d;
  auto load_tile = [&](__half* dst, int row0, int col) {
    for (int i = tid; i < EA_T * 8; i += 128) {
      const int r = i >> 3, c = i & 7;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (row0 + r < L) v = *reinterpret_cast<const uint4*>(qkv + (base + row0 + r) * ld + col + c * 8);
      *reinterpret_cast<uint4*>(dst + r * EA_LD + c * 8) = v;
    }
  };
  load_tile(sq, q0, h * 64);
  for (int i = tid; i < EA_T * EA_LDF; i += 128) so[i] = 0.f;
  if (tid < EA_T) { sm[tid] = -INFINITY; sl[tid] = 0.f; }
  const int r0 = warp * 16;
  for (int k0 = 0; k0 < L; k0 += EA_T) {
    __syncthreads();   // the previous tile's K / V are consumed (and, the first time, Q and the state are in place)
    load_tile(sk, k0, d + h * 64);
    load_tile(sv, k0, 2 * d + h * 64);
    __syncthreads();
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc;
      wmma::fill_fragment(acc, 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> a;
        wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::col_major> b;
        wmma::load_matrix_sync(a, sq + r0 * EA_LD + 16 * k, EA_LD);
        wmma::load_matrix_sync(b, sk + 16 * n * EA_LD + 16 * k, EA_LD);
        wmma::mma_sync(acc, a, b, acc);
      }
      wmma::store_matrix_sync(ss + r0 * EA_LDF + 16 * n, acc, EA_LDF, wmma::mem_row_major);
    }
    __syncwarp();
    const bool v0 = k0 + lane < L, v1 = k0 + lane + 32 < L;
    for (int i = 0; i < 16; ++i) {
      const int r = r0 + i;
      const float s0 = v0 ? ss[r * EA_LDF + lane] * 0.125f : -INFINITY;
      const float s1 = v1 ? ss[r * EA_LDF + lane + 32] * 0.125f : -INFINITY;
      const float m_old = sm[r];
      const float m_new = fmaxf(m_old, warp_max(fmaxf(s0, s1)));   // key k0 is valid: finite
      const float alpha = __expf(m_old - m_new);
      const float p0 = v0 ? __expf(s0 - m_new) : 0.f, p1 = v1 ? __expf(s1 - m_new) : 0.f;
      const float sum = warp_sum(p0 + p1);
      sp[r * EA_LD + lane] = __float2half_rn(p0);
      sp[r * EA_LD + lane + 32] = __float2half_rn(p1);
      so[r * EA_LDF + lane] *= alpha;
      so[r * EA_LDF + lane + 32] *= alpha;
      __syncwarp();
      if (lane == 0) { sm[r] = m_new; sl[r] = sl[r] * alpha + sum; }
    }
    __syncwarp();
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc;
      wmma::fill_fragment(acc, 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> a;
        wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::row_major> b;
        wmma::load_matrix_sync(a, sp + r0 * EA_LD + 16 * k, EA_LD);
        wmma::load_matrix_sync(b, sv + 16 * k * EA_LD + 16 * n, EA_LD);
        wmma::mma_sync(acc, a, b, acc);
      }
      wmma::store_matrix_sync(ss + r0 * EA_LDF + 16 * n, acc, EA_LDF, wmma::mem_row_major);
    }
    __syncwarp();
    for (int i = lane; i < 16 * 64; i += 32) {
      const int r = r0 + (i >> 6), c = i & 63;
      so[r * EA_LDF + c] += ss[r * EA_LDF + c];
    }
  }
  __syncwarp();
  for (int i = lane; i < 16 * 32; i += 32) {
    const int r = r0 + (i >> 5), c = 2 * (i & 31);
    if (q0 + r >= L) continue;
    const float inv = 1.f / sl[r];
    *reinterpret_cast<__half2*>(out + (base + q0 + r) * d + h * 64 + c) =
        __floats2half2_rn(so[r * EA_LDF + c] * inv, so[r * EA_LDF + c + 1] * inv);
  }
}

void mt_enc_attn(cudaStream_t st, const __half* qkv, const int* off, const int2* tiles, int n_tiles, __half* out, int H, int d) {
  // the opt-in shared memory size is a per-device attribute
  static bool primed[64] = {};
  int dev = 0;
  WL_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !primed[dev]) {
    WL_CUDA(cudaFuncSetAttribute(mt_enc_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EA_SMEM));
    if (dev < 64) primed[dev] = true;
  }
  launch_kernel(mt_enc_attn_kernel, dim3(n_tiles, H), dim3(128), EA_SMEM, st, qkv, off, tiles, out, d);
  note_launch(1);
}

// ============================================================================ decoder cross-attention (ragged)
// One warp per (row, head) over the keys of the row's segment (row r belongs to segment r / rows_per_seg).  Lanes own keys
// for the scores (one 128-byte K row each) and dims for the weighted V sum (coalesced 128-byte V rows).
constexpr int XA_WARPS = 4;

__global__ void __launch_bounds__(XA_WARPS * 32) mt_cross_attn_kernel(MtState s, const float* __restrict__ q,
                                                                      const __half* __restrict__ kv, long ldkv, int koff, int voff,
                                                                      const int* __restrict__ off, int rows_per_seg,
                                                                      __half* __restrict__ out, int H, int d, int R) {
  __shared__ float qs[XA_WARPS][64];
  __shared__ float sc_all[XA_WARPS][MT_MAX_SRC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * XA_WARPS + warp;
  pdl_trigger();
  if (item >= R * H) return;
  const int r = item / H, h = item % H;
  if (s.active && !s.active[r]) return;
  pdl_wait();
  const int seg = r / rows_per_seg;
  const long base = off[seg];
  const int n = (int)(off[seg + 1] - base);
  float* qv = qs[warp];
  float* sc = sc_all[warp];
  qv[2 * lane] = q[(long)r * d + h * 64 + 2 * lane] * 0.125f;
  qv[2 * lane + 1] = q[(long)r * d + h * 64 + 2 * lane + 1] * 0.125f;
  __syncwarp();
  float lmax = -INFINITY;
  for (int j = lane; j < n; j += 32) {
    const uint4* kp = reinterpret_cast<const uint4*>(kv + (base + j) * ldkv + koff + h * 64);
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint4 u = kp[c];
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        acc = fmaf(qv[c * 8 + 2 * e], f.x, acc);
        acc = fmaf(qv[c * 8 + 2 * e + 1], f.y, acc);
      }
    }
    sc[j] = acc;
    lmax = fmaxf(lmax, acc);
  }
  const float mx = warp_max(lmax);
  float lsum = 0.f;
  for (int j = lane; j < n; j += 32) {
    const float e = __expf(sc[j] - mx);
    sc[j] = e;
    lsum += e;
  }
  const float inv = 1.f / warp_sum(lsum);
  __syncwarp();
  float a0 = 0.f, a1 = 0.f;
  const __half* vp = kv + base * ldkv + voff + h * 64 + 2 * lane;
#pragma unroll 4
  for (int j = 0; j < n; ++j) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(vp + j * ldkv));
    a0 = fmaf(sc[j], f.x, a0);
    a1 = fmaf(sc[j], f.y, a1);
  }
  *reinterpret_cast<__half2*>(out + (long)r * d + h * 64 + 2 * lane) = __floats2half2_rn(a0 * inv, a1 * inv);
}

void mt_cross_attn(cudaStream_t st, const MtState& s, const float* q, const __half* kv, long ldkv, int koff, int voff, const int* off,
                   int rows_per_seg, __half* out, int R, int H, int d) {
  launch_kernel(mt_cross_attn_kernel, dim3(cdiv((long)R * H, XA_WARPS)), dim3(XA_WARPS * 32), 0, st, s, q, kv, ldkv, koff, voff,
                off, rows_per_seg, out, H, d, R);
  note_launch(1);
}

// ============================================================================ beam search: per-row candidates
// Row r (active): lse = log sum exp(logits[r]); the top n_cand (= 2K) of log_softmax, ties to the lower token.  When the
// step forces a token (forced BOS at the first step, forced EOS at the last), every other log-probability is -inf, as
// Hugging Face's ForcedBOS / ForcedEOS processors leave them: the candidates are the forced token, then the lowest others.
constexpr int MR_THREADS = 512;

struct Cand {
  float v;
  int t;
};
__device__ __forceinline__ bool cand_better(const Cand& a, const Cand& b) { return a.v > b.v || (a.v == b.v && a.t < b.t); }

__global__ void __launch_bounds__(MR_THREADS) mt_rows_kernel(MtState s, const float* __restrict__ logits, long ld, int V,
                                                             int n_cand, int max_length) {
  const int r = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  if (!s.active[r]) return;
  pdl_wait();
  const float* x = logits + (long)r * ld;
  __shared__ float red[MR_THREADS / 32];
  __shared__ Cand cw[MR_THREADS / 32];
  const int seg_len = s.pos[r] + 1;   // cur_len: tokens in the running sequence, the decoder start included
  int forced = -1;
  if (seg_len == 1 && s.forced_bos >= 0) forced = s.forced_bos;
  if (seg_len == max_length - 1 && s.forced_eos >= 0) forced = s.forced_eos;
  float* cv = s.cand_val + (long)r * MT_MAX_CAND;
  int* ct = s.cand_tok + (long)r * MT_MAX_CAND;
  if (forced >= 0) {
    if (tid < n_cand) {
      const int t = tid == 0 ? forced : (tid - 1 < forced ? tid - 1 : tid);
      cv[tid] = tid == 0 ? 0.f : -INFINITY;
      ct[tid] = t;
    }
    return;
  }
  // max, then sum of exp
  float m = -INFINITY;
  for (int i = tid; i < V; i += MR_THREADS) m = fmaxf(m, x[i]);
  m = warp_max(m);
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  if (tid < 32) {
    float v = tid < MR_THREADS / 32 ? red[tid] : -INFINITY;
    v = warp_max(v);
    if (tid == 0) red[0] = v;
  }
  __syncthreads();
  const float mx = red[0];
  __syncthreads();
  float sum = 0.f;
  for (int i = tid; i < V; i += MR_THREADS) sum += expf(x[i] - mx);
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  if (tid < 32) {
    float v = tid < MR_THREADS / 32 ? red[tid] : 0.f;
    v = warp_sum(v);
    if (tid == 0) red[0] = v;
  }
  __syncthreads();
  const float lse = mx + logf(red[0]);
  // top n_cand: every thread keeps its own sorted list, then n_cand rounds of a block arg-max over the list heads
  Cand loc[MT_MAX_CAND];
#pragma unroll
  for (int k = 0; k < MT_MAX_CAND; ++k) loc[k] = Cand{-INFINITY, 0x7fffffff};
  for (int i = tid; i < V; i += MR_THREADS) {
    Cand c{x[i], i};
    if (!cand_better(c, loc[MT_MAX_CAND - 1])) continue;
#pragma unroll
    for (int k = MT_MAX_CAND - 1; k >= 0; --k) {
      const bool shift = k > 0 && cand_better(c, loc[k - 1]);
      if (cand_better(c, loc[k])) loc[k] = shift ? loc[k - 1] : c;
    }
  }
  for (int k = 0; k < n_cand; ++k) {
    Cand best = loc[0];
    for (int o = 16; o > 0; o >>= 1) {
      Cand oc{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.t, o)};
      if (cand_better(oc, best)) best = oc;
    }
    if ((tid & 31) == 0) cw[tid >> 5] = best;
    __syncthreads();
    if (tid < 32) {
      Cand b = tid < MR_THREADS / 32 ? cw[tid] : Cand{-INFINITY, 0x7fffffff};
      for (int o = 16; o > 0; o >>= 1) {
        Cand oc{__shfl_xor_sync(0xffffffffu, b.v, o), __shfl_xor_sync(0xffffffffu, b.t, o)};
        if (cand_better(oc, b)) b = oc;
      }
      if (tid == 0) {
        cv[k] = b.v - lse;
        ct[k] = b.t;
        red[0] = __int_as_float(b.t);
      }
    }
    __syncthreads();
    if (loc[0].t == __float_as_int(red[0])) {   // a token lives in one thread's list only: that thread pops its head
#pragma unroll
      for (int j = 0; j < MT_MAX_CAND - 1; ++j) loc[j] = loc[j + 1];
      loc[MT_MAX_CAND - 1] = Cand{-INFINITY, 0x7fffffff};
    }
    __syncthreads();
  }
}

// ============================================================================ beam search: per-segment step
// Hugging Face's _beam_search for one segment, one step (generation/utils.py, transformers 5.5): the top 2K of the K x 2K
// row candidates plus running scores; EOS (or the max_length cut) closes a candidate; the K best open candidates run on;
// the first K closed ones enter the finished table with score / generated_len ** length_penalty unless the table is
// frozen; then the early-stop heuristic.  K == 1 is greedy search (arg-max, stop at EOS or max_length).  One warp.
__global__ void __launch_bounds__(32) mt_merge_kernel(MtState s, MtSearch o) {
  const int b = blockIdx.x, lane = threadIdx.x, K = o.beam, C = o.beam == 1 ? 1 : 2 * o.beam;
  pdl_trigger();
  pdl_wait();
  if (s.done[b]) return;
  const int row0 = b * K;
  const int cur_len = s.pos[row0] + 1;
  __shared__ Cand top[MT_MAX_CAND];
  __shared__ int parent[MT_MAX_CAND];
  __shared__ int hist_tmp[MT_MAX_BEAM][T_MAX];
  __shared__ short src_tmp[MT_MAX_BEAM][T_MAX];
  __shared__ int sel[MT_MAX_BEAM];           // running beams of the next step: index into top
  __shared__ int fin_from[MT_MAX_BEAM];      // finished table after the merge: < K old slot, else K + index into top
  __shared__ int fin_len_new[MT_MAX_BEAM];
  __shared__ float fin_score_new[MT_MAX_BEAM];
  __shared__ int fin_flag_new[MT_MAX_BEAM];
  __shared__ int step_done;
  // 1. top C over the K rows' candidates + running scores (flattened index row * V + token breaks ties)
  {
    Cand loc[MT_MAX_BEAM * MT_MAX_CAND / 32];
    int lrow[MT_MAX_BEAM * MT_MAX_CAND / 32];
    const int per_row = C, total = K * per_row;
#pragma unroll
    for (int i = 0; i < MT_MAX_BEAM * MT_MAX_CAND / 32; ++i) {
      const int idx = lane + 32 * i;
      loc[i] = Cand{-INFINITY, 0x7fffffff};
      lrow[i] = 0x7fff;
      if (idx < total) {
        const int k = idx / per_row, j = idx % per_row, r = row0 + k;
        loc[i] = Cand{s.cand_val[(long)r * MT_MAX_CAND + j] + s.run_score[r], s.cand_tok[(long)r * MT_MAX_CAND + j]};
        lrow[i] = k;
      }
    }
    for (int c = 0; c < C; ++c) {
      int bi = -1;
      Cand best{-INFINITY, 0x7fffffff};
      int brow = 0x7fff;
#pragma unroll
      for (int i = 0; i < MT_MAX_BEAM * MT_MAX_CAND / 32; ++i) {
        if (lrow[i] == 0x7fff) continue;
        const bool better = loc[i].v > best.v || (loc[i].v == best.v && (lrow[i] < brow || (lrow[i] == brow && loc[i].t < best.t)));
        if (bi < 0 || better) { bi = i; best = loc[i]; brow = lrow[i]; }
      }
      int key_row = brow, key_lane = lane;
      for (int off = 16; off > 0; off >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best.v, off);
        const int ot = __shfl_xor_sync(0xffffffffu, best.t, off);
        const int orow = __shfl_xor_sync(0xffffffffu, key_row, off);
        const int olane = __shfl_xor_sync(0xffffffffu, key_lane, off);
        const bool better = orow != 0x7fff && (key_row == 0x7fff || ov > best.v ||
                                                (ov == best.v && (orow < key_row || (orow == key_row && ot < best.t))));
        if (better) { best.v = ov; best.t = ot; key_row = orow; key_lane = olane; }
      }
      if (lane == 0) { top[c] = best; parent[c] = key_row; }
      if (lane == key_lane && bi >= 0) lrow[bi] = 0x7fff;
      __syncwarp();
    }
  }
  __syncwarp();
  const int eos = o.eos;
  if (lane == 0) {
    const bool at_max = cur_len + 1 >= o.max_length;
    int done = 0;
    if (K == 1) {
      sel[0] = 0;
      done = top[0].t == eos || at_max;
      if (done) {
        fin_from[0] = 1;   // the candidate itself
        fin_len_new[0] = cur_len + 1;
        fin_score_new[0] = top[0].v;
        fin_flag_new[0] = 1;
      } else {
        fin_from[0] = -1;
      }
    } else {
      // e. running beams: the K best of topk + hits * -1e9
      float rv[MT_MAX_CAND];
      for (int c = 0; c < C; ++c) {
        const bool hit = top[c].t == eos || at_max;
        rv[c] = top[c].v + (hit ? -1.0e9f : 0.f);
      }
      bool used[MT_MAX_CAND];
      for (int c = 0; c < C; ++c) used[c] = false;
      for (int k = 0; k < K; ++k) {
        int bi = -1;
        for (int c = 0; c < C; ++c)
          if (!used[c] && (bi < 0 || rv[c] > rv[bi])) bi = c;
        used[bi] = true;
        sel[k] = bi;
        s.run_next[row0 + k] = rv[bi];
      }
      // f. finished table: merge the K old entries with the C scored candidates, keep the best K (old entries first on ties)
      bool all_fin = true;
      for (int k = 0; k < K; ++k) all_fin = all_fin && s.fin_flag[row0 + k];
      const bool full = all_fin && o.early_stopping == 1;
      const bool unsat = s.unsat[b] != 0;
      const float denom = (float)pow((double)(cur_len + 1 - 1), (double)o.length_penalty);
      float mv[MT_MAX_BEAM + MT_MAX_CAND];
      int mflag[MT_MAX_BEAM + MT_MAX_CAND];
      for (int k = 0; k < K; ++k) { mv[k] = s.fin_score[row0 + k]; mflag[k] = s.fin_flag[row0 + k]; }
      for (int c = 0; c < C; ++c) {
        const bool hit = top[c].t == eos || at_max;
        const bool did = hit && c < K;
        float v = top[c].v / denom;
        v = v + (full ? -1.0e9f : 0.f);
        v = v + (!unsat ? -1.0e9f : 0.f);
        v = v + (!did ? -1.0e9f : 0.f);
        mv[K + c] = v;
        mflag[K + c] = did ? 1 : 0;
      }
      bool mused[MT_MAX_BEAM + MT_MAX_CAND];
      for (int i = 0; i < K + C; ++i) mused[i] = false;
      for (int k = 0; k < K; ++k) {
        int bi = -1;
        for (int i = 0; i < K + C; ++i)
          if (!mused[i] && (bi < 0 || mv[i] > mv[bi])) bi = i;
        mused[bi] = true;
        fin_from[k] = bi;
        fin_score_new[k] = mv[bi];
        fin_flag_new[k] = mflag[bi];
        fin_len_new[k] = bi < K ? s.fin_len[row0 + bi] : cur_len + 1;
      }
      // g. early-stop heuristic after cur_len + 1, and the segment's stopping rule
      const int new_len = cur_len + 1;
      const int bhl = (o.early_stopping == 2 && o.length_penalty > 0.f) ? o.max_length - 1 : new_len - 1;
      const float best_run = s.run_next[row0] / (float)pow((double)bhl, (double)o.length_penalty);
      float worst = fin_score_new[0];
      bool fin_all = true;
      for (int k = 0; k < K; ++k) { worst = fminf(worst, fin_score_new[k]); fin_all = fin_all && fin_flag_new[k]; }
      bool improve = false;
      for (int k = 0; k < K; ++k) improve = improve || best_run > (fin_flag_new[k] ? worst : -1.0e9f);
      const bool unsat_new = unsat && improve;
      s.unsat[b] = unsat_new ? 1 : 0;
      done = !unsat_new || (o.early_stopping == 1 && fin_all) || at_max;
    }
    step_done = done;
  }
  __syncwarp();
  // stage the old running sequences / indirection rows, then rewrite finished entries and running rows
  for (int i = lane; i < K * cur_len; i += 32) {
    const int k = i / cur_len, p = i % cur_len;
    hist_tmp[k][p] = s.hist[(long)(row0 + k) * T_MAX + p];
    src_tmp[k][p] = s.src[(long)(row0 + k) * T_MAX + p];
  }
  __syncwarp();
  if (K == 1) {
    if (fin_from[0] == 1) {
      for (int p = lane; p < cur_len; p += 32) s.fin_tok[(long)b * MT_MAX_BEAM * T_MAX + p] = hist_tmp[0][p];
      if (lane == 0) {
        s.fin_tok[(long)b * MT_MAX_BEAM * T_MAX + cur_len] = top[0].t;
        s.fin_len[row0] = fin_len_new[0];
        s.fin_score[row0] = s.run_score[row0] + s.cand_val[(long)row0 * MT_MAX_CAND];
        s.fin_flag[row0] = 1;
      }
    }
    if (lane == 0) s.run_next[row0] = s.run_score[row0] + s.cand_val[(long)row0 * MT_MAX_CAND];
  } else {
    // the merge may move a finished entry to any slot: stage the old table, then write every slot from it
    __shared__ int ftmp[MT_MAX_BEAM][T_MAX];
    for (int i = lane; i < K * T_MAX; i += 32) {
      const int k = i / T_MAX, p = i % T_MAX;
      ftmp[k][p] = s.fin_tok[((long)b * MT_MAX_BEAM + k) * T_MAX + p];
    }
    __syncwarp();
    for (int k = 0; k < K; ++k) {
      const int from = fin_from[k];
      int* dst = s.fin_tok + ((long)b * MT_MAX_BEAM + k) * T_MAX;
      if (from < K) {
        for (int p = lane; p < T_MAX; p += 32) dst[p] = ftmp[from][p];
      } else {
        const int c = from - K;
        for (int p = lane; p < cur_len; p += 32) dst[p] = hist_tmp[parent[c]][p];
        if (lane == 0) dst[cur_len] = top[c].t;
      }
    }
    if (lane < K) {
      s.fin_score[row0 + lane] = fin_score_new[lane];
      s.fin_flag[row0 + lane] = fin_flag_new[lane];
      s.fin_len[row0 + lane] = fin_len_new[lane];
    }
  }
  __syncwarp();
  if (step_done) {
    for (int k = lane; k < K; k += 32) s.active[row0 + k] = 0;
    if (lane == 0) {
      s.done[b] = 1;
      s.steps[b] = cur_len;
      atomicAdd(s.n_done, 1);
    }
    return;
  }
  for (int k = 0; k < K; ++k) {
    const int c = sel[k], pr = parent[c];
    const long r = row0 + k;
    for (int p = lane; p < cur_len; p += 32) {
      s.hist[r * T_MAX + p] = hist_tmp[pr][p];
      s.src[r * T_MAX + p] = src_tmp[pr][p];
    }
    if (lane == 0) {
      s.hist[r * T_MAX + cur_len] = top[c].t;
      s.tok_in[r] = top[c].t;
      s.pos[r] = cur_len;
      s.run_score[r] = s.run_next[r];
    }
  }
}

void mt_search_step(cudaStream_t st, const MtState& s, const MtSearch& o, const float* logits, long ld, int V, int B) {
  const int R = B * o.beam;
  const int n_cand = o.beam == 1 ? 1 : 2 * o.beam;
  launch_kernel(mt_rows_kernel, dim3(R), dim3(MR_THREADS), 0, st, s, logits, ld, V, n_cand, o.max_length);
  launch_kernel(mt_merge_kernel, dim3(B), dim3(32), 0, st, s, o);
  note_launch(2);
}

__global__ void mt_loop_condition_kernel(MtState s, cudaGraphConditionalHandle h, int B) {
  if (threadIdx.x == 0) {
    const int left = *s.steps_left - 1;
    *s.steps_left = left;
    cudaGraphSetConditional(h, (left > 0 && *s.n_done < B) ? 1u : 0u);
  }
}

void mt_loop_condition(cudaStream_t st, const MtState& s, cudaGraphConditionalHandle h, int B) {
  PdlScope no_pdl(false);
  launch_kernel(mt_loop_condition_kernel, dim3(1), dim3(32), 0, st, s, h, B);
  note_launch(1);
}

// rows of segment b: token = decoder start, position 0, running score 0 for beam 0 and -1e9 for the others (Hugging Face
// starts every beam but the first at -1e9), empty finished table at -1e9, heuristic unsatisfied
__global__ void mt_search_init_kernel(MtState s, int K, int start, int steps) {
  const int b = blockIdx.x, k = threadIdx.x;
  if (k < K) {
    const int r = b * K + k;
    s.tok_in[r] = start;
    s.pos[r] = 0;
    s.active[r] = 1;
    s.run_score[r] = k == 0 ? 0.f : -1.0e9f;
    s.fin_score[r] = -1.0e9f;
    s.fin_flag[r] = 0;
    s.fin_len[r] = 0;
    s.hist[(long)r * T_MAX] = start;
  }
  if (k == 0) {
    s.done[b] = 0;
    s.unsat[b] = 1;
    s.steps[b] = 0;
    if (b == 0) { *s.n_done = 0; *s.steps_left = steps; }
  }
}

void mt_search_init(cudaStream_t st, const MtState& s, int B, int K, int start, int steps) {
  PdlScope no_pdl(false);
  launch_kernel(mt_search_init_kernel, dim3(B), dim3(32), 0, st, s, K, start, steps);
  note_launch(1);
}

}  // namespace wl
