// K8 batched prompt prefill: the helper kernels around the GEMMs / attention kernels the engine already has.
//
// A prompt of P tokens (sot_prev + hotwords + previous text + sot sequence, up to ~450 tokens:
// whisper_live/transcriber/transcriber_faster_whisper.py:1480-1513) used to be fed one token per decode step, i.e. P - 1
// full weight streams before the first generated token.  The prefill pass pushes all prompt positions of all streams
// through the decoder stack at once -- M = sum(P_b - 1) rows per GEMM on the encoder's wgmma kernel, causal
// self-attention over the cached positions, cross-attention in groups of 8 rows per K/V stream -- and leaves the
// self-attention cache and the decode state exactly where token-by-token feeding would have left them.
//
// Row layout: stream b owns rows [rowbase_b, rowbase_b + n'_b), n'_b = its prefill positions rounded up to a multiple
// of 8 (so that a cross-attention group of 8 rows never straddles two streams); padding rows are inactive.
#include "kernels.cuh"

namespace wl {

// x[i] = E[tok[i]] + P[pos[i]] (f32) for active rows, 0 for padding; also the cache indirection of the row:
// src[i][p] = wrow[i] for p <= pos[i] (all prompt positions of a stream live in its first decode row)
__global__ void __launch_bounds__(128) prefill_embed_kernel(const int* __restrict__ tok, const int* __restrict__ pos,
                                                            const int* __restrict__ active, const int* __restrict__ wrow,
                                                            const __half* __restrict__ emb, const __half* __restrict__ pos_emb,
                                                            float* __restrict__ x, short* __restrict__ src, int d) {
  const int i = blockIdx.x;
  float* xr = x + (long)i * d;
  if (!active[i]) {
    for (int c = threadIdx.x; c < d; c += blockDim.x) xr[c] = 0.f;
    return;
  }
  const int t = tok[i], p = pos[i];
  for (int c = threadIdx.x; c < d; c += blockDim.x)
    xr[c] = __half2float(emb[(long)t * d + c]) + __half2float(pos_emb[(long)p * d + c]);
  const short w = (short)wrow[i];
  for (int q = threadIdx.x; q <= p; q += blockDim.x) src[(long)i * T_MAX + q] = w;
}

void prefill_embed(cudaStream_t st, const int* tok, const int* pos, const int* active, const int* wrow, const __half* emb,
                   const __half* pos_emb, float* x, short* src, int M, int d) {
  prefill_embed_kernel<<<M, 128, 0, st>>>(tok, pos, active, wrow, emb, pos_emb, x, src, d);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// k, v of every prompt position -> self-attention cache rows (fp16), BEFORE the attention kernel runs: position p of a
// stream attends to positions < p that other rows of the same launch produce
__global__ void __launch_bounds__(256) prefill_kv_write_kernel(const float* __restrict__ qkv, const int* __restrict__ pos,
                                                               const int* __restrict__ active, const int* __restrict__ wrow,
                                                               __half* __restrict__ kc, __half* __restrict__ vc, long row_stride,
                                                               int H, int d) {
  const int i = blockIdx.x;
  if (!active[i]) return;
  const long base = (long)wrow[i] * row_stride + (long)pos[i] * 64;
  const float* kp = qkv + (long)i * 3 * d + d;
  const float* vp = kp + d;
  for (int c = threadIdx.x * 2; c < d; c += blockDim.x * 2) {
    const int h = c >> 6, dd = c & 63;
    const long o = base + (long)h * T_MAX * 64 + dd;
    *reinterpret_cast<__half2*>(kc + o) = __floats2half2_rn(kp[c], kp[c + 1]);
    *reinterpret_cast<__half2*>(vc + o) = __floats2half2_rn(vp[c], vp[c + 1]);
  }
}

void prefill_kv_write(cudaStream_t st, const float* qkv, const int* pos, const int* active, const int* wrow, __half* kc, __half* vc,
                      long row_stride, int M, int H, int d) {
  prefill_kv_write_kernel<<<M, 256, 0, st>>>(qkv, pos, active, wrow, kc, vc, row_stride, H, d);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// copy selected rows of x (f32 [M][d]) to dst rows 0..n-1 (the decode step's residual buffer: final LayerNorm +
// vocabulary projection then run on them through the decode kernels)
__global__ void gather_rows_kernel(const float* __restrict__ x, const int* __restrict__ rows, float* __restrict__ dst, int d) {
  const int j = blockIdx.x, r = rows[j];
  for (int c = threadIdx.x; c < d; c += blockDim.x) dst[(long)j * d + c] = r >= 0 ? x[(long)r * d + c] : 0.f;
}
void gather_rows(cudaStream_t st, const float* x, const int* rows, float* dst, int n, int d) {
  gather_rows_kernel<<<n, 256, 0, st>>>(x, rows, dst, d);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// One block per logits row j: p = softmax(logits[j])[target[j]] -> out[out_index[j]] (target < 0: skip).
// no-speech probability at the sot position (K13) and the teacher-forced token probabilities of align (K14).
__global__ void __launch_bounds__(512) row_prob_kernel(const float* __restrict__ logits, int vocab, int vocab_ld,
                                                       const int* __restrict__ target, const int* __restrict__ out_index,
                                                       float* __restrict__ out) {
  const int j = blockIdx.x, tid = threadIdx.x;
  const int t = target[j];
  if (t < 0) return;
  const float* lg = logits + (long)j * vocab_ld;
  __shared__ float red[2][16];
  float m = -INFINITY;
  for (int i = tid; i < vocab; i += 512) m = fmaxf(m, lg[i]);
  m = warp_max(m);
  if ((tid & 31) == 0) red[0][tid >> 5] = m;
  __syncthreads();
  m = warp_max((tid & 31) < 16 ? red[0][tid & 31] : -INFINITY);
  float sum = 0.f;
  for (int i = tid; i < vocab; i += 512) sum += __expf(lg[i] - m);
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[1][tid >> 5] = sum;
  __syncthreads();
  sum = warp_sum((tid & 31) < 16 ? red[1][tid & 31] : 0.f);
  if (tid == 0) out[out_index[j]] = __expf(lg[t] - m) / sum;
}
void row_prob(cudaStream_t st, const float* logits, int vocab, int vocab_ld, const int* target, const int* out_index, float* out, int n) {
  row_prob_kernel<<<n, 512, 0, st>>>(logits, vocab, vocab_ld, target, out_index, out);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

}  // namespace wl

// ============================================================================ K14 alignment post-processing on the device
// Input: the cross-attention probabilities of the model's alignment heads, W[b][h][t][f] (t < T_b tokens of the
// teacher-forced sequence, f < nf_b = num_frames/2 encoder positions).  Pipeline (OpenAI whisper/timing.py, ported by
// CTranslate2; reference call site transcriber_faster_whisper.py:1657-1663): standardise over the token axis -> median
// filter (reflect padding) along time -> mean over heads -> drop the start-sequence rows and the eot row -> DTW on the
// negated matrix -> (text index, time index) path.  Round 1 did all of this on one host thread after B*nh*T blocking
// row copies; here it is three kernels and one small copy of the path.
namespace wl {

__global__ void __launch_bounds__(128) align_standardize_kernel(float* __restrict__ buf, const int* __restrict__ Tn,
                                                                const int* __restrict__ nfn, int nh) {
  const int b = blockIdx.z, h = blockIdx.y, f = blockIdx.x * 128 + threadIdx.x;
  const int T = Tn[b], nf = nfn[b];
  if (f >= nf) return;
  float* col = buf + (((long)b * nh + h) * T_MAX) * S_ENC + f;
  double mean = 0.0;
  for (int t = 0; t < T; ++t) mean += col[(long)t * S_ENC];
  mean /= T;
  double var = 0.0;
  for (int t = 0; t < T; ++t) { const double dl = col[(long)t * S_ENC] - mean; var += dl * dl; }
  const float sd = (float)sqrt(var / T);
  for (int t = 0; t < T; ++t) col[(long)t * S_ENC] = (float)((col[(long)t * S_ENC] - mean) / sd);
}

// mat[b][t][f] = mean over heads of median_width(W[b][h][t][f-pad .. f+pad]) (reflect at the ends of [0, nf))
__global__ void __launch_bounds__(128) align_median_mean_kernel(const float* __restrict__ buf, float* __restrict__ mat,
                                                                const int* __restrict__ Tn, const int* __restrict__ nfn, int nh,
                                                                int width) {
  const int b = blockIdx.z, t = blockIdx.y, f = blockIdx.x * 128 + threadIdx.x;
  const int T = Tn[b], nf = nfn[b];
  if (t >= T || f >= nf) return;
  const int pad = width / 2;
  float acc = 0.f;
  for (int h = 0; h < nh; ++h) {
    const float* row = buf + ((((long)b * nh + h) * T_MAX) + t) * S_ENC;
    float med;
    if (pad == 0 || nf <= pad) {
      med = row[f];
    } else {
      float w[16];
      for (int k = -pad; k <= pad; ++k) {
        int j = f + k;
        if (j < 0) j = -j;
        if (j >= nf) j = 2 * (nf - 1) - j;
        w[k + pad] = row[j];
      }
      // selection of the pad-th smallest (what nth_element returns): partial selection sort, width <= 15
      for (int i = 0; i <= pad; ++i) {
        int mi = i;
        for (int j = i + 1; j < width; ++j) mi = w[j] < w[mi] ? j : mi;
        const float tmp = w[i]; w[i] = w[mi]; w[mi] = tmp;
      }
      med = w[pad];
    }
    acc += med / nh;
  }
  mat[((long)b * T_MAX + t) * S_ENC + f] = acc;
}

// One CTA per stream: anti-diagonal wavefront over the (n+1) x (m+1) accumulated-cost table (n = T - 1 - n_start text
// rows incl. <|notimestamps|>, m = nf frames; one thread per row, n + 1 <= 448 <= 512), three diagonals of it in shared
// memory, the moves packed 2 bits per cell in shared memory (<= 168 KB), then the backtrace by one thread.  Tie rule of the host version it replaces (and of the
// oracle): diagonal only if strictly smaller than both, else up (text) only if strictly smaller than both, else left.
// path_out[b][.] receives the path REVERSED (end -> start), path_len[b] its length.
__global__ void __launch_bounds__(512) align_dtw_kernel(const float* __restrict__ mat, const int* __restrict__ Tn,
                                                        const int* __restrict__ nfn, int n_start, int* __restrict__ path_out,
                                                        int path_cap, int* __restrict__ path_len) {
  extern __shared__ unsigned dtw_smem[];
  const int b = blockIdx.x, i = threadIdx.x;
  const int n = Tn[b] - 1 - n_start, m = nfn[b];
  float* A0 = reinterpret_cast<float*>(dtw_smem);       // diagonal k-2, indexed by i
  float* A1 = A0 + (T_MAX + 1);                          // diagonal k-1
  float* A2 = A1 + (T_MAX + 1);                          // diagonal k
  unsigned* mv = reinterpret_cast<unsigned*>(A2 + (T_MAX + 1));   // [(n+1) * (m+1)] 2-bit moves
  if (n <= 0 || m <= 0) { if (i == 0) path_len[b] = 0; return; }
  const long words = ((long)(n + 1) * (m + 1) + 15) / 16;
  for (long w = i; w < words; w += 512) mv[w] = 0u;
  for (int q = i; q <= n; q += 512) { A0[q] = INFINITY; A1[q] = INFINITY; A2[q] = INFINITY; }
  __syncthreads();
  if (i == 0) A1[0] = 0.f;   // diagonal 0 = cell (0,0); "diagonal -1" (A0) is all inf
  // cost(i-1, j-1) = -mat[n_start + i - 1][j - 1]; this thread walks row i-1 left to right, 8 columns prefetched
  const bool has_row = i >= 1 && i <= n;
  const float* crow = mat + ((long)b * T_MAX + n_start + (has_row ? i - 1 : 0)) * S_ENC;
  float r[8];
  {
    const int j0 = 1 - i;   // column of this thread on diagonal k = 1 (loop starts at k = 1)
#pragma unroll
    for (int q = 0; q < 8; ++q) { const int j = j0 + q; r[q] = (has_row && j >= 1 && j <= m) ? -crow[j - 1] : 0.f; }
  }
  __syncthreads();
  for (int k = 1; k <= n + m; ++k) {
    // diagonal k-1 is in A1 (k = 1: only cell (0,0)); cells (i, j = k - i) of diagonal k
    const int j = k - i;
    float v = INFINITY;
    if (has_row && j >= 1 && j <= m) {
      const float c0 = A0[i - 1], c1 = A1[i - 1], c2 = A1[i];
      float cc; unsigned mvv;
      if (c0 < c1 && c0 < c2) { cc = c0; mvv = 0u; }
      else if (c1 < c0 && c1 < c2) { cc = c1; mvv = 1u; }
      else { cc = c2; mvv = 2u; }
      v = r[0] + cc;
      const long cell = (long)i * (m + 1) + j;
      atomicOr(&mv[cell >> 4], mvv << ((cell & 15) * 2));   // (two cells of one diagonal share a word only when m < 16)
    }
#pragma unroll
    for (int q = 0; q < 7; ++q) r[q] = r[q + 1];
    { const int jn = j + 8; r[7] = (has_row && jn >= 1 && jn <= m) ? -crow[jn - 1] : 0.f; }
    if (i <= n) A2[i] = v;
    __syncthreads();
    float* t = A0; A0 = A1; A1 = A2; A2 = t;
    // k == 1 special case: A0 must hold diagonal 0 = {(0,0)=0}, A1 diagonal 1 -- that is what the rotation gives
  }
  if (i == 0) {
    int ii = n, jj = m, len = 0;
    int* out = path_out + (long)b * path_cap * 2;
    while ((ii > 0 || jj > 0) && len < path_cap) {
      out[2 * len] = ii - 1; out[2 * len + 1] = jj - 1;
      ++len;
      unsigned t2;
      if (ii == 0) t2 = 2u;
      else if (jj == 0) t2 = 1u;
      else { const long cell = (long)ii * (m + 1) + jj; t2 = (mv[cell >> 4] >> ((cell & 15) * 2)) & 3u; }
      if (t2 == 0u) { --ii; --jj; }
      else if (t2 == 1u) --ii;
      else --jj;
    }
    path_len[b] = len;
  }
}

void align_postprocess(cudaStream_t st, float* buf, float* mat, const int* Tn, const int* nfn, int B, int nh, int width, int n_start,
                       int max_T, int* path_out, int path_cap, int* path_len) {
  WL_CHECK(width >= 1 && width <= 15 && (width & 1), WL_ERR_ARG, "align: median filter width %d must be odd and <= 15", width);
  dim3 g1(cdiv(S_ENC, 128), nh, B);
  align_standardize_kernel<<<g1, 128, 0, st>>>(buf, Tn, nfn, nh);
  WL_CUDA(cudaGetLastError());
  dim3 g2(cdiv(S_ENC, 128), max_T, B);
  align_median_mean_kernel<<<g2, 128, 0, st>>>(buf, mat, Tn, nfn, nh, width);
  WL_CUDA(cudaGetLastError());
  const size_t smem = 3 * (T_MAX + 1) * sizeof(float) + (((size_t)(T_MAX + 1) * (S_ENC + 1) + 15) / 16) * sizeof(unsigned) + 64;
  static bool primed = false;
  if (!primed) {
    WL_CUDA(cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    primed = true;
  }
  align_dtw_kernel<<<B, 512, smem, st>>>(mat, Tn, nfn, n_start, path_out, path_cap, path_len);
  WL_CUDA(cudaGetLastError());
  note_launch(3);
}

}  // namespace wl
