// TMA / wgmma GEMM used by every dense contraction on the hot path (K2-K9, K12).
//   C[z][m][n] = epilogue( sum_k A[z][m][k] * B[z][n][k] )      fp16 in, fp32 accumulate
// Both operands are K-major ("TN"): activations [rows, K] and nn.Linear weights [out, K].
#pragma once
#include "common.cuh"

namespace wl {

// One operand as a strided 4-D view (k fastest): element (k, r, i1, i2) at ptr[k + r*ld + i1*s1 + i2*s2].
struct GemmOperand {
  const __half* ptr = nullptr;
  long rows = 0;      // M (for A) or N (for B)
  long k = 0;         // contraction length seen by TMA (reads beyond it are zero-filled)
  long ld = 0;        // elements between consecutive rows (may be < k: overlapping rows, conv-as-GEMM)
  int n1 = 1;         // batch dims; grid z = i1 + n1*i2
  long s1 = 0;
  int n2 = 1;
  long s2 = 0;
};

enum GemmMode : int {
  GEMM_STORE = 0,      // out[z][m*ldm + n*ldn]
  GEMM_HEADSPLIT = 1,  // cross-KV cache layout: row m=(b,s), col n=(h,dd) -> out[slot[b]][h][s][dd]
};

struct GemmEpilogue {
  void* out = nullptr;
  int out_f32 = 0;           // 1: float output, 0: __half
  long ldm = 0, ldn = 1;     // element strides of the output (ldm=1 -> transposed / swap-AB store)
  long ob1 = 0, ob2 = 0;     // output batch strides
  const float* bias = nullptr;
  int bias_on_m = 0;         // bias indexed by m (swap-AB) instead of n
  int gelu = 0;              // exact erf GELU after bias
  int relu = 0;              // max(x, 0) after bias (M2M100 feed-forward)
  const float* resid = nullptr;  // fp32 residual added last; same indexing scheme as out
  long rldm = 0, rldn = 1, rb1 = 0, rb2 = 0;
  int mode = GEMM_STORE;
  // GEMM_HEADSPLIT parameters
  int hs_S = 0, hs_H = 0;
  long hs_slot_stride = 0;
  const int* hs_slots = nullptr;  // device: slot index per stream b
};

// Which persistent wgmma kernel runs a GEMM (gemm.cu).  CLASSIC: both consumer warpgroups share each 128 x BN tile.
// PINGPONG: each warpgroup owns whole 128 x 128 tiles and its epilogue overlaps the other's MMAs; chosen when every CTA
// gets at least two tiles.  AUTO picks from the shape; the others force one (tests).
enum GemmVariant : int { GEMM_AUTO = 0, GEMM_CLASSIC = 1, GEMM_PINGPONG = 2 };

// Launch on `stream`. M/N/K are the logical sizes per batch entry. Throws wl::Error.
void gemm_tn(cudaStream_t stream, const GemmOperand& A, const GemmOperand& B, int M, int N, int K,
             const GemmEpilogue& epi, GemmVariant variant = GEMM_AUTO);
// The variant GEMM_AUTO selects for a GEMM of this shape (Z batch entries).
GemmVariant gemm_tn_variant(int M, int N, int K, int Z);

// Plain CUDA-core reference of the same contract: what the GEMM unit test compares against on-device.
void gemm_tn_simt(cudaStream_t stream, const GemmOperand& A, const GemmOperand& B, int M, int N, int K,
                  const GemmEpilogue& epi);

long gemm_launch_count();

// Compact decode-step GEMM (dec_gemm.cu): out[s][r][ldn] (s < nsplit) = partial sums over K range s of
// W[n_out, K] x X[R, K]^T, fp32, no bias.  nsplit from dec_gemm_split_plan (1 for the vocabulary projection).
void dec_gemm(cudaStream_t st, const __half* W, int n_out, int K, const __half* X, int R, float* out, int ldn, long part_stride,
              int nsplit);
int dec_gemm_split_plan(int n_out, int R, int K, int max_split = 8);
long dec_gemm_launch_count();
void dec_gemm_prime();
void dec_gemm_tl_bind(unsigned long long* p);

// Small-batch decode GEMM with fused epilogue (wgemm.cu, R <= 32 rows, mma.sync + bulk-copied weight slices).
// mode 0: out_f32 = acc + bias; 1: out_f32 += acc + bias (in place); 2: out_f16 = gelu(acc + bias);
// 3: out_f32[ks] = raw partial sum of K range ks (only when K > 1280)
void wgemm(cudaStream_t st, const __half* W, int n_out, int K, const __half* X, int R, const float* bias, int mode, float* out_f32,
           __half* out_f16, long part_stride);
bool wgemm_supported(int R, int K);
int wgemm_ksplit(int K);
long wgemm_launch_count();
void wgemm_prime();
void wgemm_tl_bind(unsigned long long* p);

// Tensor map over an operand view (dims sorted by stride) + the coordinate slots of (row, i1, i2).
struct TmapInfo {
  CUtensorMap tm;
  int pos[3];
};
TmapInfo make_tmap(const GemmOperand& op, int box_rows, int box_k = 64);

}  // namespace wl
