// Decode-step GEMM (K9 / K12): Y^T[n_out, R] = W[n_out, K] * X[R, K]^T, weight-streaming, split over K.
//
// Why a second GEMM kernel next to gemm.cu: the decode step is a chain of ~200 dependent launches per token, and what
// each of them costs is dominated by fetching its instructions, not by the kernel boundary: the general GEMM kernel
// carries three epilogues, batching and tile walks, the kernels of one layer together overflow the
// SM's instruction caches, so every launch streams its code from L2 again (tools/timeline.py measures this per kernel).
// This kernel is the same TMA / wgmma pipeline cut down to what the decode step needs:
//   * one tile per CTA (grid = feature tiles x K ranges x row tiles), no persistent tile walk;
//   * one epilogue: the raw fp32 partial sum of this K range, stored transposed (consecutive features per store);
//     whoever consumes it adds the ranges and the bias in index order (bit-reproducible, no atomics);
//   * the vocabulary projection is the same thing with one K range and the logits buffer as the output.
// The weight k-blocks of the first STAGES stages are requested before griddepcontrol.wait (PDL): they stream while the
// kernel that produces X is still running.
#include <algorithm>
#include <atomic>
#include <cstdlib>

#include "gemm.cuh"

namespace wl {

static std::atomic<long> g_dec_gemm_launches{0};

struct DecGemmParams {
  float* out;          // [nsplit][R][ldn] fp32
  long part_stride;    // elements between K ranges
  int M, N, ldn;       // output features, rows, row pitch of out
  int kb_total, kb_per_split, tiles_m, nsplit;
};

constexpr int DG_BM = 128, DG_BK = 64, DG_A_BYTES = DG_BM * DG_BK * 2;

// The TMA / wgmma pipeline.  CTA = 384 threads: warp 0 is the TMA producer (its first STAGES weight k-blocks
// are requested before the dependency wait), warpgroups 1 and 2 multiply feature rows 0-63 / 64-127 of the tile into
// acc.  Returns true on the consumer threads, whose acc then holds this CTA's K range of the tile.
template <int BN, int STAGES>
__device__ __forceinline__ bool dg_pipeline(const CUtensorMap& tmW, const CUtensorMap& tmX, uint8_t* sA, uint8_t* sB, uint64_t* full,
                                            uint64_t* empty, int tile_m, int tile_n, int kb0, int num_kb, float (&acc)[BN / 2]) {
  constexpr int B_BYTES = BN * DG_BK * 2;
  const int warp = threadIdx.x >> 5;
  if (warp == 0) {
    if (elect_one()) {
      const int pre = min(num_kb, STAGES);
#pragma unroll 1
      for (int kb = 0; kb < pre; ++kb) {   // weights do not depend on the preceding kernel
        mbar_expect_tx(&full[kb], DG_A_BYTES + B_BYTES);
        tma_load_4d(sA + kb * DG_A_BYTES, &tmW, &full[kb], (kb0 + kb) * DG_BK, tile_m * DG_BM, 0, 0);
      }
      if (blockIdx.x == 0) tl_stamp_any(TL_GEMM_PART, 0);
      pdl_wait();
      if (blockIdx.x == 0) tl_stamp_any(TL_GEMM_PART, 1);
      int stage = 0;
      uint32_t phase = 0;
#pragma unroll 1
      for (int kb = 0; kb < num_kb; ++kb) {
        const int k0 = (kb0 + kb) * DG_BK;
        if (kb >= pre) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], DG_A_BYTES + B_BYTES);
          tma_load_4d(sA + stage * DG_A_BYTES, &tmW, &full[stage], k0, tile_m * DG_BM, 0, 0);
        }
        tma_load_4d(sB + stage * B_BYTES, &tmX, &full[stage], k0, tile_n * BN, 0, 0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return false;
  }
  if (warp < 4) return false;
  const int wg = (warp >> 2) - 1;
  int stage = 0, prev = -1;   // acc needs no initialisation: the first k-step of k-block 0 overwrites it (scale-d 0)
  uint32_t phase = 0;
#pragma unroll 1
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full[stage], phase);
    wgmma_fence();
    wgmma_tile_k64<BN>(acc, sA + stage * DG_A_BYTES, sB + stage * B_BYTES, wg, kb > 0);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  return true;
}

template <int BN, int STAGES>
__device__ __forceinline__ void dg_init_barriers(const CUtensorMap& tmW, const CUtensorMap& tmX, uint64_t* full, uint64_t* empty) {
  const int warp = threadIdx.x >> 5;
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
  }
  if (warp == 1 && elect_one()) {
#pragma unroll 1
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(384, 1)
dec_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const DecGemmParams p) {
  extern __shared__ uint8_t dg_smem_raw[];
  uint8_t* base = dg_smem_raw + ((1024u - (smem_u32(dg_smem_raw) & 1023u)) & 1023u);
  constexpr int B_BYTES = BN * DG_BK * 2;
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * DG_A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  uint64_t* empty = full + STAGES;

  const int tile_m = blockIdx.x % p.tiles_m;
  const int rest = blockIdx.x / p.tiles_m;
  const int split = rest % p.nsplit, tile_n = rest / p.nsplit;
  const int kb0 = split * p.kb_per_split;
  const int num_kb = min(p.kb_per_split, p.kb_total - kb0);
  pdl_trigger();
  dg_init_barriers<BN, STAGES>(tmW, tmX, full, empty);
  float acc[BN / 2];
  if (!dg_pipeline<BN, STAGES>(tmW, tmX, sA, sB, full, empty, tile_m, tile_n, kb0, num_kb, acc)) return;
  // thread rows = features (8 consecutive per store instruction), stored transposed: out[split][row][feature]
  const int m0 = tile_m * DG_BM + (((threadIdx.x >> 5) >> 2) - 1) * 64;
  float* dst = p.out + (long)split * p.part_stride;
  pdl_wait();   // the partial buffer may still be read by the kernels before this one
  wgmma_acc_foreach(acc, [&](int r, int c, float v) {
    const int m = m0 + r, n = tile_n * BN + c;
    if (m < p.M && n < p.N) dst[(long)n * p.ldn + m] = v;
  });
}

template <int BN, int STAGES>
static constexpr int dg_smem() { return STAGES * (DG_A_BYTES + BN * DG_BK * 2) + 1024 + 256; }

template <int BN, int STAGES>
static void dg_launch(cudaStream_t st, const CUtensorMap& tw, const CUtensorMap& tx, const DecGemmParams& p, int grid) {
  launch_kernel(dec_gemm_kernel<BN, STAGES>, dim3(grid), dim3(384), (size_t)dg_smem<BN, STAGES>(), st, tw, tx, p);
}
template <int BN, int STAGES>
static void dg_prime() {
  WL_CUDA(cudaFuncSetAttribute(dec_gemm_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, dg_smem<BN, STAGES>()));
}
void dec_gemm_tl_bind(unsigned long long* p) { tl_bind_tu(p); }
// Ring depth = how many weight k-blocks are in flight BEFORE the dependency wait resolves (PDL): 8 stages cover a whole
// K range of every decode GEMM but FC2 (10 k-blocks), so the weights are in shared memory when X arrives.
void dec_gemm_prime() {
  dg_prime<16, 8>();
  dg_prime<32, 8>();
  dg_prime<64, 6>();
  dg_prime<128, 6>();
}

static int dg_bn(int R) { return R <= 16 ? 16 : R <= 32 ? 32 : R <= 64 ? 64 : 128; }

// K ranges so that feature tiles x ranges x row tiles is about one CTA per SM (never more than 8 ranges: the
// consumers unroll over them, and each range must hold at least one k-block)
int dec_gemm_split_plan(int n_out, int R, int K, int max_split) {
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  const int bn = dg_bn(R);
  const int tiles = cdiv(n_out, DG_BM) * cdiv(R, bn), total_kb = cdiv(K, DG_BK);
  const int s = std::max(1, std::min(std::min(total_kb, std::min(8, max_split)), sms / std::max(1, tiles)));
  const int kbs = cdiv(total_kb, s);
  return cdiv(total_kb, kbs);
}

// out[s][r][ldn] (s < nsplit) = partial sums of W[n_out, K] x X[R, K]^T over K range s.
void dec_gemm(cudaStream_t st, const __half* W, int n_out, int K, const __half* X, int R, float* out, int ldn, long part_stride,
              int nsplit) {
  WL_CHECK(n_out > 0 && R > 0 && K > 0 && K % 8 == 0 && nsplit >= 1, WL_ERR_ARG, "dec_gemm: bad problem %dx%dx%d/%d", n_out, R, K, nsplit);
  const int bn = dg_bn(R);
  GemmOperand a, b;
  a.ptr = W; a.rows = n_out; a.k = K; a.ld = K;
  b.ptr = X; b.rows = R; b.k = K; b.ld = K;
  const TmapInfo ia = make_tmap(a, DG_BM), ib = make_tmap(b, bn);
  WL_CHECK(ia.pos[0] == 1 && ib.pos[0] == 1, WL_ERR_STATE, "dec_gemm: unexpected tensor-map layout");
  DecGemmParams p;
  p.out = out; p.part_stride = part_stride; p.M = n_out; p.N = R; p.ldn = ldn;
  p.kb_total = cdiv(K, DG_BK);
  p.kb_per_split = cdiv(p.kb_total, nsplit);
  WL_CHECK(cdiv(p.kb_total, p.kb_per_split) == nsplit, WL_ERR_ARG, "dec_gemm: %d K ranges cannot be formed from %d k-blocks", nsplit, p.kb_total);
  p.tiles_m = cdiv(n_out, DG_BM);
  p.nsplit = nsplit;
  const int grid = p.tiles_m * nsplit * cdiv(R, bn);
  switch (bn) {
    case 16: dg_launch<16, 8>(st, ia.tm, ib.tm, p, grid); break;
    case 32: dg_launch<32, 8>(st, ia.tm, ib.tm, p, grid); break;
    case 64: dg_launch<64, 6>(st, ia.tm, ib.tm, p, grid); break;
    default: dg_launch<128, 6>(st, ia.tm, ib.tm, p, grid); break;
  }
  g_dec_gemm_launches++;
}

long dec_gemm_launch_count() { return g_dec_gemm_launches.load(); }

}  // namespace wl
