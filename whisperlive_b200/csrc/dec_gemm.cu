// Decode-step GEMM (K9 / K12): Y^T[n_out, R] = W[n_out, K] * X[R, K]^T, weight-streaming, split over K.
//
// Why a second GEMM kernel next to gemm.cu: the decode step is a chain of ~200 dependent launches per token, and what
// each of them costs is dominated by fetching its instructions, not by the kernel boundary: the general GEMM kernel
// carries four epilogues, batching, tile walks and the fused post-op, the kernels of one layer together overflow the
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

// The pipeline both decode GEMMs share.  CTA = 384 threads: warp 0 is the TMA producer (its first STAGES weight k-blocks
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

// ------------------------------------------------------------------------------------------------------------------
// cgemm: the same pipeline with the K split held inside a thread-block CLUSTER.  The K ranges of one output tile are
// the CTAs of one cluster; each parks its fp32 accumulator tile in its own (by then idle) pipeline buffers, and after a
// cluster barrier every CTA sums a share of the tile's rows across the cluster through distributed shared memory --
// in rank order, so the result is bit-reproducible -- and applies the epilogue: + bias, + residual in place, or
// GELU -> fp16.  Nothing partial ever reaches L2/HBM: at 128 rows the split-K partials of one layer were 30 MB of
// write + re-read traffic per token step, the consumers (LayerNorm, attention) summed up to 8 ranges per element, and
// FC1 needed its own GELU-cast launch.
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float dsmem_ld(uint32_t local_addr, uint32_t rank) {
  uint32_t remote;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_addr), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

struct CGemmParams {
  const float* bias;   // [M] or null
  float* out_f32;      // [N][M] (modes 0, 1)
  __half* out_f16;     // [N][M] (mode 2)
  int M, N, mode;
  int kb_total, kb_per_split, tiles_m, nsplit;
};

template <int BN, int STAGES>
__global__ void __launch_bounds__(384, 1)
cgemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const CGemmParams p) {
  extern __shared__ uint8_t dg_smem_raw[];
  uint8_t* base = dg_smem_raw + ((1024u - (smem_u32(dg_smem_raw) & 1023u)) & 1023u);
  constexpr int B_BYTES = BN * DG_BK * 2;
  constexpr int NTHREADS = 384;
  static_assert(BN * DG_BM * 4 <= STAGES * DG_A_BYTES, "the accumulator tile is parked in the weight stages");
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * DG_A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  uint64_t* empty = full + STAGES;
  float* red = reinterpret_cast<float*>(sA);   // [BN rows][128 features] once the MMAs are done

  const int split = blockIdx.x % p.nsplit;     // = rank in the cluster (cluster = nsplit consecutive CTAs)
  const int rest = blockIdx.x / p.nsplit;
  const int tile_m = rest % p.tiles_m, tile_n = rest / p.tiles_m;
  const int kb0 = split * p.kb_per_split;
  const int num_kb = min(p.kb_per_split, p.kb_total - kb0);
  pdl_trigger();
  dg_init_barriers<BN, STAGES>(tmW, tmX, full, empty);
  float tile_acc[BN / 2];
  if (dg_pipeline<BN, STAGES>(tmW, tmX, sA, sB, full, empty, tile_m, tile_n, kb0, num_kb, tile_acc)) {
    // both consumer warpgroups have retired every MMA before either overwrites the stages with its tile
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const int m0 = (((threadIdx.x >> 5) >> 2) - 1) * 64;
    wgmma_acc_foreach(tile_acc, [&](int r, int c, float v) { red[c * DG_BM + m0 + r] = v; });
  }
  cluster_sync_all();   // every K range of this tile is parked (also orders this CTA's own warps)
  pdl_wait();           // (resolved long ago; every thread below touches memory of the preceding kernels)
  {
    // rows split .. split + nsplit*j of the tile are summed by this CTA, 128 features across consecutive threads
    const int ml = threadIdx.x & (DG_BM - 1), m = tile_m * DG_BM + ml;
    const int ns = p.nsplit;
    const float bias = (p.bias != nullptr && m < p.M) ? p.bias[m] : 0.f;
    const uint32_t local0 = smem_u32(red + ml);
    uint32_t remote[8];   // this thread's feature column in every rank's parked tile
#pragma unroll
    for (int r = 0; r < 8; ++r) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote[r]) : "r"(local0), "r"((uint32_t)min(r, ns - 1)));
#pragma unroll 2
    for (int n = split + ns * (int)(threadIdx.x >> 7); n < BN; n += ns * (NTHREADS >> 7)) {
      const int ng = tile_n * BN + n;
      if (ng >= p.N) break;
      const long o = (long)ng * p.M + m;
      float resid = 0.f;
      if (p.mode == 1 && m < p.M) resid = p.out_f32[o];
      float part[8];   // all ranks' loads in flight together rather than one rank after the other
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        part[r] = 0.f;
        if (r < ns) asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(part[r]) : "r"(remote[r] + (uint32_t)n * (DG_BM * 4)) : "memory");
      }
      float acc = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) acc += part[r];   // rank order: reproducible (absent ranks add +0)
      acc += bias;
      if (m < p.M) {
        if (p.mode == 2) p.out_f16[o] = __float2half_rn(gelu_erf(acc));
        else p.out_f32[o] = acc + resid;
      }
    }
  }
  cluster_sync_all();   // nobody leaves while a peer may still read its tile
}

static std::atomic<long> g_cgemm_launches{0};
static int g_cg_max_clusters[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // [cluster size] -> clusters resident at once (BN = 128 instance)

template <int BN, int STAGES>
static void cg_launch(cudaStream_t st, const CUtensorMap& tw, const CUtensorMap& tx, const CGemmParams& p, int grid) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(384);
  cfg.dynamicSmemBytes = (size_t)dg_smem<BN, STAGES>();
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)p.nsplit;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_active() ? 2 : 1;
  WL_CUDA(cudaLaunchKernelEx(&cfg, cgemm_kernel<BN, STAGES>, tw, tx, p));
}
template <int BN, int STAGES>
static void cg_prime() {
  WL_CUDA(cudaFuncSetAttribute(cgemm_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, dg_smem<BN, STAGES>()));
}
void cgemm_prime() {
  cg_prime<16, 8>();
  cg_prime<32, 8>();
  cg_prime<64, 6>();
  cg_prime<128, 6>();
  // how many clusters of each size the device holds at once (one CTA per SM, clusters do not span GPCs): the split plan
  // keeps every launch inside one wave
  for (int cs = 1; cs <= 8; ++cs) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(cs * 64);
    cfg.blockDim = dim3(384);
    cfg.dynamicSmemBytes = (size_t)dg_smem<128, 6>();
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, cgemm_kernel<128, 6>, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
    g_cg_max_clusters[cs] = n;
  }
}

// K ranges (= cluster size) for one launch: as many as fill the SMs, at most 8, every range non-empty, and the whole
// grid resident at once
int cgemm_split_plan(int n_out, int R, int K) {
  const int bn = dg_bn(R);
  const int tiles = cdiv(n_out, DG_BM) * cdiv(R, bn), total_kb = cdiv(K, DG_BK);
  int best = 1;
  for (int s = 1; s <= 8 && s <= total_kb; ++s) {
    if (cdiv(total_kb, cdiv(total_kb, s)) != s) continue;
    if (s > 1 && g_cg_max_clusters[s] < tiles) continue;
    best = s;
  }
  return best;
}

// mode 0: out_f32 = acc + bias; 1: out_f32 += acc + bias; 2: out_f16 = gelu(acc + bias).  Outputs are [R][n_out].
void cgemm(cudaStream_t st, const __half* W, int n_out, int K, const __half* X, int R, const float* bias, int mode, float* out_f32,
           __half* out_f16) {
  WL_CHECK(n_out > 0 && R > 0 && K > 0 && K % 8 == 0 && mode >= 0 && mode <= 2, WL_ERR_ARG, "cgemm: bad problem %dx%dx%d mode %d", n_out, R,
           K, mode);
  const int bn = dg_bn(R);
  GemmOperand a, b;
  a.ptr = W; a.rows = n_out; a.k = K; a.ld = K;
  b.ptr = X; b.rows = R; b.k = K; b.ld = K;
  const TmapInfo ia = make_tmap(a, DG_BM), ib = make_tmap(b, bn);
  WL_CHECK(ia.pos[0] == 1 && ib.pos[0] == 1, WL_ERR_STATE, "cgemm: unexpected tensor-map layout");
  CGemmParams p;
  p.bias = bias; p.out_f32 = out_f32; p.out_f16 = out_f16; p.M = n_out; p.N = R; p.mode = mode;
  p.nsplit = cgemm_split_plan(n_out, R, K);
  p.kb_total = cdiv(K, DG_BK);
  p.kb_per_split = cdiv(p.kb_total, p.nsplit);
  p.tiles_m = cdiv(n_out, DG_BM);
  const int grid = p.tiles_m * p.nsplit * cdiv(R, bn);
  switch (bn) {
    case 16: cg_launch<16, 8>(st, ia.tm, ib.tm, p, grid); break;
    case 32: cg_launch<32, 8>(st, ia.tm, ib.tm, p, grid); break;
    case 64: cg_launch<64, 6>(st, ia.tm, ib.tm, p, grid); break;
    default: cg_launch<128, 6>(st, ia.tm, ib.tm, p, grid); break;
  }
  g_cgemm_launches++;
}
long cgemm_launch_count() { return g_cgemm_launches.load(); }

}  // namespace wl
