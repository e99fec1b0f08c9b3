// wgmma GEMM: TMA (SWIZZLE_128B) -> smem ring -> wgmma (two consumer warpgroups, fp32 accumulators in registers) ->
// epilogue (bias / GELU / residual / layout transforms fused).
//
// CTA = 384 threads: warp 0 TMA producer, warps 4-11 two consumer warpgroups of 64 tile rows each.  Tile 128 x BN x 64.
#include "gemm.cuh"

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

namespace wl {

static std::atomic<long> g_gemm_launches{0};
long gemm_launch_count() { return g_gemm_launches.load(); }

struct GemmKParams {
  int M, N, K;
  int zn1;  // grid z = i1 + zn1 * i2
  int a_batched, b_batched;
  int a_pos[3], b_pos[3];  // tensor-map coordinate slots (1..3) of (row, i1, i2)
  GemmEpilogue e;
  int vec_ok;  // row-major output, 16-byte aligned rows: use vector stores
  int nz;           // batch entries: tiles = tiles_m * tiles_n * nz
  int n_fastest;    // tile order, see tile_decode()
};

constexpr int BM = 128;
constexpr int BK = 64;  // 64 halves = 128 bytes = one swizzle row
constexpr int A_STAGE_BYTES = BM * BK * 2;

// Epilogue kinds are compile-time so that every kernel instantiation carries exactly one, compact epilogue: the
// decode-step GEMMs run ~200 times per step on a few CTAs each, where instruction fetch of a fat multi-path
// epilogue costs more than its arithmetic.
enum EpiKind : int { EPI_ROW = 0, EPI_COL = 1, EPI_HEADSPLIT = 2 };

template <int cnt, int KIND>
__device__ __forceinline__ void epilogue_chunk(const GemmKParams& p, long m, int n0, const uint32_t (&v)[cnt], int i1, int i2) {
  const GemmEpilogue& e = p.e;
  if (m >= p.M) return;
  if constexpr (KIND == EPI_HEADSPLIT && cnt >= 8) {
    // m = (b, s), n = (h, dd); one thread writes cnt (<=32) consecutive dd of one head row.  The 16-byte pieces of a
    // 128-byte key row are stored XOR-swizzled by (s & 7): the layout ldmatrix wants in the cross-attention kernel.
    // The slot index and the bias are all loaded before the first store: the compiler cannot rule out that a store
    // changes them, so loads placed between the stores would each wait for a round trip to memory.
    const int mi = (int)m;   // m < M, an int
    const int b = mi / e.hs_S, s = mi % e.hs_S;
    const int h = n0 >> 6, dd = n0 & 63;
    const long slot = e.hs_slots[b];
    float x[cnt];
#pragma unroll
    for (int i = 0; i < cnt; ++i) x[i] = __uint_as_float(v[i]);
    if (e.bias) {
#pragma unroll
      for (int i = 0; i < cnt; i += 8) {
        if (n0 + i >= p.N) break;
#pragma unroll
        for (int j = 0; j < 8; ++j) x[i + j] += e.bias[n0 + i + j];
      }
    }
    __half* dst = (__half*)e.out + slot * e.hs_slot_stride + ((long)h * e.hs_S + s) * 64;
#pragma unroll
    for (int i = 0; i < cnt; i += 8) {
      if (n0 + i >= p.N) break;
      __align__(16) __half2 h2[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) h2[j] = __floats2half2_rn(x[i + 2 * j], x[i + 2 * j + 1]);
      *reinterpret_cast<uint4*>(dst + ((((dd + i) >> 3) ^ (s & 7)) << 3)) = *reinterpret_cast<const uint4*>(h2);
    }
    return;
  }
  const long obase = (long)i1 * e.ob1 + (long)i2 * e.ob2 + m * e.ldm;
  const long rbase = (long)i1 * e.rb1 + (long)i2 * e.rb2 + m * e.rldm;
  const float bm = (e.bias && e.bias_on_m) ? e.bias[m] : 0.f;
  if constexpr (KIND == EPI_ROW && cnt >= 8) {
    if (n0 + cnt <= p.N) {
      // The whole piece is inside the tile: every load (bias, residual) is issued before the first store.  The output
      // may be the residual itself (in place), so the compiler keeps a load that follows a store behind it, and loads
      // interleaved with the stores would cost one round trip to memory per 8 columns.  Same arithmetic, same order.
      float x[cnt];
#pragma unroll
      for (int i = 0; i < cnt; ++i) x[i] = __uint_as_float(v[i]) + bm;
      if (e.bias && !e.bias_on_m) {
#pragma unroll
        for (int i = 0; i < cnt; i += 4) {
          const float4 b4 = *reinterpret_cast<const float4*>(e.bias + n0 + i);
          x[i] += b4.x; x[i + 1] += b4.y; x[i + 2] += b4.z; x[i + 3] += b4.w;
        }
      }
      if (e.gelu) {
#pragma unroll
        for (int i = 0; i < cnt; ++i) x[i] = gelu_erf(x[i]);
      }
      if (e.relu) {
#pragma unroll
        for (int i = 0; i < cnt; ++i) x[i] = fmaxf(x[i], 0.f);
      }
      if (e.resid) {
        const float* r = e.resid + rbase + n0;
        float4 r4[cnt / 4];
#pragma unroll
        for (int i = 0; i < cnt / 4; ++i) r4[i] = *reinterpret_cast<const float4*>(r + 4 * i);
#pragma unroll
        for (int i = 0; i < cnt / 4; ++i) {
          x[4 * i] += r4[i].x; x[4 * i + 1] += r4[i].y; x[4 * i + 2] += r4[i].z; x[4 * i + 3] += r4[i].w;
        }
      }
#pragma unroll
      for (int i = 0; i < cnt; i += 8) {
        if (e.out_f32) {
          float* o = (float*)e.out + obase + n0 + i;
          *reinterpret_cast<float4*>(o) = make_float4(x[i], x[i + 1], x[i + 2], x[i + 3]);
          *reinterpret_cast<float4*>(o + 4) = make_float4(x[i + 4], x[i + 5], x[i + 6], x[i + 7]);
        } else {
          __align__(16) __half2 h2[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) h2[j] = __floats2half2_rn(x[i + 2 * j], x[i + 2 * j + 1]);
          *reinterpret_cast<uint4*>((__half*)e.out + obase + n0 + i) = *reinterpret_cast<const uint4*>(h2);
        }
      }
      return;
    }
#pragma unroll
    for (int i = 0; i < cnt; i += 8) {
      const int n = n0 + i;
      if (n >= p.N) break;
      if (n + 8 > p.N) {  // ragged tail of the last tile: element-wise
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (n + j < p.N) {
            float x1 = __uint_as_float(v[i + j]) + bm;
            if (e.bias && !e.bias_on_m) x1 += e.bias[n + j];
            if (e.gelu) x1 = gelu_erf(x1);
            if (e.relu) x1 = fmaxf(x1, 0.f);
            if (e.resid) x1 += e.resid[rbase + n + j];
            if (e.out_f32) ((float*)e.out)[obase + n + j] = x1;
            else ((__half*)e.out)[obase + n + j] = __float2half_rn(x1);
          }
        }
        continue;
      }
      float x[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = __uint_as_float(v[i + j]) + bm;
      if (e.bias && !e.bias_on_m) {
        const float4 b0 = *reinterpret_cast<const float4*>(e.bias + n), b1 = *reinterpret_cast<const float4*>(e.bias + n + 4);
        x[0] += b0.x; x[1] += b0.y; x[2] += b0.z; x[3] += b0.w;
        x[4] += b1.x; x[5] += b1.y; x[6] += b1.z; x[7] += b1.w;
      }
      if (e.gelu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = gelu_erf(x[j]);
      }
      if (e.relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = fmaxf(x[j], 0.f);
      }
      if (e.resid) {
        const float* r = e.resid + rbase + n;
        const float4 r0 = *reinterpret_cast<const float4*>(r), r1 = *reinterpret_cast<const float4*>(r + 4);
        x[0] += r0.x; x[1] += r0.y; x[2] += r0.z; x[3] += r0.w;
        x[4] += r1.x; x[5] += r1.y; x[6] += r1.z; x[7] += r1.w;
      }
      if (e.out_f32) {
        float* o = (float*)e.out + obase + n;
        *reinterpret_cast<float4*>(o) = make_float4(x[0], x[1], x[2], x[3]);
        *reinterpret_cast<float4*>(o + 4) = make_float4(x[4], x[5], x[6], x[7]);
      } else {
        __align__(16) __half2 h2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) h2[j] = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
        *reinterpret_cast<uint4*>((__half*)e.out + obase + n) = *reinterpret_cast<const uint4*>(h2);
      }
    }
    return;
  }
  if constexpr (KIND == EPI_COL || cnt < 8) {
#pragma unroll
  for (int i = 0; i < cnt; ++i) {
    const int n = n0 + i;
    if (n >= p.N) break;
    float x = __uint_as_float(v[i]) + bm;
    if (e.bias && !e.bias_on_m) x += e.bias[n];
    if (e.gelu) x = gelu_erf(x);
    if (e.relu) x = fmaxf(x, 0.f);
    if (e.resid) x += e.resid[rbase + (long)n * e.rldn];
    const long o = obase + (long)n * e.ldn;
    if (e.out_f32) ((float*)e.out)[o] = x;
    else ((__half*)e.out)[o] = __float2half_rn(x);
  }
  }
}

// Tile order inside one batch entry.  m fastest: CTAs running side by side share the B tile (right when B is the big
// operand).  n fastest (p.n_fastest): they share the A tile and sweep B -- right when B is a weight matrix that stays
// in L2 anyway and A is a large activation (FC2 of the encoder: A = 123 MB would otherwise be re-read per n tile).
__device__ __forceinline__ void tile_decode(const GemmKParams& p, int t, int tiles_m, int tiles_n, int& tile_m, int& tile_n, int& zz) {
  if (p.n_fastest) {
    tile_n = t % tiles_n;
    const int r = t / tiles_n;
    tile_m = r % tiles_m;
    zz = r / tiles_m;
  } else {
    tile_m = t % tiles_m;
    const int r = t / tiles_m;
    tile_n = r % tiles_n;
    zz = r / tiles_n;
  }
}

// Epilogue staging: each consumer warpgroup turns its register accumulator into a row per thread through shared memory,
// EPI_CH columns at a time, so that the epilogue stores whole 16-byte pieces of one output row.
template <int BN>
struct EpiStage {
  static constexpr int CH = BN < 64 ? BN : 64;   // columns per staged chunk
  static constexpr int LD = CH + 4;              // padded row pitch (floats): conflict-free float4 reads
  static constexpr int BYTES = 2 * 64 * LD * 4;  // both consumer warpgroups
};
template <int BN, int STAGES>
__host__ __device__ constexpr int gemm_smem_bytes() { return STAGES * (A_STAGE_BYTES + BN * BK * 2) + EpiStage<BN>::BYTES + 1024 + 512; }

// Where tile t's operands and output sit: tile (tile_m, tile_n) of batch entry (i1, i2).
struct TileCoord {
  int tile_m, tile_n, i1, i2;
};
__device__ __forceinline__ TileCoord tile_coord(const GemmKParams& p, int t, int tiles_m, int tiles_n) {
  TileCoord c;
  int z;
  tile_decode(p, t, tiles_m, tiles_n, c.tile_m, c.tile_n, z);
  c.i1 = z % p.zn1;
  c.i2 = z / p.zn1;
  return c;
}

// TMA producer (one elected thread): fills the stage ring with the k-blocks of this CTA's tiles t = blockIdx.x,
// blockIdx.x + gridDim.x, ... in that order, each stage once its consumers have handed it back.
template <int BN, int STAGES>
__device__ __forceinline__ void gemm_produce(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmKParams& p, uint8_t* sA,
                                             uint8_t* sB, uint64_t* full, uint64_t* empty, int tiles_m, int tiles_n,
                                             int total_tiles, int total_kb) {
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  int stage = 0;
  uint32_t phase = 0;
  bool first = true;
  // coordinate slot s (1..3) of a tensor map holds whichever of (row, i1, i2) was sorted there
  auto slot = [](const int (&pos)[3], int s, int row, int j1, int j2) {
    return pos[0] == s ? row : (pos[1] == s ? j1 : (pos[2] == s ? j2 : 0));
  };
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const TileCoord tc = tile_coord(p, t, tiles_m, tiles_n);
    const int a1 = p.a_batched ? tc.i1 : 0, a2 = p.a_batched ? tc.i2 : 0;
    const int b1 = p.b_batched ? tc.i1 : 0, b2 = p.b_batched ? tc.i2 : 0;
    const int ca1 = slot(p.a_pos, 1, tc.tile_m * BM, a1, a2), ca2 = slot(p.a_pos, 2, tc.tile_m * BM, a1, a2),
              ca3 = slot(p.a_pos, 3, tc.tile_m * BM, a1, a2);
    const int cb1 = slot(p.b_pos, 1, tc.tile_n * BN, b1, b2), cb2 = slot(p.b_pos, 2, tc.tile_n * BN, b1, b2),
              cb3 = slot(p.b_pos, 3, tc.tile_n * BN, b1, b2);
    if (first) {
      if (blockIdx.x == 0) tl_stamp_any(TL_GEMM, 0);
      pdl_wait();
      if (blockIdx.x == 0) tl_stamp_any(TL_GEMM, 1);
      first = false;
    }
    for (int kb = 0; kb < total_kb; ++kb) {
      const int k0 = kb * BK;
      mbar_wait(&empty[stage], phase ^ 1);
      mbar_expect_tx(&full[stage], A_STAGE_BYTES + B_STAGE_BYTES);
      tma_load_4d(sA + stage * A_STAGE_BYTES, tmA, &full[stage], k0, ca1, ca2, ca3);
      tma_load_4d(sB + stage * B_STAGE_BYTES, tmB, &full[stage], k0, cb1, cb2, cb3);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  }
}

// Epilogue of 64 tile rows (m0 .. m0 + 63) held by one consumer warpgroup as a 64 x BN accumulator fragment: through the
// warpgroup's staging buffer, ES::CH columns at a time, so that each thread stores whole 16-byte pieces of one output row.
// bar_id: the warpgroup's own named barrier (128 threads).
template <int BN, int KIND>
__device__ __forceinline__ void epilogue_rows64(const GemmKParams& p, const float (&acc)[BN / 2], float* stg, int bar_id, long m0,
                                                int n0, int i1, int i2) {
  using ES = EpiStage<BN>;
  const int tw = threadIdx.x & 127;
  const int row = tw & 63, half = tw >> 6;
#pragma unroll
  for (int ch = 0; ch < BN / ES::CH; ++ch) {
    wgmma_acc_foreach(acc, [&](int r, int c, float v) {
      if (c >= ch * ES::CH && c < (ch + 1) * ES::CH) stg[r * ES::LD + c - ch * ES::CH] = v;
    });
    named_bar_sync(bar_id, 128);
    constexpr int CNT = ES::CH / 2;
    uint32_t v[CNT];
    const float4* src = reinterpret_cast<const float4*>(stg + row * ES::LD + half * CNT);
#pragma unroll
    for (int i = 0; i < CNT / 4; ++i) {
      const float4 q = src[i];
      v[4 * i] = __float_as_uint(q.x); v[4 * i + 1] = __float_as_uint(q.y);
      v[4 * i + 2] = __float_as_uint(q.z); v[4 * i + 3] = __float_as_uint(q.w);
    }
    named_bar_sync(bar_id, 128);   // the next chunk reuses the staging buffer
    epilogue_chunk<CNT, KIND>(p, m0 + row, n0 + ch * ES::CH + half * CNT, v, i1, i2);
  }
}

// Persistent: each CTA walks tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...  (tile_m fastest, so CTAs
// running side by side share the B (weight) tile in L2).
// CTA = 384 threads: warp 0 TMA producer (warps 1-3 idle), warpgroups 1 and 2 the wgmma consumers of tile rows 0-63 and
// 64-127, each keeping its 64 x BN fp32 accumulator in registers and running the epilogue of its rows.
template <int BN, int STAGES, int MIN_CTAS, int KIND>
__global__ void __launch_bounds__(384, MIN_CTAS)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ GemmKParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // pointer arithmetic keeps the shared address space (LDS/STS)
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  using ES = EpiStage<BN>;
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * A_STAGE_BYTES;
  float* stg_all = reinterpret_cast<float*>(sB + STAGES * B_STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg_all) + ES::BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = (p.N + BN - 1) / BN;
  const int total_tiles = tiles_m * tiles_n * p.nz;
  const int total_kb = (p.K + BK - 1) / BK;
  pdl_trigger();

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && elect_one()) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) gemm_produce<BN, STAGES>(&tmA, &tmB, p, sA, sB, full, empty, tiles_m, tiles_n, total_tiles, total_kb);
  } else if (warp >= 4) {
    const int wg = (warp >> 2) - 1;                  // consumer warpgroup: tile rows 64 wg .. 64 wg + 63
    float* stg = stg_all + wg * 64 * ES::LD;
    int stage = 0;
    uint32_t phase = 0;
    pdl_wait();   // the residual / output buffers belong to the preceding kernels
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const TileCoord tc = tile_coord(p, t, tiles_m, tiles_n);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < total_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        wgmma_tile_k64<BN>(acc, sA + stage * A_STAGE_BYTES, sB + stage * B_STAGE_BYTES, wg, kb > 0);
        wgmma_commit();
        // one k-block of MMAs stays in flight; the stage read by the one before it is handed back to the producer
        wgmma_wait<1>();
        if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty[prev]);
      epilogue_rows64<BN, KIND>(p, acc, stg, 1 + wg, (long)tc.tile_m * BM + wg * 64, tc.tile_n * BN, tc.i1, tc.i2);
    }
  }
}

// Ping-pong variant for problems with at least two 128 x 128 tiles per CTA.  Each consumer warpgroup owns whole tiles:
// warpgroup c takes tiles j = c, c + 2, c + 4, ... of the CTA's sequence t_j = blockIdx.x + j gridDim.x, so while one
// runs its epilogue the other keeps the tensor cores busy.  An ordered pair of named barriers (PP_BAR + c) hands the
// math phase from one warpgroup to the other: the producer fills the ring in tile order, and a warpgroup may only wait
// on a stage's `full` barrier once every earlier use of that stage has been consumed.  Every output element sees the
// same m64n128k16 sequence and the same epilogue arithmetic as in gemm_tn_kernel<128, ..>: the results are identical.
// Registers: the producer warpgroup drops to PP_PRODUCER_REGS, the consumers (2 x 64 accumulators a thread) rise to
// PP_CONSUMER_REGS; 128 x 40 + 256 x 232 <= 64 K.
constexpr int PP_STAGES = 5;   // 5 x 32 KB ring + 2 x 17 KB staging: the most that fits 227 KB
constexpr int PP_BAR = 4;      // named barriers 4, 5 (1, 2: per-warpgroup epilogue staging)
constexpr int PP_PRODUCER_REGS = 40, PP_CONSUMER_REGS = 232;

template <int KIND>
__global__ void __launch_bounds__(384, 1)
gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ GemmKParams p) {
  constexpr int BN = 128, STAGES = PP_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  using ES = EpiStage<BN>;
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * A_STAGE_BYTES;
  float* stg_all = reinterpret_cast<float*>(sB + STAGES * B_STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg_all) + ES::BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = (p.N + BN - 1) / BN;
  const int total_tiles = tiles_m * tiles_n * p.nz;
  const int total_kb = (p.K + BK - 1) / BK;
  pdl_trigger();

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && elect_one()) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);   // one arrival per warp of the warpgroup that consumed the stage
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<PP_PRODUCER_REGS>();
    if (warp == 0 && elect_one())
      gemm_produce<BN, STAGES>(&tmA, &tmB, p, sA, sB, full, empty, tiles_m, tiles_n, total_tiles, total_kb);
    return;
  }
  setmaxnreg_inc<PP_CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;
  float* stg = stg_all + wg * 64 * ES::LD;
  pdl_wait();   // the residual / output buffers belong to the preceding kernels
  if (wg == 1) named_bar_arrive(PP_BAR, 256);   // warpgroup 0 takes the first tile (grid <= tiles: it exists)
  for (int j = wg, t = blockIdx.x + wg * gridDim.x; t < total_tiles; j += 2, t += 2 * gridDim.x) {
    const TileCoord tc = tile_coord(p, t, tiles_m, tiles_n);
    // every tile has total_kb k-blocks: tile j starts at ring position j * total_kb
    const long it0 = (long)j * total_kb;
    int stage = (int)(it0 % STAGES);
    uint32_t phase = (uint32_t)((it0 / STAGES) & 1);
    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
    named_bar_sync(PP_BAR + wg, 256);   // our turn: the other warpgroup has issued all MMAs of tile j - 1
    int prev = -1;
    for (int kb = 0; kb < total_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      wgmma_fence();
      wgmma_tile_k64<BN>(acc[0], sA + stage * A_STAGE_BYTES, sB + stage * B_STAGE_BYTES, 0, kb > 0);
      wgmma_tile_k64<BN>(acc[1], sA + stage * A_STAGE_BYTES, sB + stage * B_STAGE_BYTES, 1, kb > 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if (t + gridDim.x < total_tiles) named_bar_arrive(PP_BAR + (wg ^ 1), 256);   // tile j + 1 may start its MMAs
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty[prev]);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      epilogue_rows64<BN, KIND>(p, acc[h], stg, 1 + wg, (long)tc.tile_m * BM + h * 64, tc.tile_n * BN, tc.i1, tc.i2);
  }
}

// ------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  });
  WL_CHECK(fn != nullptr, WL_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  return fn;
}

struct TmapKey {
  const void* ptr;
  long rows, k, ld, s1, s2;
  int n1, n2, box_rows, box_k;
  bool operator<(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) < 0; }
};

// Tensor map + where the (row, i1, i2) coordinates sit among its dims 1..3.  TMA wants strides in
// ascending order (each a multiple of the previous), so the view's dims are sorted by stride: e.g. the
// per-head Q/K operand of attention is {k, head (128 B), row (2*ld B), batch}.
static TmapInfo get_tmap(const GemmOperand& op, int box_rows, int box_k = BK);
TmapInfo make_tmap(const GemmOperand& op, int box_rows, int box_k) { return get_tmap(op, box_rows, box_k); }

static TmapInfo get_tmap(const GemmOperand& op, int box_rows, int box_k) {
  static std::map<TmapKey, TmapInfo> cache;
  static std::mutex mu;
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = op.ptr; key.rows = op.rows; key.k = op.k; key.ld = op.ld; key.s1 = op.s1; key.s2 = op.s2;
  key.n1 = op.n1; key.n2 = op.n2; key.box_rows = box_rows; key.box_k = box_k;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  WL_CHECK(((uintptr_t)op.ptr & 15) == 0, WL_ERR_ARG, "GEMM operand pointer must be 16-byte aligned");
  struct D { long size, stride; int role; };
  std::vector<D> real, single;
  const D all[3] = {{op.rows, op.ld, 0}, {op.n1, op.s1, 1}, {op.n2, op.s2, 2}};
  for (const D& d : all) ((d.role == 0 || d.size > 1) ? real : single).push_back(d);
  std::stable_sort(real.begin(), real.end(), [](const D& x, const D& y) { return x.stride < y.stride; });
  std::vector<D> order = real;
  for (D d : single) {
    d.stride = order.back().stride * order.back().size;
    order.push_back(d);
  }
  TmapInfo info;
  cuuint64_t dims[4] = {(cuuint64_t)op.k, 1, 1, 1};
  cuuint64_t strides[3];
  cuuint32_t box[4] = {(cuuint32_t)box_k, 1, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 3; ++i) {
    WL_CHECK(order[i].stride > 0 && (order[i].stride * 2) % 16 == 0, WL_ERR_ARG,
             "GEMM operand stride %ld elements (dim role %d) is not a positive multiple of 16 bytes", order[i].stride, order[i].role);
    dims[1 + i] = (cuuint64_t)order[i].size;
    strides[i] = (cuuint64_t)order[i].stride * 2;
    if (order[i].role == 0) box[1 + i] = (cuuint32_t)box_rows;
    info.pos[order[i].role] = 1 + i;
  }
  CUresult r = encode_fn()(&info.tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)op.ptr, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  WL_CHECK(r == CUDA_SUCCESS, WL_ERR_CUDA,
           "cuTensorMapEncodeTiled failed (%d) dims={%llu,%llu,%llu,%llu} strides={%llu,%llu,%llu} box_rows=%d", (int)r,
           (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
           (unsigned long long)strides[0], (unsigned long long)strides[1], (unsigned long long)strides[2], box_rows);
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, info);
  return info;
}

static int num_sms() {
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  return sms;
}

template <int BN, int STAGES, int MIN_CTAS, int KIND>
static void launch_cfg(cudaStream_t stream, const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, int Z) {
  constexpr int smem = gemm_smem_bytes<BN, STAGES>();
  GemmKParams q = p;
  q.nz = Z;
  const long tiles = (long)cdiv(p.N, BN) * cdiv(p.M, BM) * Z;
  const int grid = (int)std::min<long>(tiles, (long)num_sms() * MIN_CTAS);
  launch_kernel(gemm_tn_kernel<BN, STAGES, MIN_CTAS, KIND>, dim3(grid), dim3(384), (size_t)smem, stream, ta, tb, q);
  g_gemm_launches++;
}

template <int KIND>
static void launch_pingpong(cudaStream_t stream, const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, int Z) {
  constexpr int smem = gemm_smem_bytes<128, PP_STAGES>();
  GemmKParams q = p;
  q.nz = Z;
  const long tiles = (long)cdiv(p.N, 128) * cdiv(p.M, BM) * Z;
  const int grid = (int)std::min<long>(tiles, num_sms());
  launch_kernel(gemm_pingpong_kernel<KIND>, dim3(grid), dim3(384), (size_t)smem, stream, ta, tb, q);
  g_gemm_launches++;
}

template <int BN, int STAGES, int MIN_CTAS, int KIND>
static void prime_cfg() {
  constexpr int smem = gemm_smem_bytes<BN, STAGES>();
  WL_CUDA(cudaFuncSetAttribute(gemm_tn_kernel<BN, STAGES, MIN_CTAS, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}

// opt-in shared memory sizes must be set outside stream capture: done once from wl_init
template <int KIND>
static void prime_kind() {
  prime_cfg<16, 8, 1, KIND>();
  prime_cfg<32, 8, 1, KIND>();
  prime_cfg<64, 6, 1, KIND>();
  prime_cfg<128, 5, 1, KIND>();
}
void gemm_tl_bind(unsigned long long* p) { tl_bind_tu(p); }
template <int KIND>
static void prime_pingpong() {
  constexpr int smem = gemm_smem_bytes<128, PP_STAGES>();
  WL_CUDA(cudaFuncSetAttribute(gemm_pingpong_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}
void gemm_prime() {
  prime_kind<EPI_ROW>();
  prime_kind<EPI_COL>();
  prime_kind<EPI_HEADSPLIT>();
  prime_pingpong<EPI_ROW>();
  prime_pingpong<EPI_COL>();
  prime_pingpong<EPI_HEADSPLIT>();
}

template <int KIND>
static void launch_kind(int bn, cudaStream_t stream, const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, int Z) {
  switch (bn) {
    case 16: launch_cfg<16, 8, 1, KIND>(stream, ta, tb, p, Z); break;
    case 32: launch_cfg<32, 8, 1, KIND>(stream, ta, tb, p, Z); break;
    case 64: launch_cfg<64, 6, 1, KIND>(stream, ta, tb, p, Z); break;
    case 128: launch_cfg<128, 5, 1, KIND>(stream, ta, tb, p, Z); break;
    default: WL_CHECK(false, WL_ERR_ARG, "unsupported BN %d", bn);
  }
}

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

static GemmKParams make_params(const GemmOperand& A, const GemmOperand& B, int M, int N, int K, const GemmEpilogue& epi,
                               int* Z) {
  WL_CHECK(M > 0 && N > 0 && K > 0, WL_ERR_ARG, "gemm_tn: empty problem %dx%dx%d", M, N, K);
  const int za = A.n1 * A.n2, zb = B.n1 * B.n2;
  WL_CHECK(za == 1 || zb == 1 || (A.n1 == B.n1 && A.n2 == B.n2), WL_ERR_ARG, "gemm_tn: batch shapes differ");
  GemmKParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.a_batched = za > 1; p.b_batched = zb > 1;
  p.zn1 = za > 1 ? A.n1 : B.n1;
  *Z = za > zb ? za : zb;
  p.e = epi;
  p.vec_ok = 0;
  // B (N x K halves) small enough to live in L2 while A is larger than B: sweep n fastest
  p.n_fastest = (zb == 1 && (long)N * K * 2 <= (24L << 20) && (long)M * K > (long)N * K) ? 1 : 0;
  if (epi.mode == GEMM_STORE && epi.ldn == 1) {
    const int a = epi.out_f32 ? 4 : 8;  // elements per 16 bytes
    bool ok = ((uintptr_t)epi.out & 15) == 0 && epi.ldm % 8 == 0 && epi.ob1 % 8 == 0 && epi.ob2 % 8 == 0;
    (void)a;
    if (epi.bias && !epi.bias_on_m) ok = ok && ((uintptr_t)epi.bias & 15) == 0;
    if (epi.resid)
      ok = ok && epi.rldn == 1 && ((uintptr_t)epi.resid & 15) == 0 && epi.rldm % 4 == 0 && epi.rb1 % 4 == 0 && epi.rb2 % 4 == 0;
    p.vec_ok = ok ? 1 : 0;
  }
  if (epi.mode == GEMM_HEADSPLIT) {
    WL_CHECK(!epi.out_f32 && !epi.gelu && !epi.relu && !epi.resid && !epi.bias_on_m && N % 64 == 0 && epi.hs_slots, WL_ERR_ARG,
             "gemm_tn: bad head-split epilogue");
  }
  return p;
}

static int pick_bn(int N) {
  static const int force_bn = env_int("WLB200_BN", 0);
  if (force_bn) return force_bn;
  if (N <= 16) return 16;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  return 128;   // 64 x 128 fp32 accumulator per consumer warpgroup = 64 registers a thread
}

// Ping-pong only pays when each CTA has a second tile whose MMAs can hide the first one's epilogue.
static bool pingpong_pays(int bn, long tiles) { return bn == 128 && tiles >= 2L * num_sms(); }

GemmVariant gemm_tn_variant(int M, int N, int K, int Z) {
  (void)K;
  const int bn = pick_bn(N);
  return pingpong_pays(bn, (long)cdiv(M, BM) * cdiv(N, bn) * Z) ? GEMM_PINGPONG : GEMM_CLASSIC;
}

void gemm_tn(cudaStream_t stream, const GemmOperand& A, const GemmOperand& B, int M, int N, int K, const GemmEpilogue& epi,
             GemmVariant variant) {
  int Z;
  GemmKParams p = make_params(A, B, M, N, K, epi, &Z);
  int bn = pick_bn(N);
  if (epi.mode == GEMM_HEADSPLIT && bn < 64) bn = 64;
  const TmapInfo ia = get_tmap(A, BM), ib = get_tmap(B, bn);
  const CUtensorMap& ta = ia.tm;
  const CUtensorMap& tb = ib.tm;
  for (int i = 0; i < 3; ++i) { p.a_pos[i] = ia.pos[i]; p.b_pos[i] = ib.pos[i]; }
  bool pingpong = pingpong_pays(bn, (long)cdiv(M, BM) * cdiv(N, bn) * Z);
  if (variant != GEMM_AUTO) {
    WL_CHECK(variant == GEMM_CLASSIC || bn == 128, WL_ERR_ARG, "gemm_tn: the ping-pong kernel needs N tiles of 128");
    pingpong = variant == GEMM_PINGPONG;
  }
  if (pingpong) {
    if (epi.mode == GEMM_HEADSPLIT) launch_pingpong<EPI_HEADSPLIT>(stream, ta, tb, p, Z);
    else if (p.vec_ok) launch_pingpong<EPI_ROW>(stream, ta, tb, p, Z);
    else launch_pingpong<EPI_COL>(stream, ta, tb, p, Z);
  } else if (epi.mode == GEMM_HEADSPLIT) launch_kind<EPI_HEADSPLIT>(bn, stream, ta, tb, p, Z);
  else if (p.vec_ok) launch_kind<EPI_ROW>(bn, stream, ta, tb, p, Z);
  else launch_kind<EPI_COL>(bn, stream, ta, tb, p, Z);
}

// ------------------------------------------------------------------------------------ SIMT reference
__global__ void gemm_tn_simt_kernel(GemmOperand A, GemmOperand B, GemmKParams p) {
  const long n = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const long m = blockIdx.y;
  const int z = blockIdx.z;
  if (n >= p.N) return;
  const int i1 = z % p.zn1, i2 = z / p.zn1;
  const __half* a = A.ptr + (p.a_batched ? (long)i1 * A.s1 + (long)i2 * A.s2 : 0) + m * A.ld;
  const __half* b = B.ptr + (p.b_batched ? (long)i1 * B.s1 + (long)i2 * B.s2 : 0) + n * B.ld;
  float acc = 0.f;
  const int ka = (int)(A.k < p.K ? A.k : p.K), kb = (int)(B.k < p.K ? B.k : p.K);
  const int kk = ka < kb ? ka : kb;
  for (int k = 0; k < kk; ++k) acc = fmaf(__half2float(a[k]), __half2float(b[k]), acc);
  uint32_t v[1] = {__float_as_uint(acc)};
  GemmKParams q = p;
  q.vec_ok = 0;
  if (q.e.mode == GEMM_HEADSPLIT) {
    const GemmEpilogue& e = q.e;
    const int bb = (int)(m / e.hs_S), s = (int)(m % e.hs_S);
    float x = acc + (e.bias ? e.bias[n] : 0.f);
    ((__half*)e.out)[(long)e.hs_slots[bb] * e.hs_slot_stride + ((long)(n >> 6) * e.hs_S + s) * 64 + (((((int)n & 63) >> 3) ^ (s & 7)) << 3) + (n & 7)] = __float2half_rn(x);
    return;
  }
  epilogue_chunk<1, EPI_COL>(q, m, (int)n, v, i1, i2);
}

void gemm_tn_simt(cudaStream_t stream, const GemmOperand& A, const GemmOperand& B, int M, int N, int K, const GemmEpilogue& epi) {
  int Z;
  GemmKParams p = make_params(A, B, M, N, K, epi, &Z);
  dim3 grid(cdiv(N, 128), M, Z);
  gemm_tn_simt_kernel<<<grid, 128, 0, stream>>>(A, B, p);
  WL_CUDA(cudaGetLastError());
  g_gemm_launches++;
}

}  // namespace wl
