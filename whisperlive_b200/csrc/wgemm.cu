// Small-batch decode GEMM (K9, R <= 32 decoder rows): Y[R, n_out] = X[R, K] * W[n_out, K]^T with the epilogue fused.
//
// At 4-8 streams per GPU (the 8-GPU point of the scaling series) a decode linear layer is a 3-13 MB weight stream and
// a few MFLOP; what it costs is its place on the dependency chain of the token step.  This kernel is built for that:
//   * the CTA's whole weight slice (NF output features x <= 1280 of K, <= 105 KB) is requested with cp.async.bulk
//     BEFORE griddepcontrol.wait, i.e. while the kernel that produces X is still running; after the wait the only
//     global traffic on the critical path is X itself (16 rows x K fp16, an L2 hit);
//   * warp-level mma.sync m16n8k16 (M = the 16 decoder rows, N = 8 output features): no warpgroup MMA, no tensor
//     maps, no mbarrier ring -- and about 3 KB of SASS (the decode step's launches are instruction-fetch bound, see
//     dec_gemm.cu); the 128-row wgmma tiles would be 87 % padding at 16 rows;
//   * the 8 warps split K, reduce through shared memory in a fixed order (bit-reproducible), and the epilogue writes
//     FINAL values: + bias, + residual (in place), GELU -> fp16, or a raw partial sum when K is split over CTAs
//     (FC2, K = 4d) -- so LayerNorm, self- and cross-attention read one value instead of summing 4-8 partials,
//     and the GELU-cast kernel disappears.
// k is permuted inside every 32-wide chunk so that both operands are read with 16-byte accesses: lane (g, tq) takes
// X[row g / g+8][k0 + 8 tq .. +8) and W[feature g][k0 + 8 tq .. +8); the two m16n8k16 steps of a chunk use halves
// {0,1 | 2,3} and {4,5 | 6,7} of those 8 values as the fragment's (k = 2tq, 2tq+1 | 2tq+8, 2tq+9) slots.  A permutation
// of k applied to both operands leaves the dot products unchanged.
#include <algorithm>
#include <atomic>
#include <cstdlib>

#include "gemm.cuh"
#include "kernels.cuh"

namespace wl {

static std::atomic<long> g_wgemm_launches{0};
long wgemm_launch_count() { return g_wgemm_launches.load(); }

constexpr int WG_WARPS = 8;
constexpr int WG_CH = 5;            // 32-wide k chunks per warp: K range per CTA <= 8 * 5 * 32 = 1280
constexpr int WG_MAX_NF = 40;       // output features per CTA

struct WgemmParams {
  const __half* W;     // [n_out][K]
  const __half* X;     // [R][K]
  const float* bias;   // [n_out] or null
  float* out_f32;      // mode 0: [R][n_out]; mode 1: x [R][n_out] updated in place; mode 3: [ksplit][R][n_out] partial sums
  __half* out_f16;     // mode 2: [R][n_out] gelu(acc + bias)
  long part_stride;    // mode 3: elements between K ranges
  int n_out, K, R, nf, kr, ksplit, mode;
};

__device__ __forceinline__ void mma_16816_f32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int MT>   // m16 tiles: 1 (R <= 16) or 2 (R <= 32)
__global__ void __launch_bounds__(WG_WARPS * 32) wgemm_kernel(const WgemmParams p) {
  extern __shared__ uint8_t wg_smem_raw[];
  uint8_t* base = wg_smem_raw + ((128u - (smem_u32(wg_smem_raw) & 127u)) & 127u);
  const int pitch = p.kr * 2 + 64;                        // bytes per weight row: = 64 mod 128 -> conflict-free 16-byte reads
  const int ntl = p.nf >> 3;                              // n-tiles (8 features) per CTA
  uint8_t* sW = base;                                     // [nf][pitch]
  float* red = reinterpret_cast<float*>(sW + p.nf * pitch);   // [8 warps][ntl][MT][16*8]
  uint64_t* bar = reinterpret_cast<uint64_t*>(red + WG_WARPS * ntl * MT * 128);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, tq = lane & 3;
  const int fgroup = blockIdx.x / p.ksplit, ks = blockIdx.x - fgroup * p.ksplit;
  const int f0 = fgroup * p.nf;
  const int nf = min(p.nf, p.n_out - f0);                 // multiple of 8 (host-checked)
  const int k0 = ks * p.kr;
  const int kr = min(p.kr, p.K - k0);
  const int nchunks = kr >> 5;
  pdl_trigger();
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (warp == 0 && elect_one()) {
    // weights: one bulk copy per feature row, all in flight before the dependency wait
    mbar_expect_tx(bar, (uint32_t)(nf * kr * 2));
#pragma unroll 1
    for (int f = 0; f < nf; ++f) bulk_load_1d(sW + f * pitch, p.W + (long)(f0 + f) * p.K + k0, (uint32_t)(kr * 2), bar);
  }
  // epilogue assignment without divisions: thread (er = tid / 16, fl = tid % 16) owns rows er (+16 with two m-tiles)
  // and features fl, fl + 16, fl + 32 (< nf) of the CTA's tile.  Their bias (a weight) is fetched before the dependency
  // wait and the residual right after it, so that the epilogue itself is shared-memory sums and one store each -- no
  // global round trip left at the end of the chain.
  constexpr int EF = (WG_MAX_NF + 15) / 16;
  const int er = tid >> 4, fl = tid & 15;
  float ebias[EF], eres[MT][EF];
#pragma unroll
  for (int i = 0; i < EF; ++i) {
    const int f = fl + 16 * i;
    ebias[i] = (f < nf && p.mode != 3 && p.bias != nullptr) ? __ldg(p.bias + f0 + f) : 0.f;
  }
  tl_stamp(TL_GEMM_PART, 0);
  pdl_wait();
  tl_stamp(TL_GEMM_PART, 1);
  // A fragments: this warp's chunks (c = warp, warp + 8, ...) of X, 16 bytes per (row, chunk) per lane
  uint4 xa[MT][WG_CH][2];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < WG_CH; ++i) {
      const int c = warp + i * WG_WARPS;
      const int r0 = mt * 16 + g, r1 = r0 + 8;
      const __half* xp = p.X + k0 + c * 32 + tq * 8;
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      xa[mt][i][0] = (c < nchunks && r0 < p.R) ? __ldcg(reinterpret_cast<const uint4*>(xp + (long)r0 * p.K)) : z;
      xa[mt][i][1] = (c < nchunks && r1 < p.R) ? __ldcg(reinterpret_cast<const uint4*>(xp + (long)r1 * p.K)) : z;
    }
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < EF; ++i) {
      const int f = fl + 16 * i, r = mt * 16 + er;
      eres[mt][i] = (p.mode == 1 && f < nf && r < p.R) ? __ldcg(p.out_f32 + (long)r * p.n_out + f0 + f) : 0.f;
    }
  mbar_wait(bar, 0);
  const int ntiles = nf >> 3;
#pragma unroll 1
  for (int nt = 0; nt < ntiles; ++nt) {
    float acc[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.f;
    const uint8_t* wrow = sW + (nt * 8 + g) * pitch + tq * 16;
#pragma unroll
    for (int i = 0; i < WG_CH; ++i) {
      const int c = warp + i * WG_WARPS;
      if (c < nchunks) {
        const uint4 wb = *reinterpret_cast<const uint4*>(wrow + c * 64);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma_16816_f32(acc[mt], xa[mt][i][0].x, xa[mt][i][1].x, xa[mt][i][0].y, xa[mt][i][1].y, wb.x, wb.y);
          mma_16816_f32(acc[mt], xa[mt][i][0].z, xa[mt][i][1].z, xa[mt][i][0].w, xa[mt][i][1].w, wb.z, wb.w);
        }
      }
    }
    // acc[mt] = D[row g | g+8][feature 2tq, 2tq+1] of this warp's K slice -> red[warp][nt][mt][row][feature]
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float* rp = red + ((warp * ntl + nt) * MT + mt) * 128;
      *reinterpret_cast<float2*>(rp + g * 8 + 2 * tq) = make_float2(acc[mt][0], acc[mt][1]);
      *reinterpret_cast<float2*>(rp + (g + 8) * 8 + 2 * tq) = make_float2(acc[mt][2], acc[mt][3]);
    }
  }
  __syncthreads();
  // fixed-order sum over the 8 warps + epilogue
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < EF; ++i) {
      const int f = fl + 16 * i, r = mt * 16 + er;
      if (f < nf && r < p.R) {
        const float* rp = red + (((f >> 3) * MT + mt) * 128) + er * 8 + (f & 7);
        float v = ebias[i];
#pragma unroll
        for (int w = 0; w < WG_WARPS; ++w) v += rp[w * ntl * MT * 128];
        const long o = (long)r * p.n_out + f0 + f;
        if (p.mode == 2) p.out_f16[o] = __float2half_rn(gelu_erf(v));
        else p.out_f32[(p.mode == 3 ? (long)ks * p.part_stride : 0L) + o] = v + eres[mt][i];
      }
    }
}

static int wg_smem_bytes(int MT, int nf = WG_MAX_NF, int kr = WG_WARPS * WG_CH * 32) {
  return 128 + nf * (kr * 2 + 64) + WG_WARPS * (nf / 8) * MT * 128 * 4 + 64;
}
void wgemm_tl_bind(unsigned long long* p) { tl_bind_tu(p); }
void wgemm_prime() {
  WL_CUDA(cudaFuncSetAttribute(wgemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_bytes(1)));
  WL_CUDA(cudaFuncSetAttribute(wgemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_bytes(2)));
}

bool wgemm_supported(int R, int K) { return R >= 1 && R <= 32 && K % 32 == 0; }

// K ranges of at most 1280 (a multiple of 32 each); 1 unless K > 1280
int wgemm_ksplit(int K) {
  const int cap = WG_WARPS * WG_CH * 32;
  return cdiv(K, cap);
}

// mode 0: out_f32 = acc + bias; 1: out_f32 += acc + bias (in place); 2: out_f16 = gelu(acc + bias);
// 3: out_f32[ks] = raw partial sum of K range ks (K > 1280: the consumer adds the ranges and the bias)
void wgemm(cudaStream_t st, const __half* W, int n_out, int K, const __half* X, int R, const float* bias, int mode, float* out_f32,
           __half* out_f16, long part_stride) {
  WL_CHECK(wgemm_supported(R, K) && n_out % 8 == 0, WL_ERR_ARG, "wgemm: unsupported problem R=%d n_out=%d K=%d", R, n_out, K);
  const int ksplit = wgemm_ksplit(K);
  WL_CHECK(ksplit == 1 || mode == 3, WL_ERR_ARG, "wgemm: K=%d needs %d K ranges: only the partial-sum epilogue supports that", K, ksplit);
  WL_CHECK(mode != 3 || ksplit <= 8, WL_ERR_ARG, "wgemm: too many K ranges");
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  WgemmParams p;
  p.W = W; p.X = X; p.bias = bias; p.out_f32 = out_f32; p.out_f16 = out_f16; p.part_stride = part_stride;
  p.n_out = n_out; p.K = K; p.R = R; p.ksplit = ksplit; p.mode = mode;
  // K range per CTA: equal ranges, multiples of 32
  p.kr = cdiv(cdiv(K, ksplit), 32) * 32;
  // features per CTA: the smallest multiple of 8 (<= 40) for which the grid fits one wave of one CTA per SM; the weight
  // slice of every CTA is then in flight before the dependency wait
  int nf = 8;
  while (nf < WG_MAX_NF && cdiv(n_out, nf) * ksplit > sms) nf += 8;
  p.nf = nf;
  const int grid = cdiv(n_out, nf) * ksplit;
  if (R <= 16) launch_kernel(wgemm_kernel<1>, dim3(grid), dim3(WG_WARPS * 32), (size_t)wg_smem_bytes(1, nf, p.kr), st, p);
  else launch_kernel(wgemm_kernel<2>, dim3(grid), dim3(WG_WARPS * 32), (size_t)wg_smem_bytes(2, nf, p.kr), st, p);
  g_wgemm_launches++;
}

}  // namespace wl
