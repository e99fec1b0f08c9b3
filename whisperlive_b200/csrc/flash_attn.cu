// K5: fused encoder self-attention on wgmma -- scores never leave the SM.
//   one CTA = 128 queries of one (stream, head); loop over 12 key tiles of 128:
//     S = Q K^T            wgmma m64n128k16 x4, Q and K from shared memory, S in registers
//     online softmax       in registers (a row's 128 scores are spread over the 4 threads of a quad)
//     O += P V             wgmma m64n64k16 x8 with P as the register A operand (fp16): the S accumulator fragment is
//                          already laid out as the A fragment, so P never goes through shared memory
//   warp 0: TMA producer (Q once, K / V^T tiles through a 4-stage mbarrier ring); warpgroups 1 and 2: query rows 0-63 and
//   64-127, each with its own running (max, sum, O).
#include <cstdlib>

#include "gemm.cuh"
#include "kernels.cuh"

namespace wl {

constexpr int FA_BQ = 128, FA_BK = 128, FA_STAGES = 4;
constexpr int FA_Q_BYTES = FA_BQ * 128;              // 128 rows x 64 halves
constexpr int FA_K_BYTES = FA_BK * 128;              // 128 keys x 64 halves
constexpr int FA_V_BYTES = 2 * 64 * 128;             // two k-blocks of [64 dd][64 keys]
constexpr int FA_STAGE_BYTES = FA_K_BYTES + FA_V_BYTES;
constexpr int FA_SMEM = 1024 + FA_Q_BYTES + FA_STAGES * FA_STAGE_BYTES + 256;
constexpr int FA_NT = (S_ENC + FA_BK - 1) / FA_BK;   // 12 key tiles

struct FaParams {
  int q_pos[3], k_pos[3], v_pos[3];
  __half* out;   // [B*1500][d]
  int d;
  float scale_log2;  // softmax scale * log2(e)
};

__device__ __forceinline__ float fa_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void fa_coords(int (&c)[4], const int (&pos)[3], int k0, int row, int i1, int i2) {
  c[0] = k0; c[1] = c[2] = c[3] = 0;
  c[pos[0]] = row; c[pos[1]] = i1; c[pos[2]] = i2;
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(384, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, const __grid_constant__ FaParams p) {
  extern __shared__ uint8_t fa_raw[];
  uint8_t* base = fa_raw + ((1024u - (smem_u32(fa_raw) & 1023u)) & 1023u);   // pointer arithmetic keeps the shared address space (LDS/STS)
  uint8_t* sQ = base;
  uint8_t* sKV = sQ + FA_Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + FA_STAGES * FA_STAGE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [FA_STAGES]
  uint64_t* kv_empty = kv_full + FA_STAGES;     // [FA_STAGES]

  const int warp = threadIdx.x >> 5;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  if (warp == 1 && elect_one()) {
    mbar_init(q_full, 1);
    for (int i = 0; i < FA_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }   // one arrival per consumer warp
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) {
      int c[4];
      mbar_expect_tx(q_full, FA_Q_BYTES);
      fa_coords(c, p.q_pos, 0, qt * FA_BQ, h, b);
      tma_load_4d(sQ, &tmQ, q_full, c[0], c[1], c[2], c[3]);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < FA_NT; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        uint8_t* sk = sKV + stage * FA_STAGE_BYTES;
        mbar_expect_tx(&kv_full[stage], FA_STAGE_BYTES);
        fa_coords(c, p.k_pos, 0, j * FA_BK, h, b);
        tma_load_4d(sk, &tmK, &kv_full[stage], c[0], c[1], c[2], c[3]);
        fa_coords(c, p.v_pos, j * FA_BK, 0, h, b);
        tma_load_4d(sk + FA_K_BYTES, &tmV, &kv_full[stage], c[0], c[1], c[2], c[3]);
        fa_coords(c, p.v_pos, j * FA_BK + 64, 0, h, b);
        tma_load_4d(sk + FA_K_BYTES + 64 * 128, &tmV, &kv_full[stage], c[0], c[1], c[2], c[3]);
        if (++stage == FA_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // Thread (warp w of the warpgroup, lane l) holds query rows 16 w + l / 4 and 16 w + l / 4 + 8 of its warpgroup's
    // 64, and of each 8-column group the columns 2 (l % 4), 2 (l % 4) + 1 (see wgmma_acc_foreach).
    const int wg = (warp >> 2) - 1, lane = lane_id();
    const uint64_t qdesc = wgmma_desc_sw128(smem_u32(sQ + wg * 64 * 128));
    float o[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // m in the scaled log2 domain; l: this thread's share
    mbar_wait(q_full, 0);
#pragma unroll 1
    for (int j = 0; j < FA_NT; ++j) {
      const int st = j % FA_STAGES;
      mbar_wait(&kv_full[st], (uint32_t)(j / FA_STAGES) & 1u);
      const uint8_t* sk = sKV + st * FA_STAGE_BYTES;
      float s[64];
      const uint64_t kdesc = wgmma_desc_sw128(smem_u32(sk));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<FA_BK>(s, qdesc + (uint64_t)(2 * k), kdesc + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      // Only the 12th key tile is ragged (1500 = 11 x 128 + 92): keys beyond the sequence get probability 0.
      const int nvalid = S_ENC - j * FA_BK;
      if (nvalid < FA_BK) {
#pragma unroll
        for (int e = 0; e < 64; ++e)
          if (8 * (e >> 2) + 2 * (lane & 3) + (e & 1) >= nvalid) s[e] = -INFINITY;
      }
      float alpha[2], neg_mx[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * i], s[4 * c + 2 * i + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float mn = fmaxf(m[i], mx * p.scale_log2);
        alpha[i] = (m[i] == -INFINITY) ? 0.f : fa_exp2(m[i] - mn);
        m[i] = mn;
        neg_mx[i] = -mn;
      }
      // probabilities, packed straight into the A fragments of P V (k-step kk = keys 16 kk .. 16 kk + 15)
      uint32_t pa[8][4];
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {   // r: (row half i = r & 1, column group 2 kk + (r >> 1))
          const int e = 8 * kk + 2 * r, i = r & 1;
          const float p0 = fa_exp2(fmaf(s[e], p.scale_log2, neg_mx[i]));
          const float p1 = fa_exp2(fmaf(s[e + 1], p.scale_log2, neg_mx[i]));
          sum[i] += p0 + p1;
          pa[kk][r] = pack_half2(p0, p1);
        }
      }
#pragma unroll
      for (int e = 0; e < 32; ++e) o[e] *= alpha[(e >> 1) & 1];
      l[0] = l[0] * alpha[0] + sum[0];
      l[1] = l[1] * alpha[1] + sum[1];
      const uint64_t vdesc = wgmma_desc_sw128(smem_u32(sk + FA_K_BYTES));
      wgmma_fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_rs_n64(o, pa[kk], vdesc + (uint64_t)((kk >> 2) * (64 * 128 >> 4) + (kk & 3) * 2), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (lane == 0) mbar_arrive(&kv_empty[st]);   // this warp's reads of the K / V stage are complete
    }
    float inv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float t = l[i];
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      inv[i] = 1.f / t;
    }
    const int r0 = qt * FA_BQ + wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int qrow = r0 + 8 * i;
      if (qrow < S_ENC) {
        __half* dst = p.out + ((long)b * S_ENC + qrow) * p.d + h * 64 + 2 * (lane & 3);
#pragma unroll
        for (int c = 0; c < 8; ++c)
          *reinterpret_cast<__half2*>(dst + 8 * c) = __floats2half2_rn(o[4 * c + 2 * i] * inv[i], o[4 * c + 2 * i + 1] * inv[i]);
      }
    }
  }
}

void flash_attn_prime() {
  WL_CUDA(cudaFuncSetAttribute(flash_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
}

// qk: [nb][1500][2d] fp16 (q | k), vt: [nb][d][S_PAD] fp16 (V transposed per head), out: [nb*1500][d] fp16
void encoder_attention_fused(cudaStream_t st, const __half* qk, const __half* vt, __half* out, int nb, int H, int d) {
  GemmOperand q, k, v;
  q.ptr = qk; q.rows = S_ENC; q.k = 64; q.ld = 2L * d; q.n1 = H; q.s1 = 64; q.n2 = nb; q.s2 = (long)S_ENC * 2 * d;
  k = q;
  k.ptr = qk + d;
  v.ptr = vt; v.rows = 64; v.k = S_PAD; v.ld = S_PAD; v.n1 = H; v.s1 = 64L * S_PAD; v.n2 = nb; v.s2 = (long)d * S_PAD;
  const TmapInfo iq = make_tmap(q, FA_BQ), ik = make_tmap(k, FA_BK), iv = make_tmap(v, 64);
  FaParams p;
  for (int i = 0; i < 3; ++i) { p.q_pos[i] = iq.pos[i]; p.k_pos[i] = ik.pos[i]; p.v_pos[i] = iv.pos[i]; }
  p.out = out; p.d = d;
  p.scale_log2 = 0.125f * 1.4426950408889634f;
  dim3 grid(FA_NT, H, nb);
  flash_attn_kernel<<<grid, 384, FA_SMEM, st>>>(iq.tm, ik.tm, iv.tm, p);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

}  // namespace wl
