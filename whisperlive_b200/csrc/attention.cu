// Decoder attention kernels (fp16 K/V storage, fp32 accumulation and softmax).
//   K10 decoder_self_attn : KV cache append + attention over <=448 positions with beam indirection, one warp per
//       (row, head), CUDA-core math (a few KB of work per warp).
//   K11 decoder_cross_attn: all rows (beams) of a stream against the stream's persistent encoder K/V -- persistent
//       CTAs, K/V streamed HBM -> smem by a producer warp (cp.async.bulk + mbarrier ring), consumed by 4 warps with
//       mma.sync on the pre-swizzled chunks; partial softmaxes per key range merged by a small combine kernel.
//   Reference call site of both: ctranslate2 Whisper.generate, transcriber_faster_whisper.py:1394-1407.
#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>

#include "kernels.cuh"

namespace wl {

// ============================================================================ K10 self attention
// One WARP per (row, head): at most 448 cached positions x 64 dims is far too little work for a thread block, and
// 2560 blocks (32 streams x beam 4 x 20 heads) would need several waves.  No block-level barriers: lanes own
// positions for the scores (one 128-byte K row each), dims for the weighted V sum (coalesced 128-byte V rows).
constexpr int SA_WARPS = 4;

template <bool PLAIN>   // PLAIN: q / k / v arrive as final values (wgemm path, batched prefill); else bias + <= 8 split-K partial sums
__global__ void __launch_bounds__(SA_WARPS * 32) self_attn_kernel(DecodeState s, PartialSrc qkv, __half* __restrict__ kc,
                                                                 __half* __restrict__ vc, long row_stride,
                                                                 __half* __restrict__ out, int H, int d, int R) {
  __shared__ float qs[SA_WARPS][64];
  __shared__ float vn_all[SA_WARPS][64];
  __shared__ float sc_all[SA_WARPS][T_MAX];
  __shared__ short ssrc_all[SA_WARPS][T_MAX];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * SA_WARPS + warp;
  pdl_trigger();
  if (item >= R * H) return;
  const int r = item / H, h = item % H;
  if (!s.active[r]) return;          // per-step state: written before this step's first kernel started
  const int pos = s.pos[r];
  const int n = pos + 1;
  float* q = qs[warp];
  float* vnew = vn_all[warp];
  float* sc = sc_all[warp];
  short* ssrc = ssrc_all[warp];
  // q / k / v of this (row, head), dims 2*lane and 2*lane+1: bias + the split-K partial sums, in range order
  const int c0 = h * 64 + 2 * lane;
  float2 qv = make_float2(0.f, 0.f), kv = qv, vv = qv;
  if (!PLAIN && qkv.bias) {
    qv = __ldg(reinterpret_cast<const float2*>(qkv.bias + c0));
    kv = __ldg(reinterpret_cast<const float2*>(qkv.bias + d + c0));
    vv = __ldg(reinterpret_cast<const float2*>(qkv.bias + 2 * d + c0));
  }
  // Everything about the CACHED positions (< pos) predates this decode step -- the indirection table was written by the
  // previous step's search kernel, the K/V rows by earlier steps (or, in the batched prefill, by the kernel before this
  // one) -- so it is fetched BEFORE the dependency wait: the table, the K row of position `lane` and the first eight
  // 16-byte V pieces of this lane.  After the wait only q / k / v of the new position are one L2 round trip away.
  {
    const short* src = s.src + (long)r * T_MAX;
#pragma unroll 1
    for (int p = lane; p < pos; p += 32) ssrc[p] = src[p];
  }
  __syncwarp();
  uint4 kpre[8];
  if (lane < pos) {
    const uint4* kp = reinterpret_cast<const uint4*>(kc + (long)ssrc[lane] * row_stride + ((long)h * T_MAX + lane) * 64);
#pragma unroll
    for (int c = 0; c < 8; ++c) kpre[c] = kp[c];
  }
  const int c8 = lane & 7, pg = lane >> 3;
  const long hoff = (long)h * T_MAX * 64 + c8 * 8;
  uint4 vpre[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int p = pg + 4 * i;
    vpre[i] = p < pos ? *reinterpret_cast<const uint4*>(vc + (long)ssrc[p] * row_stride + hoff + (long)p * 64) : make_uint4(0u, 0u, 0u, 0u);
  }
  tl_stamp(TL_SELF, 0);
  pdl_wait();
  tl_stamp(TL_SELF, 1);
  if (PLAIN) {
    const float* row = qkv.ptr + (long)r * 3 * d + c0;
    qv = __ldcg(reinterpret_cast<const float2*>(row));
    kv = __ldcg(reinterpret_cast<const float2*>(row + d));
    vv = __ldcg(reinterpret_cast<const float2*>(row + 2 * d));
  } else {
    // at most 8 K ranges (dec_gemm_split_plan); predicated so that all 24 loads are in flight together, summed in order
    const float* row = qkv.ptr + (long)r * 3 * d + c0;
    const float2 z2 = make_float2(0.f, 0.f);
    float2 qa[8], ka[8], va[8];
#pragma unroll
    for (int sp = 0; sp < 8; ++sp) {
      const float* p = row + (long)sp * qkv.stride;
      const bool on = sp < qkv.nsplit;
      qa[sp] = on ? __ldcg(reinterpret_cast<const float2*>(p)) : z2;
      ka[sp] = on ? __ldcg(reinterpret_cast<const float2*>(p + d)) : z2;
      va[sp] = on ? __ldcg(reinterpret_cast<const float2*>(p + 2 * d)) : z2;
    }
#pragma unroll
    for (int sp = 0; sp < 8; ++sp) {
      qv.x += qa[sp].x; qv.y += qa[sp].y; kv.x += ka[sp].x; kv.y += ka[sp].y; vv.x += va[sp].x; vv.y += va[sp].y;
    }
  }
  qv.x *= 0.125f; qv.y *= 0.125f;
  *reinterpret_cast<float2*>(q + 2 * lane) = qv;
  *reinterpret_cast<float2*>(vnew + 2 * lane) = vv;
  {
    const int wr = s.wrow != nullptr ? s.wrow[r] : r;
    const long o = (long)wr * row_stride + ((long)h * T_MAX + pos) * 64 + 2 * lane;
    *reinterpret_cast<__half2*>(kc + o) = __floats2half2_rn(kv.x, kv.y);
    *reinterpret_cast<__half2*>(vc + o) = __floats2half2_rn(vv.x, vv.y);
  }
  const float dot_new = warp_sum(qv.x * kv.x + qv.y * kv.y);   // the new position uses the unrounded k (as before)
  float lmax = -INFINITY;
#pragma unroll 1
  for (int p = lane; p < n; p += 32) {
    float acc = dot_new;
    if (p != pos) {
      uint4 u[8];
      if (p == lane) {
#pragma unroll
        for (int c = 0; c < 8; ++c) u[c] = kpre[c];
      } else {
        const uint4* kp = reinterpret_cast<const uint4*>(kc + (long)ssrc[p] * row_stride + ((long)h * T_MAX + p) * 64);
#pragma unroll
        for (int c = 0; c < 8; ++c) u[c] = kp[c];
      }
      acc = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const __half2* h2 = reinterpret_cast<const __half2*>(&u[c]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h2[e]);
          acc = fmaf(q[c * 8 + 2 * e], f.x, acc);
          acc = fmaf(q[c * 8 + 2 * e + 1], f.y, acc);
        }
      }
    }
    sc[p] = acc;
    lmax = fmaxf(lmax, acc);
  }
  const float mx = warp_max(lmax);
  float lsum = 0.f;
#pragma unroll 1
  for (int p = lane; p < n; p += 32) {
    const float e = __expf(sc[p] - mx);
    sc[p] = e;
    lsum += e;
  }
  const float inv = 1.f / warp_sum(lsum);
  __syncwarp();
  // weighted V sum: lane = (position group pg = lane / 8, 16-byte dim chunk c8 = lane % 8).  The 4 groups stride over
  // the cached positions with independent 16-byte loads (8 in flight per lane), then fold with two shuffles, instead of
  // walking the positions one by one with a dependent (index -> V row) load pair each.
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {          // positions pg + 4 i < 32: prefetched before the wait
    const int p = pg + 4 * i;
    const float w = p < pos ? sc[p] : 0.f;
    const __half2* h2 = reinterpret_cast<const __half2*>(&vpre[i]);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      acc[2 * e] = fmaf(w, f.x, acc[2 * e]);
      acc[2 * e + 1] = fmaf(w, f.y, acc[2 * e + 1]);
    }
  }
#pragma unroll 4
  for (int p = pg + 32; p < pos; p += 4) {
    const float w = sc[p];
    const uint4 u = *reinterpret_cast<const uint4*>(vc + (long)ssrc[p] * row_stride + hoff + (long)p * 64);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      acc[2 * e] = fmaf(w, f.x, acc[2 * e]);
      acc[2 * e + 1] = fmaf(w, f.y, acc[2 * e + 1]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 8);
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 16);
  }
  if (pg == 0) {
    const float wn = sc[pos];
    __align__(16) __half2 o2[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      o2[e] = __floats2half2_rn(fmaf(wn, vnew[c8 * 8 + 2 * e], acc[2 * e]) * inv, fmaf(wn, vnew[c8 * 8 + 2 * e + 1], acc[2 * e + 1]) * inv);
    *reinterpret_cast<uint4*>(out + (long)r * d + h * 64 + c8 * 8) = *reinterpret_cast<const uint4*>(o2);
  }
}

void decoder_self_attn(cudaStream_t st, const DecodeState& s, const PartialSrc& qkv, __half* kcache, __half* vcache,
                       long cache_row_stride, __half* out, int R, int H, int d) {
  if (qkv.nsplit == 1 && qkv.bias == nullptr)
    launch_kernel(self_attn_kernel<true>, dim3(cdiv((long)R * H, SA_WARPS)), dim3(SA_WARPS * 32), 0, st, s, qkv, kcache, vcache,
                  cache_row_stride, out, H, d, R);
  else
    launch_kernel(self_attn_kernel<false>, dim3(cdiv((long)R * H, SA_WARPS)), dim3(SA_WARPS * 32), 0, st, s, qkv, kcache, vcache,
                  cache_row_stride, out, H, d, R);
  note_launch(1);
}

// ============================================================================ K11 cross attention
// Per (stream, head, key range): S = q K^T and O = P V on the warp-level tensor-core path (mma.sync m16n8k16,
// fp16 operands, fp32 accumulate; N = 8 = the stream's beam rows).  The kernel is an HBM stream of the encoder
// K/V (246 MB per layer at 32 streams) -- the arithmetic is ~0.1 GFLOP per CTA, so it stays on mma.sync rather
// than wgmma (M = 64-row warpgroup tiles buy nothing here); what matters is that the consumer
// warps issue ~40 instructions per 16 KB chunk instead of ~400 on the CUDA-core path, which left the kernel
// issue-bound at half of the HBM rate.
//   * K/V chunks (128 keys x 64 dims, 16 KB contiguous) arrive by cp.async.bulk into a ring of XA_STAGES buffers.
//     The pool stores every 128-byte key row with its 16-byte pieces XOR-swizzled by (key & 7) (written that way
//     by the cross-KV GEMM epilogue), so ldmatrix reads the chunks bank-conflict free without a tensor map.
//   * q is split into fp16 hi + lo parts (two MMAs): scores keep fp32-level accuracy in q; K is fp16 storage.
//   * two passes over the key range (scores -> exact max/sum -> weights), so no online rescaling; P is fed to the
//     second MMA as fp16, the row sum is taken over the same rounded values.
constexpr int XA_CHUNK = 128;                 // keys per pipeline stage
constexpr int XA_STAGES = 3;                  // x 3 CTAs per SM at beam <= 4: 144 KB of K/V in flight per SM
constexpr int XA_STAGE_BYTES = XA_CHUNK * 128;  // 64 halves per key
constexpr int XA_NCHUNK = (S_ENC + XA_CHUNK - 1) / XA_CHUNK;  // 12
constexpr int XA_TAIL_KEYS = S_ENC - (XA_NCHUNK - 1) * XA_CHUNK;  // 92 keys in the last chunk
constexpr int MAX_STREAMS_CAP = 256;          // streams per decode call the live list can hold
constexpr int XA_MAX_QSPLIT = 4;              // K ranges of the q projection the kernel sums (engine.cu caps the plan)

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D (16x8, f32) += A (16x16, f16, row) * B (16x8, f16, col)
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// A consumer warp hands a ring stage it has read with ldmatrix back to the producer.  The stage is refilled by
// cp.async.bulk (async proxy), so the generic-proxy ldmatrix reads must be ordered before that write by a proxy fence;
// the mbarrier arrive alone does not do it.  With CUDA 12.9, ptxas scheduled the arrive before the MMA that consumes the
// last fragment, with no wait on that ldmatrix: the next chunk could overwrite K/V not yet read, and a stream's
// attention output then depended on which other streams were still decoding.
__device__ __forceinline__ void release_stage(uint64_t* empty, int lane) {
  __syncwarp();
  fence_proxy_async();
  if (lane == 0) mbar_arrive(empty);
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int NQ> struct XaCfg {
  static constexpr int SW = NQ <= 2 ? 2 : NQ <= 4 ? 4 : 8;   // score columns kept per key (fp32)
};

template <int NQ>
__global__ void __launch_bounds__(160) cross_attn_kernel(DecodeState s, PartialSrc q,
                                                         const __half* __restrict__ kc, const __half* __restrict__ vc,
                                                         long slot_stride, float* __restrict__ part,
                                                         float* __restrict__ probs, __half* __restrict__ out, int B,
                                                         int rows_per_stream, int H, int d, int nsplit, int cps) {
  constexpr int SW = XaCfg<NQ>::SW;
  extern __shared__ uint8_t xa_smem_raw[];
  uint8_t* base = xa_smem_raw + ((128u - (smem_u32(xa_smem_raw) & 127u)) & 127u);   // pointer arithmetic keeps the shared address space (LDS/STS)
  const int nk_cap = cps * XA_CHUNK;
  const int ph_ld = nk_cap + 8;                                         // halves; +8 -> rows 16 B apart mod 128 B (conflict-free B fragments)
  uint8_t* stage_buf = base;                                            // XA_STAGES x 16 KB
  // S [cps*128][SW] holds the scores, then exp(); the same bytes serve as q staging [8][64] before the first sweep and
  // as the cross-warp output reduction [4][8][64] after the second one (S is dead by then).
  float* S = reinterpret_cast<float*>(base + XA_STAGES * XA_STAGE_BYTES);
  float* ored = S;
  const int s_floats = max(nk_cap * SW, 4 * 8 * 64);
  __half* Ph = reinterpret_cast<__half*>(S + s_floats);                 // [NQ][ph_ld] weights for the P V MMA
  float* red = reinterpret_cast<float*>(Ph + (long)NQ * ph_ld);         // [2][4][8]
  uint64_t* full = reinterpret_cast<uint64_t*>(red + 64);
  uint64_t* empty = full + XA_STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ uint8_t live[MAX_STREAMS_CAP];
  __shared__ int n_live_sh;
  pdl_trigger();

  if (tid == 0) {
    for (int i = 0; i < XA_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);
    }
    mbar_fence_init();
  }
  if (warp == 0) {
    // Compact list of the streams still decoding.  `done` was written by the previous step's search kernel, which
    // completed before this step's first kernel started, so it may be read ahead of the dependency wait.
    int base_n = 0;
    for (int b0 = 0; b0 < B; b0 += 32) {
      const bool alive = (b0 + lane < B) && !s.done[b0 + lane];
      const unsigned m = __ballot_sync(0xffffffffu, alive);
      if (alive) live[base_n + __popc(m & ((1u << lane) - 1u))] = (uint8_t)(b0 + lane);
      base_n += __popc(m);
    }
    if (lane == 0) n_live_sh = base_n;
  }
  {
    // the last chunk holds 92 keys: rows 92..127 of every ring buffer must be finite (their weights are exactly 0,
    // but 0 x NaN would poison the P V product).  Later full chunks leave finite K/V values there.
    constexpr int TAIL16 = (XA_CHUNK - XA_TAIL_KEYS) * 8;   // 16-byte pieces per buffer
    for (int i = tid; i < XA_STAGES * TAIL16; i += 160) {
      const int st = i / TAIL16, o = i % TAIL16;
      *reinterpret_cast<uint4*>(stage_buf + st * XA_STAGE_BYTES + XA_TAIL_KEYS * 128 + o * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async();
  }
  __syncthreads();
  // Persistent CTA: work items (live stream, head, key range) it, it + grid, ...  The producer warp runs ahead into
  // the next item's K chunks while the consumers are still reducing / writing out the current one.
  const int total_items = n_live_sh * H * nsplit;

  if (warp == 4) {
    // ------------------------------------------------------------------ producer warp
    // Encoder K/V, slot ids and done flags all predate this decode step: nothing here needs the dependency wait.
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
#pragma unroll 1
      for (int it = blockIdx.x; it < total_items; it += gridDim.x) {
        const unsigned bh = (unsigned)it / (unsigned)nsplit, bi = bh / (unsigned)H;
        const int sp = it - (int)bh * nsplit, h = (int)(bh - bi * (unsigned)H), b = live[bi];
        const int c_begin = sp * cps, c_end = min(XA_NCHUNK, c_begin + cps);
        const long head_off = (long)s.slot[b] * slot_stride + (long)h * S_ENC * 64;
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
          const __half* src = (pass == 0 ? kc : vc) + head_off;
#pragma unroll 1
          for (int c = c_begin; c < c_end; ++c) {
            const int nkeys = min(XA_CHUNK, S_ENC - c * XA_CHUNK);
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_expect_tx(&full[stage], nkeys * 128);
            bulk_load_1d(stage_buf + stage * XA_STAGE_BYTES, src + (long)c * XA_CHUNK * 64, nkeys * 128, &full[stage]);
            if (++stage == XA_STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumer warps (128 threads)
  tl_stamp(TL_CROSS, 0);
  pdl_wait();   // q comes from the projection GEMM right before this kernel
  tl_stamp(TL_CROSS, 1);
  const int g = lane >> 2, tq = lane & 3;    // mma fragment coordinates: group (row / n index), thread-in-group
  int stage = 0;
  uint32_t phase = 0;
  constexpr int MAX_QSPLIT = XA_MAX_QSPLIT;     // the q projection is split over at most this many K ranges
  float qraw[4][1 + MAX_QSPLIT];                // this thread's 4 entries of q[8][64]: bias + raw partial sums
  // The item loop is rotated by half an item so that the q fetch exists ONCE in the code: "iteration -1" only requests
  // the first item's q; every later iteration requests the next item's q in the middle of the current one (its
  // latency hides behind the softmax pass and the V sweep).  The kernel is launched once per layer per token; its
  // instruction footprint is part of what every launch costs (see dec_gemm.cu).
#pragma unroll 1
  for (int it = (int)blockIdx.x - (int)gridDim.x; it < total_items; it += gridDim.x) {
  const bool real = it >= 0;
  int sp = 0, h = 0, b = 0;
  if (real) {
    const unsigned bh = (unsigned)it / (unsigned)nsplit, bi = bh / (unsigned)H;
    sp = it - (int)bh * nsplit; h = (int)(bh - bi * (unsigned)H); b = live[bi];
  }
  const int c_begin = sp * cps, c_end = min(XA_NCHUNK, c_begin + cps);
  const int nchunks = c_end - c_begin;
  const int row0 = b * rows_per_stream;
  uint32_t qh[4][2], ql[4][2];
  if (real) {
  // q rows of this (stream, head) as [8][64] fp32 in shared memory (rows >= rows_per_stream are zero), pre-scaled by 1/8
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float a = qraw[e][0];   // bias
#pragma unroll
    for (int sq = 0; sq < MAX_QSPLIT; ++sq) a += qraw[e][1 + sq];   // K ranges in index order
    ored[tid + e * 128] = a * 0.125f;
  }
  consumers_sync();
  // B fragments of q^T (k = dim, n = row): lane holds q[g][ks*16 + 2*tq + {0,1}] and [.. + 8], as hi + lo halves
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float2 v = *reinterpret_cast<const float2*>(ored + g * 64 + ks * 16 + r * 8 + 2 * tq);
      const __half2 hi = __floats2half2_rn(v.x, v.y);
      const float2 hf = __half22float2(hi);
      qh[ks][r] = *reinterpret_cast<const uint32_t*>(&hi);
      ql[ks][r] = pack_half2(v.x - hf.x, v.y - hf.y);
    }
  consumers_sync();   // ored is reused at the end

  // ---- pass 1: scores.  Warp w owns keys [32w, 32w+32) of every chunk: 2 m-tiles x 4 k-steps.
  const int ld_row = (lane & 7) + ((lane >> 3) & 1) * 8;   // ldmatrix: row this lane addresses inside a 16-row tile
#pragma unroll 1
  for (int ci = 0; ci < nchunks; ++ci) {
    const int nkeys = min(XA_CHUNK, S_ENC - (c_begin + ci) * XA_CHUNK);
    mbar_wait(&full[stage], phase);
    const uint32_t buf = smem_u32(stage_buf + stage * XA_STAGE_BYTES);
    float sc[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      sc[mt][0] = sc[mt][1] = sc[mt][2] = sc[mt][3] = 0.f;
      const int key_l = warp * 32 + mt * 16 + ld_row;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t a[4];
        const int piece = ks * 2 + (lane >> 4);
        ldmatrix_x4(a, buf + key_l * 128 + ((piece ^ (key_l & 7)) << 4));
        mma_16816(sc[mt], a, qh[ks][0], qh[ks][1]);
        mma_16816(sc[mt], a, ql[ks][0], ql[ks][1]);
      }
    }
    release_stage(&empty[stage], lane);   // K fragments are in registers now
    if (++stage == XA_STAGES) { stage = 0; phase ^= 1; }
    if (2 * tq < SW) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int k0 = warp * 32 + mt * 16 + g;
        const float2 lo = k0 < nkeys ? make_float2(sc[mt][0], sc[mt][1]) : make_float2(-INFINITY, -INFINITY);
        const float2 hi = k0 + 8 < nkeys ? make_float2(sc[mt][2], sc[mt][3]) : make_float2(-INFINITY, -INFINITY);
        *reinterpret_cast<float2*>(S + ((long)ci * XA_CHUNK + k0) * SW + 2 * tq) = lo;
        *reinterpret_cast<float2*>(S + ((long)ci * XA_CHUNK + k0 + 8) * SW + 2 * tq) = hi;
      }
    }
  }
  }   // real: scores of this item are in S
  // request the next item's q partial sums now: they arrive while the softmax pass and the V sweep run
  if (it + (int)gridDim.x < total_items) {
    const int item = it + (int)gridDim.x;
    const unsigned bh2 = (unsigned)item / (unsigned)nsplit, bi2 = bh2 / (unsigned)H;
    const int h2 = (int)(bh2 - bi2 * (unsigned)H), b2 = live[bi2];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 128, j = idx >> 6, dd = idx & 63;
      const bool ok = j < rows_per_stream;
      qraw[e][0] = (ok && q.bias) ? __ldg(q.bias + h2 * 64 + dd) : 0.f;
      const float* qp = q.ptr + (long)(b2 * rows_per_stream + (ok ? j : 0)) * d + h2 * 64 + dd;
#pragma unroll
      for (int sq = 0; sq < MAX_QSPLIT; ++sq) qraw[e][1 + sq] = (ok && sq < q.nsplit) ? __ldcg(qp + (long)sq * q.stride) : 0.f;
    }
  }
  if (!real) continue;
  consumers_sync();
  // ---- softmax statistics over this CTA's key range
  const int nk_pad = nchunks * XA_CHUNK;
  float mx[NQ], sm[NQ];
#pragma unroll
  for (int j = 0; j < NQ; ++j) mx[j] = -INFINITY;
#pragma unroll 1
  for (int k = tid; k < nk_pad; k += 128) {
#pragma unroll
    for (int j = 0; j < NQ; ++j) mx[j] = fmaxf(mx[j], S[(long)k * SW + j]);
  }
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    mx[j] = warp_max(mx[j]);
    if (lane == 0) red[warp * 8 + j] = mx[j];
  }
  consumers_sync();
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    mx[j] = fmaxf(fmaxf(red[j], red[8 + j]), fmaxf(red[16 + j], red[24 + j]));
    sm[j] = 0.f;
  }
  float sm32[NQ];   // exact fp32 sums: only the alignment probabilities use them
#pragma unroll
  for (int j = 0; j < NQ; ++j) sm32[j] = 0.f;
#pragma unroll 1
  for (int k = tid; k < nk_pad; k += 128) {
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      const float e32 = __expf(S[(long)k * SW + j] - mx[j]);
      const __half eh = __float2half_rn(e32);
      Ph[(long)j * ph_ld + k] = eh;
      sm[j] += __half2float(eh);
      if (probs != nullptr) {
        S[(long)k * SW + j] = e32;
        sm32[j] += e32;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NQ; ++j) {
    sm[j] = warp_sum(sm[j]);
    if (lane == 0) red[32 + warp * 8 + j] = sm[j];
  }
  consumers_sync();
#pragma unroll
  for (int j = 0; j < NQ; ++j) sm[j] = red[32 + j] + red[40 + j] + red[48 + j] + red[56 + j];
  if (probs != nullptr && nsplit == 1) {
    // K14 word alignment reads the attention probabilities themselves: exact fp32 exp / fp32 sum
    consumers_sync();
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      sm32[j] = warp_sum(sm32[j]);
      if (lane == 0) red[32 + warp * 8 + j] = sm32[j];
    }
    consumers_sync();
#pragma unroll
    for (int j = 0; j < NQ; ++j) sm32[j] = red[32 + j] + red[40 + j] + red[48 + j] + red[56 + j];
    for (int k = tid; k < S_ENC; k += 128) {
#pragma unroll
      for (int j = 0; j < NQ; ++j)
        if (j < rows_per_stream) probs[((long)(row0 + j) * H + h) * S_ENC + k] = S[(long)k * SW + j] / sm32[j];
    }
  }
  // ---- pass 2: O^T[dd][j] += V^T[dd][key] P^T[key][j].  Warp w owns keys [32w, 32w+32): 2 k-steps x 4 m-tiles of dd.
  float o[4][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) o[mt][0] = o[mt][1] = o[mt][2] = o[mt][3] = 0.f;
  const int ldt_row = (lane & 7) + (lane >> 4) * 8;       // .trans tiles: matrices 2,3 are the second 8 keys
#pragma unroll 1
  for (int ci = 0; ci < nchunks; ++ci) {
    mbar_wait(&full[stage], phase);
    const uint32_t buf = smem_u32(stage_buf + stage * XA_STAGE_BYTES);
    // rolled: unrolled, ptxas hoists the second k-step's ldmatrix loads above the first one's MMAs and the 8-row
    // instantiation spills
#pragma unroll 1
    for (int kk = 0; kk < 2; ++kk) {
      const int kbase = warp * 32 + kk * 16;
      uint32_t b0 = 0u, b1 = 0u;
      if (g < NQ) {
        const __half* pp = Ph + (long)g * ph_ld + ci * XA_CHUNK + kbase + 2 * tq;
        b0 = *reinterpret_cast<const uint32_t*>(pp);
        b1 = *reinterpret_cast<const uint32_t*>(pp + 8);
      }
      const int key_l = kbase + ldt_row;
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        uint32_t a[4];
        const int piece = mt * 2 + ((lane >> 3) & 1);
        ldmatrix_x4_trans(a, buf + key_l * 128 + ((piece ^ (key_l & 7)) << 4));
        mma_16816(o[mt], a, b0, b1);
      }
    }
    release_stage(&empty[stage], lane);
    if (++stage == XA_STAGES) { stage = 0; phase ^= 1; }
  }
  // reduce the 4 warps (key quarters) through smem: lane holds O[j = 2tq + {0,1}][dd = mt*16 + g (+8)]
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
    float* ob = ored + (warp * 8 + 2 * tq) * 64 + mt * 16 + g;
    ob[0] = o[mt][0];
    ob[64] = o[mt][1];
    ob[8] = o[mt][2];
    ob[64 + 8] = o[mt][3];
  }
  consumers_sync();
  if (nsplit == 1) {   // the whole key range was here: normalise and store the attention output directly
    for (int idx = tid; idx < NQ * 64; idx += 128) {
      const int j = idx >> 6, dd = idx & 63;
      if (j < rows_per_stream) {
        const float ov = ored[(0 * 8 + j) * 64 + dd] + ored[(1 * 8 + j) * 64 + dd] + ored[(2 * 8 + j) * 64 + dd] +
                         ored[(3 * 8 + j) * 64 + dd];
        float l = sm[0];
#pragma unroll
        for (int jj = 1; jj < NQ; ++jj) l = j == jj ? sm[jj] : l;
        out[(long)(row0 + j) * d + h * 64 + dd] = __float2half_rn(ov / l);
      }
    }
    consumers_sync();   // ored / red are reused by the next item
    continue;
  }
  float* pbase = part + ((long)b * H + h) * nsplit * MAX_ROWS_PER_STREAM * 66;
  float* dst = pbase + (long)sp * MAX_ROWS_PER_STREAM * 66;
  for (int idx = tid; idx < NQ * 64; idx += 128) {
    const int j = idx >> 6, dd = idx & 63;
    if (j < rows_per_stream) {
      const float ov = ored[(0 * 8 + j) * 64 + dd] + ored[(1 * 8 + j) * 64 + dd] + ored[(2 * 8 + j) * 64 + dd] +
                       ored[(3 * 8 + j) * 64 + dd];
      dst[j * 66 + 2 + dd] = ov;
    }
  }
  if (tid < NQ && tid < rows_per_stream) {
    dst[tid * 66 + 0] = mx[tid];
    dst[tid * 66 + 1] = sm[tid];
  }
  consumers_sync();   // ored is rewritten by the next item
  }   // item loop
}

// Merge the nsplit partial softmaxes of every (row, head), in key-range order.  A separate (tiny) kernel on purpose:
// merging inside cross_attn_kernel (last key range to arrive, found with a fence + atomic) makes every persistent CTA
// pay the fence/atomic round trip once per item in the middle of its K/V stream, which grows with the stream count.
__global__ void __launch_bounds__(64) cross_attn_combine_kernel(DecodeState s, const float* __restrict__ part, __half* __restrict__ out,
                                                                int rows_per_stream, int H, int d, int nsplit) {
  const int r = blockIdx.y, h = blockIdx.x, dd = threadIdx.x;
  const int b = r / rows_per_stream, j = r - b * rows_per_stream;
  pdl_trigger();
  if (s.done[b]) return;
  tl_stamp(TL_COMBINE, 0);
  pdl_wait();
  tl_stamp(TL_COMBINE, 1);
  const float* p = part + (((long)b * H + h) * nsplit) * MAX_ROWS_PER_STREAM * 66 + j * 66;
  // loads of up to 6 ranges in flight together (what cross_attn_pick_nsplit chooses in practice), a rolled loop for more
  float m[6], l[6], o[6];
#pragma unroll
  for (int sp = 0; sp < 6; ++sp) {
    const float* ps = p + (long)sp * MAX_ROWS_PER_STREAM * 66;
    const bool on = sp < nsplit;
    m[sp] = on ? __ldcg(ps) : -INFINITY;
    l[sp] = on ? __ldcg(ps + 1) : 0.f;
    o[sp] = on ? __ldcg(ps + 2 + dd) : 0.f;
  }
  float M = -INFINITY;
#pragma unroll
  for (int sp = 0; sp < 6; ++sp) M = fmaxf(M, m[sp]);
#pragma unroll 1
  for (int sp = 6; sp < nsplit; ++sp) M = fmaxf(M, __ldcg(p + (long)sp * MAX_ROWS_PER_STREAM * 66));
  float L = 0.f, acc = 0.f;
#pragma unroll
  for (int sp = 0; sp < 6; ++sp) {
    const float w = sp < nsplit ? __expf(m[sp] - M) : 0.f;
    L += l[sp] * w;
    acc += o[sp] * w;
  }
#pragma unroll 1
  for (int sp = 6; sp < nsplit; ++sp) {
    const float* ps = p + (long)sp * MAX_ROWS_PER_STREAM * 66;
    const float w = __expf(__ldcg(ps) - M);
    L += __ldcg(ps + 1) * w;
    acc += __ldcg(ps + 2 + dd) * w;
  }
  out[(long)r * d + h * 64 + dd] = __float2half_rn(acc / L);
}

static int xa_template_nq(int rows_per_stream) {
  return rows_per_stream == 1 ? 1 : rows_per_stream == 2 ? 2 : rows_per_stream <= 4 ? 4 : rows_per_stream == 5 ? 5 : 8;
}
static int xa_smem_bytes(int cps, int NQ) {
  const int sw = NQ <= 2 ? 2 : NQ <= 4 ? 4 : 8;
  const int nk = cps * XA_CHUNK;
  return 128 + XA_STAGES * XA_STAGE_BYTES + std::max(nk * sw, 4 * 8 * 64) * 4 + NQ * (nk + 8) * 2 + 64 * 4 + 2 * XA_STAGES * 8 + 64;
}

// resident CTAs per SM for this key-range length, asked from the runtime (cached): the grid of the persistent
// kernel is exactly occupancy x SMs
static int xa_occupancy(int NQ, int cps) {
  static std::mutex mu;
  static std::map<int, int> cache;
  std::lock_guard<std::mutex> lk(mu);
  const int key = NQ * 64 + cps;
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  const void* k = NQ == 1   ? (const void*)cross_attn_kernel<1>
                  : NQ == 2 ? (const void*)cross_attn_kernel<2>
                  : NQ == 4 ? (const void*)cross_attn_kernel<4>
                  : NQ == 5 ? (const void*)cross_attn_kernel<5>
                            : (const void*)cross_attn_kernel<8>;
  int occ = 0;
  WL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, 160, (size_t)xa_smem_bytes(cps, NQ)));
  occ = std::max(1, occ);
  cache[key] = occ;
  return occ;
}

// Choose how many CTAs share one (stream, head): the grid should fill whole waves of resident CTAs
// (occupancy is set by shared memory: the score / weight buffers shrink with the split).
int cross_attn_pick_nsplit(int B, int H, int num_sms, int rows_per_stream) {
  const int NQ = xa_template_nq(rows_per_stream);
  // cost of a split = waves of resident CTAs x (chunks per CTA + a fixed per-CTA cost of ~3 chunk times: q reduction,
  // pipeline fill, the softmax pass between the two sweeps, partial write-out); ties go to fewer partials
  int best_ns = 1;
  double best_cost = 1e30;
  for (int ns = 1; ns <= XA_NCHUNK; ++ns) {
    const int cps = (XA_NCHUNK + ns - 1) / ns;
    const int real = (XA_NCHUNK + cps - 1) / cps;
    if (real != ns) continue;
    const int occ = xa_occupancy(NQ, cps);
    const long slots = (long)occ * num_sms, items = (long)B * H * ns;
    const long waves = (items + slots - 1) / slots;
    const double cost = (double)waves * (cps + 3.0);
    if (cost < best_cost - 1e-9) { best_cost = cost; best_ns = ns; }
  }
  return best_ns;
}

template <int NQ>
static void launch_cross(cudaStream_t st, const DecodeState& s, const PartialSrc& q, const __half* kc, const __half* vc,
                         long slot_stride, const CrossAttnWorkspace& ws, __half* out, int B, int rows_per_stream, int H, int d,
                         int nsplit) {
  const int cps = (XA_NCHUNK + nsplit - 1) / nsplit;
  const int smem = xa_smem_bytes(cps, NQ);
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  const int occ = xa_occupancy(NQ, cps);
  WL_CHECK(B <= MAX_STREAMS_CAP, WL_ERR_ARG, "cross attention: %d streams exceed the compiled cap %d", B, MAX_STREAMS_CAP);
  dim3 grid((unsigned)std::min<long>((long)B * H * nsplit, (long)occ * sms));
  if (ws.ev0) WL_CUDA(cudaEventRecord(ws.ev0, st));
  launch_kernel(cross_attn_kernel<NQ>, grid, dim3(160), (size_t)smem, st, s, q, kc, vc, slot_stride, ws.part, ws.probs, out, B,
                rows_per_stream, H, d, nsplit, cps);
  if (ws.ev1) WL_CUDA(cudaEventRecord(ws.ev1, st));
  note_launch(1);
}

template <int NQ>
static void prime_cross() {
  WL_CUDA(cudaFuncSetAttribute(cross_attn_kernel<NQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
}
void attention_tl_bind(unsigned long long* p) { tl_bind_tu(p); }
void attention_prime() {
  prime_cross<1>();
  prime_cross<2>();
  prime_cross<4>();
  prime_cross<5>();
  prime_cross<8>();
}

void decoder_cross_attn(cudaStream_t st, const DecodeState& s, const PartialSrc& q, const __half* kc, const __half* vc,
                        long slot_stride, const CrossAttnWorkspace& ws, __half* out, int B, int rows_per_stream, int H,
                        int d, int nsplit) {
  WL_CHECK(rows_per_stream >= 1 && rows_per_stream <= MAX_ROWS_PER_STREAM, WL_ERR_ARG, "rows per stream %d", rows_per_stream);
  WL_CHECK(q.nsplit >= 1 && q.nsplit <= XA_MAX_QSPLIT, WL_ERR_ARG, "cross attention: q arrives in %d K ranges (1..%d supported)", q.nsplit, XA_MAX_QSPLIT);
  if (rows_per_stream == 1) launch_cross<1>(st, s, q, kc, vc, slot_stride, ws, out, B, rows_per_stream, H, d, nsplit);
  else if (rows_per_stream == 2) launch_cross<2>(st, s, q, kc, vc, slot_stride, ws, out, B, rows_per_stream, H, d, nsplit);
  else if (rows_per_stream <= 4) launch_cross<4>(st, s, q, kc, vc, slot_stride, ws, out, B, rows_per_stream, H, d, nsplit);
  else if (rows_per_stream == 5) launch_cross<5>(st, s, q, kc, vc, slot_stride, ws, out, B, rows_per_stream, H, d, nsplit);
  else launch_cross<8>(st, s, q, kc, vc, slot_stride, ws, out, B, rows_per_stream, H, d, nsplit);
  if (nsplit > 1) {
    launch_kernel(cross_attn_combine_kernel, dim3(H, B * rows_per_stream), dim3(64), 0, st, s, ws.part, out, rows_per_stream, H, d, nsplit);
    note_launch(1);
  }
}

}  // namespace wl
