// Speaker embeddings (wespeaker ResNet34 over Kaldi fbank, the protocol named in whisperlive_b200/speaker.py) for every
// stream of a wl_spk_embed call in one set of launches.  Stream b's fbank frames sit at frame_off[b] of one frame axis;
// an activation of a stage is channels-last fp16 [position][C] with the positions of stream b at pos_off[b] in the
// order (time, frequency): position = pos_off[b] + t * H + h.  Every kernel finds a row's stream in those tables.
//
//   spk_fbank_kernel  one CTA per frame: DC removal, preemphasis, Hamming window, 512-point FFT in shared memory,
//                     power, 80 mel bins, log -- fp32
//   spk_cmn_kernel    per-stream, per-bin mean over frames (subtracted by the stem, its consumer)
//   spk_stem_kernel   conv3x3 1 -> 32 in fp32 with the folded BN and ReLU, fp16 channels-last out
//   spk_conv_kernel   implicit-GEMM 3x3 / 1x1 conv on the tensor cores: M = positions, N = C_out, K = taps x C_in;
//                     mma.sync m16n8k16 (fp16 in, fp32 accumulate) fed by ldmatrix from a 3-stage cp.async ring.  The
//                     zero padding at the frequency edges and at each stream's first and last frame is a cp.async
//                     zero-fill decided from the position tables, so no stream reads a neighbour's frames, and nothing
//                     like im2col is ever materialised.  Epilogue: bias, optional residual (may alias the output: each
//                     element is read and written by the same thread), ReLU, fp16 store.
//   spk_pool_kernel   TSTP per stream, fp32, two-pass variance; spk_embed_kernel: seg_1 for all streams
//
// A row's result depends only on its own stream's inputs and a fixed summation order, so a stream's embedding is
// bit-identical whichever streams share the call.
#include "kernels.cuh"

namespace wl {

constexpr int SPK_FRAME = 400, SPK_SHIFT = 160, SPK_NFFT = 512, SPK_MEL = 80, SPK_BINS = SPK_NFFT / 2 + 1;
constexpr float SPK_SCALE = 32768.f, SPK_PREEMPH = 0.97f, SPK_LOG_FLOOR = 1.1920928955078125e-07f;
constexpr float SPK_POOL_EPS = 1e-7f;

__device__ __forceinline__ int spk_stream_of(const long* off, int B, long g) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------ fbank
__global__ void __launch_bounds__(256) spk_fbank_kernel(const float* __restrict__ pcm, const long* __restrict__ pcm_off,
                                                        const long* __restrict__ frame_off, int B,
                                                        const float* __restrict__ melw, const int* __restrict__ mel_range,
                                                        float* __restrict__ feat) {
  __shared__ float x[SPK_FRAME];
  __shared__ float re[SPK_NFFT], im[SPK_NFFT];
  __shared__ float red[8];
  const int tid = threadIdx.x;
  const long g = blockIdx.x;
  const int b = spk_stream_of(frame_off, B, g);
  const float* src = pcm + pcm_off[b] + (g - frame_off[b]) * SPK_SHIFT;
  float s = 0.f;
  for (int i = tid; i < SPK_FRAME; i += 256) {
    const float v = src[i] * SPK_SCALE;
    x[i] = v;
    s += v;
  }
  s = warp_sum(s);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  float mean = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) mean += red[w];
  mean *= 1.f / SPK_FRAME;
  // DC removal, preemphasis (x[0] against itself), Hamming window; written in bit-reversed order for the FFT
  for (int i = tid; i < SPK_NFFT; i += 256) {
    float v = 0.f;
    if (i < SPK_FRAME) {
      const float cur = x[i] - mean, prev = x[i > 0 ? i - 1 : 0] - mean;
      const float win = 0.54f - 0.46f * cospif(2.f * i / (float)(SPK_FRAME - 1));
      v = (cur - SPK_PREEMPH * prev) * win;
    }
    const int r = __brev(i) >> (32 - 9);
    re[r] = v;
    im[r] = 0.f;
  }
  __syncthreads();
  for (int h = 1; h < SPK_NFFT; h <<= 1) {
    const int j = tid, k = j & (h - 1), i0 = (j - k) * 2 + k, i1 = i0 + h;
    float sn, cs;
    sincospif(-(float)k / (float)h, &sn, &cs);
    const float br = re[i1] * cs - im[i1] * sn, bi = re[i1] * sn + im[i1] * cs;
    const float ar = re[i0], ai = im[i0];
    __syncthreads();
    re[i0] = ar + br; im[i0] = ai + bi;
    re[i1] = ar - br; im[i1] = ai - bi;
    __syncthreads();
  }
  float* power = re;   // in place: bin k's power replaces re[k] once every thread has read its bins
  float pw[2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int k = tid + q * 256;
    pw[q] = k < SPK_BINS ? re[k] * re[k] + im[k] * im[k] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 2; ++q)
    if (tid + q * 256 < SPK_BINS) power[tid + q * 256] = pw[q];
  __syncthreads();
  if (tid < SPK_MEL) {
    const int k0 = mel_range[2 * tid], k1 = mel_range[2 * tid + 1];
    float e = 0.f;
    for (int k = k0; k < k1; ++k) e = fmaf(melw[tid * SPK_BINS + k], power[k], e);
    feat[g * SPK_MEL + tid] = logf(fmaxf(e, SPK_LOG_FLOOR));
  }
}

// mean[b][m] over stream b's frames: 4 partial sums per bin in a fixed order
__global__ void __launch_bounds__(4 * SPK_MEL) spk_cmn_kernel(const float* __restrict__ feat, const long* __restrict__ frame_off,
                                                              float* __restrict__ mean) {
  __shared__ float part[4][SPK_MEL];
  const int b = blockIdx.x, m = threadIdx.x % SPK_MEL, q = threadIdx.x / SPK_MEL;
  const long f0 = frame_off[b], T = frame_off[b + 1] - f0;
  float s = 0.f;
  for (long t = q; t < T; t += 4) s += feat[(f0 + t) * SPK_MEL + m];
  part[q][m] = s;
  __syncthreads();
  if (q == 0) mean[b * SPK_MEL + m] = ((part[0][m] + part[1][m]) + (part[2][m] + part[3][m])) / (float)T;
}

// ------------------------------------------------------------------------------------------------ stem
// out[p][c] = relu(bias[c] + sum_{dh, dt} w[c][(dh+1)*3 + dt+1] * (feat - mean)(h + dh, t + dt)), zero outside the stream
__global__ void __launch_bounds__(256) spk_stem_kernel(const float* __restrict__ feat, const float* __restrict__ mean,
                                                       const long* __restrict__ frame_off, int B, long positions,
                                                       const float* __restrict__ w, const float* __restrict__ bias,
                                                       __half* __restrict__ out) {
  __shared__ float sw[9][32], sb[32];
  for (int i = threadIdx.x; i < 9 * 32; i += blockDim.x) sw[i % 9][i / 9] = w[i];
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= positions) return;
  const long g = p / SPK_MEL;
  const int h = (int)(p - g * SPK_MEL);
  const int b = spk_stream_of(frame_off, B, g);
  const long f0 = frame_off[b], T = frame_off[b + 1] - f0, t = g - f0;
  float v[9];
#pragma unroll
  for (int dh = -1; dh <= 1; ++dh)
#pragma unroll
    for (int dt = -1; dt <= 1; ++dt) {
      const int hh = h + dh;
      const long tt = t + dt;
      v[(dh + 1) * 3 + dt + 1] = (hh >= 0 && hh < SPK_MEL && tt >= 0 && tt < T)
                                     ? feat[(f0 + tt) * SPK_MEL + hh] - mean[b * SPK_MEL + hh] : 0.f;
    }
  uint4 o[4];
  __half* oh = reinterpret_cast<__half*>(o);
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    float a = sb[c];
#pragma unroll
    for (int k = 0; k < 9; ++k) a = fmaf(sw[k][c], v[k], a);
    oh[c] = __float2half_rn(fmaxf(a, 0.f));
  }
  uint4* dst = reinterpret_cast<uint4*>(out + p * 32);
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[i] = o[i];
}

// ------------------------------------------------------------------------------------------------ implicit-GEMM conv
constexpr int SC_BM = 128, SC_BK = 32, SC_STAGES = 3, SC_PITCH = SC_BK + 8;   // 80-byte smem rows: ldmatrix conflict-free

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void spk_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 4 warps, each 32 rows x BN columns of the 128 x BN tile
template <int BN>
__global__ void __launch_bounds__(128) spk_conv_kernel(const SpkConvParams p) {
  __shared__ __align__(128) __half As[SC_STAGES][SC_BM][SC_PITCH];
  __shared__ __align__(128) __half Bs[SC_STAGES][BN][SC_PITCH];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long m0 = (long)blockIdx.x * SC_BM;
  const int n0 = blockIdx.y * BN;
  const int K = p.taps * p.C_in, cblocks = p.C_in / SC_BK, KT = K / SC_BK;

  // geometry of this thread's A row
  const long m = m0 + tid;
  bool row_ok = m < p.M;
  long base = 0, T_in = 0;
  int to = 0, ho = 0;
  if (row_ok) {
    const int b = spk_stream_of(p.out_off, p.B, m);
    const long local = m - p.out_off[b];
    to = (int)(local / p.H_out);
    ho = (int)(local - (long)to * p.H_out);
    base = p.in_off[b];
    T_in = (p.in_off[b + 1] - base) / p.H_in;
  }

  auto load_stage = [&](int s, int kt) {
    const int tap = kt / cblocks, cb = kt - tap * cblocks;
    const int dh = p.taps == 9 ? tap / 3 - 1 : 0, dt = p.taps == 9 ? tap % 3 - 1 : 0;
    const int hi = ho * p.stride + dh;
    const long ti = (long)to * p.stride + dt;
    const bool ok = row_ok && hi >= 0 && hi < p.H_in && ti >= 0 && ti < T_in;
    const __half* src = ok ? p.x + ((base + ti * p.H_in + hi) * p.C_in + cb * SC_BK) : p.x;
#pragma unroll
    for (int c = 0; c < 4; ++c) cp_async16(&As[s][tid][c * 8], src + (ok ? c * 8 : 0), ok);
#pragma unroll
    for (int i = tid; i < BN * 4; i += 128) {
      const int r = i >> 2, c = i & 3;
      cp_async16(&Bs[s][r][c * 8], p.w + (long)(n0 + r) * K + kt * SC_BK + c * 8, true);
    }
  };

  float acc[2][BN / 8][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;

#pragma unroll
  for (int s = 0; s < SC_STAGES - 1; ++s) {
    if (s < KT) load_stage(s, s);
    cp_async_commit();
  }
#pragma unroll 1
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<SC_STAGES - 2>();
    __syncthreads();
    const int nk = kt + SC_STAGES - 1;
    if (nk < KT) load_stage(nk % SC_STAGES, nk);
    cp_async_commit();
    const int s = kt % SC_STAGES;
#pragma unroll
    for (int k16 = 0; k16 < SC_BK; k16 += 16) {
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) ldmatrix_x4(a[mt], &As[s][warp * 32 + mt * 16 + (lane & 15)][k16 + (lane >> 4) * 8]);
#pragma unroll
      for (int np = 0; np < BN / 16; ++np) {
        uint32_t bf[4];
        ldmatrix_x4(bf, &Bs[s][np * 16 + (lane & 7) + ((lane >> 4) << 3)][k16 + ((lane >> 3) & 1) * 8]);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          spk_mma(acc[mt][2 * np], a[mt], bf[0], bf[1]);
          spk_mma(acc[mt][2 * np + 1], a[mt], bf[2], bf[3]);
        }
      }
    }
  }
  cp_async_wait<0>();

  const int g = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const long r = m0 + warp * 32 + mt * 16 + g + half * 8;
      if (r >= p.M) continue;
#pragma unroll
      for (int nt = 0; nt < BN / 8; ++nt) {
        const int n = n0 + nt * 8 + 2 * tq;
        float v0 = acc[mt][nt][2 * half] + p.bias[n], v1 = acc[mt][nt][2 * half + 1] + p.bias[n + 1];
        const long o = r * p.C_out + n;
        if (p.res) {
          const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(p.res + o));
          v0 += rv.x;
          v1 += rv.y;
        }
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        *reinterpret_cast<__half2*>(p.out + o) = __floats2half2_rn(v0, v1);
      }
    }
}

// ------------------------------------------------------------------------------------------------ pooling + embedding
// pooled[b][f] (mean) and pooled[b][2560 + f] (sqrt(unbiased var + 1e-7)) of feature f = c * H + h over the stream's T'
__global__ void __launch_bounds__(256) spk_pool_kernel(const __half* __restrict__ x, const long* __restrict__ pos_off, int H,
                                                       float* __restrict__ pooled) {
  const int b = blockIdx.x, h = blockIdx.y, c = threadIdx.x;   // C = 256
  const long p0 = pos_off[b], T = (pos_off[b + 1] - p0) / H;
  const __half* px = x + (p0 + h) * 256 + c;
  float s = 0.f;
  for (long t = 0; t < T; ++t) s += __half2float(px[t * H * 256]);
  const float mean = s / (float)T;
  float q = 0.f;
  for (long t = 0; t < T; ++t) {
    const float d = __half2float(px[t * H * 256]) - mean;
    q = fmaf(d, d, q);
  }
  const int f = c * H + h, F = 256 * H;
  pooled[(long)b * 2 * F + f] = mean;
  pooled[(long)b * 2 * F + F + f] = sqrtf(q / (float)(T - 1) + SPK_POOL_EPS);
}

constexpr int SE_STREAMS = 8;
// emb[b][j] = bias[j] + sum_k wt[k][j] pooled[b][k], SE_STREAMS streams per CTA so each weight is read once per CTA
__global__ void __launch_bounds__(256) spk_embed_kernel(const float* __restrict__ pooled, const float* __restrict__ wt,
                                                        const float* __restrict__ bias, int B, int F2, float* __restrict__ emb) {
  extern __shared__ float sp[];   // [SE_STREAMS][F2]
  const int b0 = blockIdx.x * SE_STREAMS, nb = min(SE_STREAMS, B - b0), j = threadIdx.x;
  for (int i = j; i < nb * F2; i += 256) sp[i] = pooled[(long)b0 * F2 + i];
  __syncthreads();
  float a[SE_STREAMS];
#pragma unroll
  for (int s = 0; s < SE_STREAMS; ++s) a[s] = 0.f;
  for (int k = 0; k < F2; ++k) {
    const float wv = wt[(long)k * 256 + j];
#pragma unroll
    for (int s = 0; s < SE_STREAMS; ++s)
      if (s < nb) a[s] = fmaf(wv, sp[s * F2 + k], a[s]);
  }
  for (int s = 0; s < nb; ++s) emb[(long)(b0 + s) * 256 + j] = a[s] + bias[j];
}

// ------------------------------------------------------------------------------------------------ launchers
void spk_fbank(cudaStream_t st, const float* pcm, const long* pcm_off, const long* frame_off, int B, long frames,
               const float* melw, const int* mel_range, float* feat, float* mean) {
  spk_fbank_kernel<<<(unsigned)frames, 256, 0, st>>>(pcm, pcm_off, frame_off, B, melw, mel_range, feat);
  WL_CUDA(cudaGetLastError());
  spk_cmn_kernel<<<B, 4 * SPK_MEL, 0, st>>>(feat, frame_off, mean);
  WL_CUDA(cudaGetLastError());
  note_launch(2);
}

void spk_stem(cudaStream_t st, const float* feat, const float* mean, const long* frame_off, int B, long frames, const float* w,
              const float* bias, __half* out) {
  const long positions = frames * SPK_MEL;
  spk_stem_kernel<<<cdiv(positions, 256), 256, 0, st>>>(feat, mean, frame_off, B, positions, w, bias, out);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

bool spk_conv_supported(int C_in, int C_out, int taps, int stride) {
  return C_in % SC_BK == 0 && C_in > 0 && (C_out == 32 || (C_out % 64 == 0 && C_out > 0)) && (taps == 9 || taps == 1) &&
         (stride == 1 || stride == 2);
}

void spk_conv(cudaStream_t st, const SpkConvParams& p) {
  WL_CHECK(spk_conv_supported(p.C_in, p.C_out, p.taps, p.stride), WL_ERR_ARG, "spk_conv: unsupported C_in %d C_out %d taps %d stride %d",
           p.C_in, p.C_out, p.taps, p.stride);
  if (p.M <= 0) return;
  const unsigned gm = (unsigned)cdiv(p.M, SC_BM);
  if (p.C_out == 32) spk_conv_kernel<32><<<dim3(gm, 1), 128, 0, st>>>(p);
  else spk_conv_kernel<64><<<dim3(gm, p.C_out / 64), 128, 0, st>>>(p);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

void spk_pool_embed(cudaStream_t st, const __half* x, const long* pos_off, int B, int H, const float* wt, const float* bias,
                    float* pooled, float* emb) {
  spk_pool_kernel<<<dim3(B, H), 256, 0, st>>>(x, pos_off, H, pooled);
  WL_CUDA(cudaGetLastError());
  const int F2 = 2 * 256 * H;
  const size_t smem = (size_t)SE_STREAMS * F2 * sizeof(float);
  WL_CUDA(cudaFuncSetAttribute(spk_embed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  spk_embed_kernel<<<cdiv(B, SE_STREAMS), 256, smem, st>>>(pooled, wt, bias, B, F2, emb);
  WL_CUDA(cudaGetLastError());
  note_launch(2);
}

}  // namespace wl
