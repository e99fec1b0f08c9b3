// Silero VAD (16 kHz) speech probabilities on the device, fp32 throughout so that threshold decisions match the
// float64 restatement of the network (tests/vad_oracle.py).  Two kernels per wl_vad call:
//
//   vad_front_kernel  every frame of every stream at once: the frame's 576 input samples (64 of context, zeros before
//                     the stream starts and after it ends), reflection pad 64 on the right, STFT magnitude (4 x 129),
//                     four conv1d(k=3, pad=1) + ReLU blocks, and the LSTM input projection W_ih x + b_ih + b_hh.
//   vad_lstm_kernel   the recurrence, one 4-CTA cluster per stream: each CTA keeps the W_hh rows of 32 hidden units
//                     (their i, f, g, o gates) in registers, and the new h of its units is written into every CTA's
//                     shared memory through DSMEM once per step; then ReLU, the 1x1 output conv and a sigmoid.
//
// The frame protocol constants (frame 512, context 64, right reflection pad 64, one extra frame when the length is a
// multiple of 512, PyTorch gate order i, f, g, o) are named once in whisperlive_b200/vad.py; they are restated here.
#include <cooperative_groups.h>

#include "kernels.cuh"

namespace cg = cooperative_groups;

namespace wl {

constexpr int VF = 8;        // frames per front-end CTA (the weights read from L2 are reused across them)
constexpr int VT = 256;      // front-end threads
constexpr int V_FRAME = 512, V_CTX = 64, V_IN = V_FRAME + V_CTX, V_PADR = 64, V_PADDED = V_IN + V_PADR;
constexpr int V_NFFT = 256, V_HOP = 128, V_BINS = 129, V_T0 = (V_PADDED - V_NFFT) / V_HOP + 1;   // 4 STFT steps
constexpr int V_H = 128, V_G = 4 * V_H;
constexpr int V_CL = 4;                    // CTAs per LSTM cluster
constexpr int V_UNITS = V_H / V_CL;        // hidden units per CTA
static_assert(V_T0 == 4, "STFT steps");

__device__ __forceinline__ float vsigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// Binary search of the stream that owns global frame g: frame_off[b] <= g < frame_off[b + 1].
__device__ __forceinline__ int vad_stream_of(const long* frame_off, int B, long g) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (frame_off[mid] <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Weights in the layout wl_vad_load_tensor stores (output channel fastest, so consecutive threads read consecutive
// addresses): basis [256][258], conv c [ci][3][co], W_ih [128][512].
__global__ void __launch_bounds__(VT) vad_front_kernel(VadWeights w, const float* __restrict__ pcm, const long* __restrict__ pcm_off,
                                                       const long* __restrict__ frame_off, int B, long total, float* __restrict__ gx) {
  __shared__ float bufA[VF * V_PADDED];       // input frames, then conv0 / conv2 outputs
  __shared__ float bufB[VF * V_BINS * V_T0];  // magnitudes, then conv1 / conv3 outputs
  const int tid = threadIdx.x;
  const long g0 = (long)blockIdx.x * VF;

  // ---- frame inputs: sample j of frame t is the stream's sample t*512 - 64 + j (zero outside the stream); positions
  // 576..639 reflect 574..511 (the pad excludes the edge sample)
  for (int i = tid; i < VF * V_PADDED; i += VT) {
    const int f = i / V_PADDED, j = i % V_PADDED;
    const long g = g0 + f;
    float v = 0.f;
    if (g < total) {
      const int b = vad_stream_of(frame_off, B, g);
      const long t = g - frame_off[b], n = pcm_off[b + 1] - pcm_off[b];
      const int jj = j < V_IN ? j : 2 * (V_IN - 1) - j;
      const long p = t * V_FRAME - V_CTX + jj;
      if (p >= 0 && p < n) v = pcm[pcm_off[b] + p];
    }
    bufA[i] = v;
  }
  __syncthreads();

  // ---- STFT magnitude: bin k from rows k (real) and k + 129 (imaginary) of the basis; two threads per bin, four frames each
  for (int item = tid; item < 2 * V_BINS; item += VT) {
    const int bin = item % V_BINS, f0 = (item / V_BINS) * (VF / 2);
    float re[VF / 2][V_T0], im[VF / 2][V_T0];
#pragma unroll
    for (int f = 0; f < VF / 2; ++f)
#pragma unroll
      for (int t = 0; t < V_T0; ++t) re[f][t] = im[f][t] = 0.f;
    for (int k = 0; k < V_NFFT; ++k) {
      const float wr = __ldg(w.basis + k * (2 * V_BINS) + bin), wi = __ldg(w.basis + k * (2 * V_BINS) + bin + V_BINS);
#pragma unroll
      for (int f = 0; f < VF / 2; ++f)
#pragma unroll
        for (int t = 0; t < V_T0; ++t) {
          const float x = bufA[(f0 + f) * V_PADDED + t * V_HOP + k];
          re[f][t] = fmaf(wr, x, re[f][t]);
          im[f][t] = fmaf(wi, x, im[f][t]);
        }
    }
#pragma unroll
    for (int f = 0; f < VF / 2; ++f)
#pragma unroll
      for (int t = 0; t < V_T0; ++t)
        bufB[((f0 + f) * V_BINS + bin) * V_T0 + t] = sqrtf(re[f][t] * re[f][t] + im[f][t] * im[f][t]);
  }
  __syncthreads();

  // ---- conv0: 129 -> 128, 4 steps (bufB -> bufA)
  {
    const int co = tid & 127, f0 = (tid >> 7) * (VF / 2);
    float acc[VF / 2][V_T0];
    const float bias = __ldg(w.b0 + co);
#pragma unroll
    for (int f = 0; f < VF / 2; ++f)
#pragma unroll
      for (int t = 0; t < V_T0; ++t) acc[f][t] = bias;
    for (int ci = 0; ci < V_BINS; ++ci)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float wv = __ldg(w.w0 + (ci * 3 + k) * 128 + co);
#pragma unroll
        for (int f = 0; f < VF / 2; ++f)
#pragma unroll
          for (int t = 0; t < V_T0; ++t) {
            const int ti = t + k - 1;
            if (ti >= 0 && ti < V_T0) acc[f][t] = fmaf(wv, bufB[((f0 + f) * V_BINS + ci) * V_T0 + ti], acc[f][t]);
          }
      }
#pragma unroll
    for (int f = 0; f < VF / 2; ++f)
#pragma unroll
      for (int t = 0; t < V_T0; ++t) bufA[((f0 + f) * 128 + co) * V_T0 + t] = fmaxf(acc[f][t], 0.f);
  }
  __syncthreads();

  // ---- conv1: 128 -> 64, stride 2, 4 -> 2 steps (bufA -> bufB)
  {
    const int co = tid & 63, f0 = (tid >> 6) * (VF / 4);
    float acc[VF / 4][2];
    const float bias = __ldg(w.b1 + co);
#pragma unroll
    for (int f = 0; f < VF / 4; ++f) acc[f][0] = acc[f][1] = bias;
    for (int ci = 0; ci < 128; ++ci)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float wv = __ldg(w.w1 + (ci * 3 + k) * 64 + co);
#pragma unroll
        for (int f = 0; f < VF / 4; ++f)
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int ti = 2 * t + k - 1;
            if (ti >= 0 && ti < V_T0) acc[f][t] = fmaf(wv, bufA[((f0 + f) * 128 + ci) * V_T0 + ti], acc[f][t]);
          }
      }
#pragma unroll
    for (int f = 0; f < VF / 4; ++f)
#pragma unroll
      for (int t = 0; t < 2; ++t) bufB[((f0 + f) * 64 + co) * 2 + t] = fmaxf(acc[f][t], 0.f);
  }
  __syncthreads();

  // ---- conv2: 64 -> 64, stride 2, 2 -> 1 step (bufB -> bufA); only taps k = 1, 2 see data (k = 0 is the left pad)
  {
    const int co = tid & 63, f0 = (tid >> 6) * (VF / 4);
    float acc[VF / 4];
    const float bias = __ldg(w.b2 + co);
#pragma unroll
    for (int f = 0; f < VF / 4; ++f) acc[f] = bias;
    for (int ci = 0; ci < 64; ++ci)
#pragma unroll
      for (int k = 1; k < 3; ++k) {
        const float wv = __ldg(w.w2 + (ci * 3 + k) * 64 + co);
#pragma unroll
        for (int f = 0; f < VF / 4; ++f) acc[f] = fmaf(wv, bufB[((f0 + f) * 64 + ci) * 2 + (k - 1)], acc[f]);
      }
#pragma unroll
    for (int f = 0; f < VF / 4; ++f) bufA[(f0 + f) * 64 + co] = fmaxf(acc[f], 0.f);
  }
  __syncthreads();

  // ---- conv3: 64 -> 128, 1 step (bufA -> bufB); only the centre tap sees data
  {
    const int co = tid & 127, f0 = (tid >> 7) * (VF / 2);
    float acc[VF / 2];
    const float bias = __ldg(w.b3 + co);
#pragma unroll
    for (int f = 0; f < VF / 2; ++f) acc[f] = bias;
    for (int ci = 0; ci < 64; ++ci) {
      const float wv = __ldg(w.w3 + (ci * 3 + 1) * 128 + co);
#pragma unroll
      for (int f = 0; f < VF / 2; ++f) acc[f] = fmaf(wv, bufA[(f0 + f) * 64 + ci], acc[f]);
    }
#pragma unroll
    for (int f = 0; f < VF / 2; ++f) bufB[(f0 + f) * 128 + co] = fmaxf(acc[f], 0.f);
  }
  __syncthreads();

  // ---- LSTM input projection: gx[g][r] = b_ih[r] + b_hh[r] + W_ih[r] . x, rows tid and tid + 256
  {
    float acc[2][VF];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int r = tid + j * VT;
      const float bias = __ldg(w.b_ih + r) + __ldg(w.b_hh + r);
#pragma unroll
      for (int f = 0; f < VF; ++f) acc[j][f] = bias;
    }
    for (int k = 0; k < V_H; ++k) {
      const float w0 = __ldg(w.w_ih + k * V_G + tid), w1 = __ldg(w.w_ih + k * V_G + tid + VT);
#pragma unroll
      for (int f = 0; f < VF; ++f) {
        const float x = bufB[f * 128 + k];
        acc[0][f] = fmaf(w0, x, acc[0][f]);
        acc[1][f] = fmaf(w1, x, acc[1][f]);
      }
    }
#pragma unroll
    for (int f = 0; f < VF; ++f)
      if (g0 + f < total) {
        gx[(g0 + f) * V_G + tid] = acc[0][f];
        gx[(g0 + f) * V_G + tid + VT] = acc[1][f];
      }
  }
}

// One cluster per stream.  Thread tid of CTA `rank` owns gate row (tid / 32) * 128 + rank * 32 + tid % 32 (gate order
// i, f, g, o) and keeps that row of W_hh in registers.  Warp 0 updates c and h of the CTA's 32 units and writes h into
// the next h buffer of all four CTAs; one cluster barrier per step orders those writes before the next step's reads
// (the buffers alternate, so no step overwrites an h another CTA may still be reading).  After the barrier warp 1 of
// rank 0 turns the full h into the frame's probability.
__global__ void __cluster_dims__(V_CL, 1, 1) __launch_bounds__(V_UNITS * 4)
vad_lstm_kernel(VadWeights w, const float* __restrict__ gx, const long* __restrict__ frame_off, float* __restrict__ probs) {
  __shared__ __align__(16) float h[2][V_H];
  __shared__ float gate[V_UNITS * 4];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank(), tid = threadIdx.x;
  const int b = blockIdx.x / V_CL;
  const int u = tid & (V_UNITS - 1), row = (tid / V_UNITS) * V_H + rank * V_UNITS + u;
  const long f0 = frame_off[b], n = frame_off[b + 1] - f0;

  float wr[V_H];
  const float4* wrow = reinterpret_cast<const float4*>(w.w_hh + (long)row * V_H);
#pragma unroll
  for (int k = 0; k < V_H / 4; ++k) {
    const float4 v = __ldg(wrow + k);
    wr[4 * k] = v.x; wr[4 * k + 1] = v.y; wr[4 * k + 2] = v.z; wr[4 * k + 3] = v.w;
  }
  float wo[4] = {0.f, 0.f, 0.f, 0.f}, bo = 0.f;
  if (rank == 0 && tid >= 32 && tid < 64) {
#pragma unroll
    for (int j = 0; j < 4; ++j) wo[j] = __ldg(w.w_out + (tid - 32) * 4 + j);
    bo = __ldg(w.b_out);
  }
  for (int i = tid; i < 2 * V_H; i += blockDim.x) (&h[0][0])[i] = 0.f;
  float* hdst[V_CL];
#pragma unroll
  for (int r = 0; r < V_CL; ++r) hdst[r] = cluster.map_shared_rank(&h[0][0], r);
  float cst = 0.f;
  cluster.sync();   // every CTA's h is zeroed before any CTA writes into it

  float gnext = n > 0 ? __ldg(gx + f0 * V_G + row) : 0.f;
  for (long t = 0; t < n; ++t) {
    const int cur = (int)(t & 1);
    const float gcur = gnext;
    if (t + 1 < n) gnext = __ldg(gx + (f0 + t + 1) * V_G + row);
    const float4* hv = reinterpret_cast<const float4*>(h[cur]);
    float a0 = gcur, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int k = 0; k < V_H / 4; ++k) {
      const float4 x = hv[k];
      a0 = fmaf(wr[4 * k], x.x, a0);
      a1 = fmaf(wr[4 * k + 1], x.y, a1);
      a2 = fmaf(wr[4 * k + 2], x.z, a2);
      a3 = fmaf(wr[4 * k + 3], x.w, a3);
    }
    gate[tid] = (a0 + a1) + (a2 + a3);
    __syncthreads();
    if (tid < V_UNITS) {
      const float ig = vsigmoid(gate[u]), fg = vsigmoid(gate[V_UNITS + u]);
      const float gg = tanhf(gate[2 * V_UNITS + u]), og = vsigmoid(gate[3 * V_UNITS + u]);
      cst = fg * cst + ig * gg;
      const float hn = og * tanhf(cst);
#pragma unroll
      for (int r = 0; r < V_CL; ++r) hdst[r][(cur ^ 1) * V_H + rank * V_UNITS + u] = hn;
    }
    cluster.sync();
    if (rank == 0 && tid >= 32 && tid < 64) {
      const float* hn = h[cur ^ 1] + (tid - 32) * 4;
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) s = fmaf(wo[j], fmaxf(hn[j], 0.f), s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (tid == 32) probs[f0 + t] = vsigmoid(s + bo);
    }
  }
}

void vad_front(cudaStream_t st, const VadWeights& w, const float* pcm, const long* pcm_off, const long* frame_off, int B,
               long total_frames, float* gx) {
  if (total_frames <= 0) return;
  const long grid = (total_frames + VF - 1) / VF;
  vad_front_kernel<<<(unsigned)grid, VT, 0, st>>>(w, pcm, pcm_off, frame_off, B, total_frames, gx);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

void vad_lstm(cudaStream_t st, const VadWeights& w, const float* gx, const long* frame_off, int B, float* probs) {
  vad_lstm_kernel<<<B * V_CL, V_UNITS * 4, 0, st>>>(w, gx, frame_off, probs);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

}  // namespace wl
