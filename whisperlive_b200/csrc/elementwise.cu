// Row-wise helper kernels: feature layout prep, LayerNorm, softmax, decoder token embedding.
#include <algorithm>

#include <cuda_bf16.h>

#include "kernels.cuh"

namespace wl {

void elementwise_tl_bind(unsigned long long* p) { tl_bind_tu(p); }

// ---------------------------------------------------------------------------- cast_weight_f16
__global__ void cast_weight_kernel(const float* __restrict__ in, __half* __restrict__ out, long n, long b, long k) {
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += stride) {
    // output index i = (a, kk, bb); input index = (a, bb, kk)
    const long bb = i % b, kk = (i / b) % k, a = i / (b * k);
    out[i] = __float2half_rn(in[(a * b + bb) * k + kk]);
  }
}
void cast_weight_f16(cudaStream_t st, const float* in, __half* out, long a, long b, long k) {
  const long n = a * b * k;
  const int grid = (int)std::min<long>((n + 255) / 256, 132L * 16);
  cast_weight_kernel<<<grid, 256, 0, st>>>(in, out, n, b, k);
  WL_CUDA(cudaGetLastError());
}

// ---------------------------------------------------------------------------- convert_weight (typed upload)
// One 16-byte load per thread and iteration: V source values.  Value j of the source becomes fp32 exactly (fp16 and
// bf16 widen exactly, int8 is (float)q / scale[row] with IEEE division), then __float2half_rn for fp16 targets.  The
// write goes to the relayout index of cast_weight_kernel ([a][b][k] -> [a][k][b]; b = k = 1 is the identity).
__device__ __forceinline__ float widen(float x) { return x; }
__device__ __forceinline__ float widen(__half x) { return __half2float(x); }
__device__ __forceinline__ float widen(__nv_bfloat16 x) { return __bfloat162float(x); }

__device__ __forceinline__ float load_scale(const void* s, int dt, long row) {
  if (dt == WDT_F16) return __half2float(((const __half*)s)[row]);
  if (dt == WDT_BF16) return __bfloat162float(((const __nv_bfloat16*)s)[row]);
  return ((const float*)s)[row];
}

template <class S>
__device__ __forceinline__ float src_value(S x, const void*, int, long) { return widen(x); }
template <>
__device__ __forceinline__ float src_value<int8_t>(int8_t q, const void* scale, int sdt, long row) {
  return __fdiv_rn((float)q, load_scale(scale, sdt, row));
}

__device__ __forceinline__ void store_out(float* out, long i, float v, int&) { out[i] = v; }
__device__ __forceinline__ void store_out(__half* out, long i, float v, int& bad) {
  const __half h = __float2half_rn(v);
  bad += __hisinf(h) && !isinf(v);   // a finite value beyond the fp16 range
  out[i] = h;
}

template <class S, class O>
__global__ void __launch_bounds__(256) convert_weight_kernel(const S* __restrict__ in, const void* __restrict__ scale, int sdt,
                                                             O* __restrict__ out, long n, long cols, long b, long k,
                                                             int* __restrict__ overflow) {
  constexpr int V = 16 / sizeof(S);
  const long stride = (long)gridDim.x * blockDim.x, nvec = n / V;
  const bool plain = b == 1 && k == 1;
  int bad = 0;
  for (long v = blockIdx.x * (long)blockDim.x + threadIdx.x; v < nvec; v += stride) {
    union { uint4 u; S s[V]; } x;
    x.u = __ldg(reinterpret_cast<const uint4*>(in) + v);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const long i = v * V + j;   // source index (a, bb, kk)
      const float f = src_value<S>(x.s[j], scale, sdt, i / cols);
      long o = i;
      if (!plain) {
        const long kk = i % k, bb = (i / k) % b, a = i / (b * k);
        o = (a * k + kk) * b + bb;
      }
      store_out(out, o, f, bad);
    }
  }
  // the ragged tail, fewer than V values
  for (long i = nvec * V + blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += stride) {
    const float f = src_value<S>(in[i], scale, sdt, i / cols);
    long o = i;
    if (!plain) {
      const long kk = i % k, bb = (i / k) % b, a = i / (b * k);
      o = (a * k + kk) * b + bb;
    }
    store_out(out, o, f, bad);
  }
  if (bad) atomicAdd(overflow, bad);
}

template <class O>
static void convert_weight_t(cudaStream_t st, const void* in, int dt, const void* scale, int sdt, O* out, long a, long b, long k,
                             long cols, int* overflow, int num_sms) {
  const long n = a * b * k;
  const int V = dt == WDT_F32 ? 4 : dt == WDT_I8 ? 16 : 8;
  const int grid = (int)std::max<long>(1, std::min<long>((n / V + 255) / 256, (long)num_sms * 8));
  if (dt == WDT_F32) convert_weight_kernel<<<grid, 256, 0, st>>>((const float*)in, scale, sdt, out, n, cols, b, k, overflow);
  else if (dt == WDT_F16) convert_weight_kernel<<<grid, 256, 0, st>>>((const __half*)in, scale, sdt, out, n, cols, b, k, overflow);
  else if (dt == WDT_BF16) convert_weight_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)in, scale, sdt, out, n, cols, b, k, overflow);
  else convert_weight_kernel<<<grid, 256, 0, st>>>((const int8_t*)in, scale, sdt, out, n, cols, b, k, overflow);
  WL_CUDA(cudaGetLastError());
}
void convert_weight_f16(cudaStream_t st, const void* in, int dt, const void* scale, int sdt, __half* out, long a, long b, long k,
                        long cols, int* overflow, int num_sms) {
  convert_weight_t(st, in, dt, scale, sdt, out, a, b, k, cols, overflow, num_sms);
}
void convert_weight_f32(cudaStream_t st, const void* in, int dt, const void* scale, int sdt, float* out, long n, long cols,
                        int* overflow, int num_sms) {
  convert_weight_t(st, in, dt, scale, sdt, out, n, 1, 1, cols, overflow, num_sms);
}

// ---------------------------------------------------------------------------- gather_windows
__global__ void gather_windows_kernel(const float* __restrict__ mel, const long* __restrict__ mel_off, const int* __restrict__ frames,
                                      const int* __restrict__ win_stream, const int* __restrict__ win_seek,
                                      const int* __restrict__ win_len, float* __restrict__ feat, int n_mels) {
  const int w = blockIdx.z, m = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3000) return;
  const int sidx = win_stream[w], T = frames[sidx], seek = win_seek[w], len = win_len[w];
  float v = 0.f;
  if (t < len && seek + t < T) v = mel[mel_off[sidx] + (long)m * T + seek + t];
  feat[((long)w * n_mels + m) * 3000 + t] = v;
}
void gather_windows(cudaStream_t st, const float* mel, const long* mel_off, const int* frames, const int* win_stream, const int* win_seek,
                    const int* win_len, float* feat, int n_windows, int n_mels) {
  dim3 grid(cdiv(3000, 256), n_mels, n_windows);
  gather_windows_kernel<<<grid, 256, 0, st>>>(mel, mel_off, frames, win_stream, win_seek, win_len, feat, n_mels);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ---------------------------------------------------------------------------- prep_features
// [B][n_mels][3000] f32 -> [B][3002][n_mels] fp16 with one zero row before and after (conv k=3, pad=1
// becomes a plain strided GEMM over overlapping rows).  32x32 smem transpose tiles.
__global__ void prep_features_kernel(const float* __restrict__ in, __half* __restrict__ out, int n_mels) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  const float* src = in + (long)b * n_mels * 3000;
  __half* dst = out + (long)b * 3002 * n_mels;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int m = m0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (m < n_mels && t < 3000) ? src[(long)m * 3000 + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int t = t0 + i, m = m0 + threadIdx.x;
    if (t < 3000 && m < n_mels) dst[(long)(t + 1) * n_mels + m] = __float2half_rn(tile[threadIdx.x][i]);
  }
  if (blockIdx.x == 0 && threadIdx.y == 0) {
    const int m = m0 + threadIdx.x;
    if (m < n_mels) {
      dst[m] = __float2half_rn(0.f);
      dst[(long)3001 * n_mels + m] = __float2half_rn(0.f);
    }
  }
}

void prep_features(cudaStream_t st, const float* feats, __half* out, int B, int n_mels) {
  dim3 grid(cdiv(3000, 32), cdiv(n_mels, 32), B), block(32, 8);
  prep_features_kernel<<<grid, block, 0, st>>>(feats, out, n_mels);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ---------------------------------------------------------------------------- layernorm_rows
// One warp per row, float4 loads, the row lives in registers (d <= 1280 -> 10 float4 per lane), two-pass
// statistics.  Kept deliberately compact: in the decode loop this kernel runs ~100 times per step on a
// handful of rows, where a long unrolled body costs more in instruction fetch than in arithmetic.
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                        const float* __restrict__ be, __half* __restrict__ y,
                                                        float* __restrict__ y32, long rows, int d) {
  const long row = blockIdx.x * 8L + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int n4 = d >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x + row * d);
  float4 v[10];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int c = i * 32 + lane;
    v[i] = c < n4 ? x4[c] : make_float4(0.f, 0.f, 0.f, 0.f);
    sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(sum) / d;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i * 32 + lane < n4) {
      const float a = v[i].x - mean, b2 = v[i].y - mean, c2 = v[i].z - mean, d2 = v[i].w - mean;
      sq += (a * a + b2 * b2) + (c2 * c2 + d2 * d2);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / d + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(be);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int c = i * 32 + lane;
    if (c < n4) {
      const float4 gg = g4[c], bb = b4[c];
      float4 o;
      o.x = (v[i].x - mean) * rstd * gg.x + bb.x;
      o.y = (v[i].y - mean) * rstd * gg.y + bb.y;
      o.z = (v[i].z - mean) * rstd * gg.z + bb.z;
      o.w = (v[i].w - mean) * rstd * gg.w + bb.w;
      if (y) {
        __align__(8) __half2 h[2] = {__floats2half2_rn(o.x, o.y), __floats2half2_rn(o.z, o.w)};
        *reinterpret_cast<uint2*>(y + row * d + 4 * c) = *reinterpret_cast<const uint2*>(h);
      }
      if (y32) *reinterpret_cast<float4*>(y32 + row * d + 4 * c) = o;
    }
  }
}

// Decode-step variant: one block of d/4 threads per row, ONE float4 per thread -- no column loop, no bounds checks, a
// hundred-odd instructions in all.  The decode step launches this ~100 times per token on a handful of rows; what a
// launch costs there is the instruction fetch of whatever it executes (the kernels of a layer do not fit the SM's
// instruction caches together), so it is written for size rather than generality.  It also folds in the residual update that the preceding split-K GEMM left as partial sums:
// x += bias + sum_s partial_s, in a fixed order (bit-reproducible).
__global__ void __launch_bounds__(384) layernorm_update_kernel(float* __restrict__ x, PartialSrc upd, const float* __restrict__ g,
                                                               const float* __restrict__ be, __half* __restrict__ y, int d) {
  const long row = blockIdx.x;
  __shared__ float red[2][12];
  const int tid = threadIdx.x, nw = blockDim.x >> 5;
  pdl_trigger();
  // bias, gamma, beta are weights: fetched before waiting for the producer kernel
  float4 v = (upd.nsplit > 0 && upd.bias) ? __ldg(reinterpret_cast<const float4*>(upd.bias) + tid) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + tid), bb = __ldg(reinterpret_cast<const float4*>(be) + tid);
  float4* x4 = reinterpret_cast<float4*>(x + row * d) + tid;
  tl_stamp(TL_LN, 0);
  pdl_wait();
  tl_stamp(TL_LN, 1);
  {
    const float4 a = *x4;
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
  }
  if (upd.nsplit > 0) {
    // K ranges in index order; at most 8 (dec_gemm_split_plan), predicated so that all loads are in flight together
    const float4* p4 = reinterpret_cast<const float4*>(upd.ptr + row * d) + tid;
    const long st4 = upd.stride >> 2;
    float4 q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) q[s] = s < upd.nsplit ? __ldcg(p4 + s * st4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int s = 0; s < 8; ++s) { v.x += q[s].x; v.y += q[s].y; v.z += q[s].z; v.w += q[s].w; }
    *x4 = v;
  }
  float sum = warp_sum((v.x + v.y) + (v.z + v.w));
  if ((tid & 31) == 0) red[0][tid >> 5] = sum;
  __syncthreads();
  sum = warp_sum((tid & 31) < nw ? red[0][tid & 31] : 0.f);   // every warp folds the (<= 12) warp sums itself
  const float mean = sum / d;
  const float a = v.x - mean, b2 = v.y - mean, c2 = v.z - mean, d2 = v.w - mean;
  float sq = warp_sum((a * a + b2 * b2) + (c2 * c2 + d2 * d2));
  if ((tid & 31) == 0) red[1][tid >> 5] = sq;
  __syncthreads();
  sq = warp_sum((tid & 31) < nw ? red[1][tid & 31] : 0.f);
  const float rstd = rsqrtf(sq / d + 1e-5f);
  __align__(8) __half2 h[2] = {__floats2half2_rn(a * rstd * gg.x + bb.x, b2 * rstd * gg.y + bb.y),
                               __floats2half2_rn(c2 * rstd * gg.z + bb.z, d2 * rstd * gg.w + bb.w)};
  *reinterpret_cast<uint2*>(y + row * d + 4 * tid) = *reinterpret_cast<const uint2*>(h);
}

void layernorm_update_rows(cudaStream_t st, float* x, const PartialSrc& upd, const float* gamma, const float* beta, __half* y,
                           int rows, int d) {
  WL_CHECK(d <= 1536 && d % 128 == 0, WL_ERR_ARG, "layernorm_update: unsupported width %d", d);
  WL_CHECK(upd.nsplit >= 0 && upd.nsplit <= 8 && (upd.nsplit == 0 || upd.stride % 4 == 0), WL_ERR_ARG,
           "layernorm_update: at most 8 K ranges, stride a multiple of 4");
  launch_kernel(layernorm_update_kernel, dim3(rows), dim3(d / 4), 0, st, x, upd, gamma, beta, y, d);
  note_launch(1);
}

void layernorm_rows(cudaStream_t st, const float* x, const float* gamma, const float* beta, __half* y, float* y32, long rows,
                    int d) {
  WL_CHECK(d <= 1280 && d % 4 == 0, WL_ERR_ARG, "layernorm: unsupported width %d", d);
  const int grid = cdiv(rows, 8);
  layernorm_kernel<<<grid, 256, 0, st>>>(x, gamma, beta, y, y32, rows, d);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ---------------------------------------------------------------------------- gelu_cast
__global__ void __launch_bounds__(256) gelu_cast_kernel(PartialSrc in, __half* __restrict__ out, int rows, int cols) {
  const long i4 = blockIdx.x * 256L + threadIdx.x;          // float4 index
  const int c4n = cols >> 2;
  pdl_trigger();
  if (i4 >= (long)rows * c4n) return;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (in.bias) v = __ldg(reinterpret_cast<const float4*>(in.bias) + (int)(i4 % c4n));
  tl_stamp(TL_GELU, 0);
  pdl_wait();
  tl_stamp(TL_GELU, 1);
  const float4* p4 = reinterpret_cast<const float4*>(in.ptr) + i4;
  const long st4 = in.stride >> 2;
  float4 q[4];
#pragma unroll
  for (int s = 0; s < 4; ++s) q[s] = s < in.nsplit ? __ldcg(p4 + s * st4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int s = 0; s < 4; ++s) { v.x += q[s].x; v.y += q[s].y; v.z += q[s].z; v.w += q[s].w; }
#pragma unroll 1
  for (int s = 4; s < in.nsplit; ++s) {   // more than 4 ranges: narrow FC1s at few rows (tiny at 17..32 rows gets 6)
    const float4 p = __ldcg(p4 + s * st4);
    v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
  }
  __align__(8) __half2 h[2] = {__floats2half2_rn(gelu_erf(v.x), gelu_erf(v.y)), __floats2half2_rn(gelu_erf(v.z), gelu_erf(v.w))};
  *reinterpret_cast<uint2*>(out + 4 * i4) = *reinterpret_cast<const uint2*>(h);
}

void gelu_cast(cudaStream_t st, const PartialSrc& in, __half* out, int rows, int cols) {
  WL_CHECK(cols % 4 == 0, WL_ERR_ARG, "gelu_cast: cols must be a multiple of 4");
  WL_CHECK(in.stride % 4 == 0, WL_ERR_ARG, "gelu_cast: partial stride must be a multiple of 4");
  launch_kernel(gelu_cast_kernel, dim3(cdiv((long)rows * cols / 4, 256)), dim3(256), 0, st, in, out, rows, cols);
  note_launch(1);
}

// ---------------------------------------------------------------------------- softmax_rows
// One warp per row of <= 1536 scores held in registers.
__global__ void __launch_bounds__(256) softmax_kernel(const float* __restrict__ s, __half* __restrict__ p, long rows, int n,
                                                      int ld_in, int ld_out, float scale) {
  const long row = blockIdx.x * 8L + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* sr = s + row * ld_in;
  float v[48];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 48; ++i) {
    const int c = i * 32 + lane;
    v[i] = c < n ? sr[c] * scale : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 48; ++i) {
    v[i] = __expf(v[i] - mx);
    sum += v[i];
  }
  const float inv = 1.f / warp_sum(sum);
  __half* pr = p + row * ld_out;
#pragma unroll
  for (int i = 0; i < 48; ++i) {
    const int c = i * 32 + lane;
    if (c < ld_out) pr[c] = __float2half_rn(c < n ? v[i] * inv : 0.f);
  }
}

void softmax_rows(cudaStream_t st, const float* s, __half* p, long rows, int n, int ld_in, int ld_out, float scale) {
  WL_CHECK(n <= 1536 && ld_out <= 1536, WL_ERR_ARG, "softmax_rows: row too long (%d)", n);
  softmax_kernel<<<cdiv(rows, 8), 256, 0, st>>>(s, p, rows, n, ld_in, ld_out, scale);
  WL_CUDA(cudaGetLastError());
  note_launch(1);
}

// ---------------------------------------------------------------------------- decoder_embed
__global__ void decoder_embed_kernel(DecodeState s, const __half* __restrict__ emb, const __half* __restrict__ pos_emb,
                                     float* __restrict__ x, int d) {
  const int r = blockIdx.x;
  pdl_trigger();
  pdl_wait();
  tl_stamp(TL_EMBED, 1);
  if (!s.active[r]) return;
  const int tok = s.tok_in[r], pos = s.pos[r];
  for (int c = threadIdx.x; c < d; c += blockDim.x)
    x[(long)r * d + c] = __half2float(emb[(long)tok * d + c]) + __half2float(pos_emb[(long)pos * d + c]);
  if (threadIdx.x == 0) s.src[(long)r * T_MAX + pos] = (short)r;
}

void decoder_embed(cudaStream_t st, const DecodeState& s, const __half* emb, const __half* pos_emb, float* x, int R, int d) {
  // First kernel of a decode step, deliberately NOT a programmatic dependent: it starts only after everything before
  // the step (decode_init, the previous step's search kernels) has completed, so the kernels of this step may read
  // that per-step state (done flags, slots, positions) ahead of their own dependency wait.
  PdlScope no_pdl(false);
  launch_kernel(decoder_embed_kernel, dim3(R), dim3(128), 0, st, s, emb, pos_emb, x, d);
  note_launch(1);
}

}  // namespace wl
