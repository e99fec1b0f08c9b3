// Shared device/host helpers for libwlb200 (sm_90a).
// PTX wrappers for mbarrier, TMA (cp.async.bulk[.tensor]) and wgmma, hand-written from the PTX ISA.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <utility>

#define WL_OK 0
#define WL_ERR_CUDA -1
#define WL_ERR_ARG -2
#define WL_ERR_STATE -3
#define WL_ERR_NOMEM -4

namespace wl {

struct Error {
  int code;
  std::string msg;
};

#define WL_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      char _b[512];                                                                           \
      snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      throw wl::Error{WL_ERR_CUDA, _b};                                                       \
    }                                                                                         \
  } while (0)

#define WL_CHECK(cond, code, ...)                                  \
  do {                                                             \
    if (!(cond)) {                                                 \
      char _b[512];                                                \
      snprintf(_b, sizeof(_b), __VA_ARGS__);                       \
      throw wl::Error{code, std::string(_b)};                      \
    }                                                              \
  } while (0)

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }
void note_launch(int n);  // kernel launch accounting (misc.cu)

// Launches issued while a PdlScope(true) is alive carry the programmatic-stream-serialization attribute (the decoder
// step: ~420 short dependent kernels per token, whose launch ramps and weight prefetch overlap the predecessor's
// tail).  WLB200_PDL=0 disables it.
bool pdl_active();
struct PdlScope {
  explicit PdlScope(bool on);
  ~PdlScope();
  bool prev;
};

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
static inline void launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_active() ? 1 : 0;
  WL_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...));
}

// ----------------------------------------------------------------------------------- in-graph timeline (debug)
// WLB200_TIMELINE=<file>: every decode-step kernel stamps %globaltimer at entry (what=0) and right after its
// dependency wait (what=1) from one thread of block 0 into a device log (slot 0 = entry counter).  The deltas between
// consecutive "ready" stamps are the per-kernel cost INSIDE the replayed CUDA graph, which ncu cannot show
// (tools/timeline.py).  One pointer per translation unit (no relocatable device code), bound by tl_bind().
constexpr unsigned TL_CAP = 1u << 20;
static __device__ unsigned long long* wl_tl_buf = nullptr;
// Compiled in only with -DWLB200_TL=1 (python -m whisperlive_b200.build --timeline): even one thread's worth of
// stamping code is instruction-cache footprint in kernels that are launched 400 times per token.
#ifndef WLB200_TL
#define WLB200_TL 0
#endif
__device__ __forceinline__ void tl_stamp_any(int kernel_id, int what) {
  if (!WLB200_TL) return;
  unsigned long long* buf = wl_tl_buf;
  if (buf != nullptr) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned idx = atomicAdd(reinterpret_cast<unsigned*>(buf), 1u);
    if (idx < TL_CAP) buf[1 + idx] = (t << 8) | ((unsigned long long)kernel_id << 2) | (unsigned long long)what;
  }
}
__device__ __forceinline__ void tl_stamp(int kernel_id, int what) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) tl_stamp_any(kernel_id, what);
}
static inline void tl_bind_tu(unsigned long long* p) { cudaMemcpyToSymbol(wl_tl_buf, &p, sizeof(p)); }
enum TlKernel : int { TL_EMBED = 1, TL_LN = 2, TL_GEMM_PART = 3, TL_SELF = 4, TL_CROSS = 5, TL_COMBINE = 6, TL_GELU = 7,
                      TL_SROWS = 8, TL_SSTREAMS = 9, TL_GEMM = 10, TL_DSTEP = 11 };

// ----------------------------------------------------------------------------------- generic
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 r;\n\t"
      "elect.sync r|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// GELU in its exact erf form, 0.5 x (1 + erf(x / sqrt 2)).  erf is evaluated with Abramowitz-Stegun 7.1.26
// (|error| <= 1.5e-7, i.e. fp32 rounding level): with p = poly(t) t exp(-z^2), t = 1 / (1 + 0.3275911 z),
// z = |x| / sqrt 2, gelu(x) = max(x, 0) - |x| p / 2.  Two MUFU ops (rcp.approx, ex2.approx) + 11 FP32 ops and
// no branches -- the epilogue of the 4d-wide MLP GEMM evaluates it 61 M times per encoder layer pass.
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f)));
  const float w = ax * 0.84932180028801904272f;   // sqrt(log2(e) / 2): exp(-x^2 / 2) = 2^(-w^2)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-w * w));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  return fmaxf(x, 0.f) - ax * (poly * t * e);
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor in the stream is still running; it must execute pdl_wait() before it touches anything
// the predecessor wrote (weights and other long-lived data may be fetched earlier).  pdl_trigger() lets the
// successor's CTAs be scheduled as soon as every CTA of this grid has issued it.  Both are no-ops for kernels
// launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Named barriers (ids 1..15; 0 is __syncthreads).  `arrive` signals without waiting, so a barrier of n threads can hand a
// turn from one warpgroup (arrive) to another (sync).
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Per-warpgroup register budget (every warp of the warpgroup executes it): producers give registers back, consumers
// take them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ----------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 4-D tiled load: coordinates innermost first.
__device__ __forceinline__ void tma_load_4d(void* dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// 1-D bulk copy global -> shared, bytes multiple of 16, 16B-aligned both sides.
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ----------------------------------------------------------------------------------- wgmma (warpgroup MMA)
// D[regs] (+)= A * B^T over one warpgroup (4 consecutive warps starting at a multiple of 4): M = 64 rows, fp16 inputs,
// fp32 accumulate.  Accumulator fragment of thread t = 32 w + l: element d[4 c + 2 i + j] is row 16 w + l / 4 + 8 i,
// column 8 c + 2 (l % 4) + j.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// A and B both from shared memory, both K-major (descriptors from wgmma_desc_sw128); scale_d = 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_ss<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7"
      "}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// Shared-memory matrix descriptor of a K-major operand tile stored as rows of 128 bytes with the 128-byte swizzle (what
// TMA SWIZZLE_128B writes): 8-row groups are 1024 B apart (SBO), LBO unused, tile base 1024-byte aligned.
// bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout (1 = SWIZZLE_128B).  Advancing 16 halves along
// K inside the swizzled row is +2 on the descriptor (32 bytes >> 4).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// 128 x BN x 64 tile step shared by the TMA-fed GEMMs: warpgroup wg (0 or 1) multiplies rows 64 wg .. 64 wg + 63 of
// the A stage (128 rows x 128 B, SW128) with the BN rows of the B stage.
template <int BN>
__device__ __forceinline__ void wgmma_tile_k64(float (&acc)[BN / 2], const uint8_t* sa, const uint8_t* sb, int wg, bool accumulate) {
  const uint64_t adesc = wgmma_desc_sw128(smem_u32(sa + wg * 64 * 128));
  const uint64_t bdesc = wgmma_desc_sw128(smem_u32(sb));
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_ss<BN>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (accumulate || k > 0) ? 1u : 0u);
}

// Calls f(row, col, value) for every accumulator element this thread holds (row in 0..63 of its warpgroup).
template <int R, class F>
__device__ __forceinline__ void wgmma_acc_foreach(const float (&d)[R], F&& f) {
  const int l = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r0 = 16 * w + (l >> 2), c0 = 2 * (l & 3);
#pragma unroll
  for (int c = 0; c < R / 4; ++c)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) f(r0 + 8 * i, 8 * c + c0 + j, d[4 * c + 2 * i + j]);
}
#endif  // __CUDACC__

}  // namespace wl
