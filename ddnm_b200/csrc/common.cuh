// Shared helpers for the ddnm_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace ddnm {

// ---------------------------------------------------------------------------------------------
// Error handling: every C-ABI entry point catches ddnm::Error and stores the message thread-locally.
// ---------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define DDNM_CHECK(cond, msg)                                                                     \
  do {                                                                                            \
    if (!(cond)) throw ::ddnm::Error(std::string(msg) + " [" #cond "] at " __FILE__ ":" + std::to_string(__LINE__)); \
  } while (0)

#define CUDA_CHECK(expr)                                                                          \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      throw ::ddnm::Error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " in " #expr " at " __FILE__ ":" + \
                          std::to_string(__LINE__));                                              \
  } while (0)

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
// One-time per-DEVICE actions (cudaFuncSetAttribute is a per-device setting): true the first time `flags` sees the current device.
inline bool first_use_on_device(bool (&flags)[64]) {
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (flags[dev]) return false;
  flags[dev] = true;
  return true;
}
inline long long cdivll(long long a, long long b) { return (a + b - 1) / b; }

// Stream-ordered scratch that is returned to the pool on every exit path (a DDNM_CHECK throw inside a sampling loop must not
// leak the loop's buffers).
struct StreamBuf {
  float* p = nullptr;
  cudaStream_t st = nullptr;
  StreamBuf(size_t elems, cudaStream_t s) : st(s) {
    cudaError_t e = cudaMallocAsync((void**)&p, elems * sizeof(float), s);
    if (e != cudaSuccess) throw Error(std::string("CUDA error: ") + cudaGetErrorString(e) + " in cudaMallocAsync (sampler scratch)");
  }
  ~StreamBuf() {
    if (p) cudaFreeAsync(p, st);
  }
  StreamBuf(const StreamBuf&) = delete;
  StreamBuf& operator=(const StreamBuf&) = delete;
};

// One GroupNorm running sum: a two's-complement fixed-point accumulator with 48 fractional bits kept as two carry-free words
// (value = (hi * 2^32 + lo) * 2^-48, see stat_add).  Partial sums from many CTAs are added with integer atomics, so the total
// does not depend on the order in which they arrive: a forward pass is bit-reproducible run to run (floating-point atomics
// are not).  Range +-2^47, resolution 2^-48 (what a float partial sum loses below that is far under the fp32 noise of the
// statistics themselves).
struct StatAcc {
  unsigned long long lo;
  long long hi;
};

// Programmatic dependent launch (PDL): consecutive kernels of the forward carry cudaLaunchAttributeProgrammaticStreamSerialization,
// so a kernel's CTAs may be scheduled (and run their prologue: barrier init, descriptor prefetch) while the
// previous kernel's last CTAs drain; pdl_prologue() at the top of every such kernel (1) releases ITS successor and (2) blocks
// until the predecessor grid has completed and flushed, before any dependent global access.  Captured into the CUDA graph these
// become programmatic edges.  DDNM_PDL=0 launches everything fully serialised (A/B measurements).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (pdl_enabled()) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (cluster > 1) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = cluster;
    at[na].val.clusterDim.y = 1;
    at[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
  if (e != cudaSuccess) throw Error(std::string("CUDA error: ") + cudaGetErrorString(e) + " in cudaLaunchKernelEx");
}

// A strided NHWC fp32 activation view: element (n, y, x, c) at p[((n*H + y)*W + x)*ld + c].
// ld >= C lets a tensor live inside a channel slice of a wider (concat) buffer.
// st (optional): per-(image, channel) running sums for GroupNorm, st[(n*st_ld + c)*2 + {0,1}] = {sum, sum of squares}
// over the image's pixels; filled by the kernel that PRODUCES the tensor (tensor-core epilogue / gn_stats), so the
// normalisation never re-reads the tensor just to reduce it.
struct View {
  float* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0, ld = 0;
  StatAcc* st = nullptr;
  int st_ld = 0;
  long long pixels() const { return (long long)N * H * W; }
  View slice(int c0, int c) const {
    View v = *this;
    v.p = p + c0;
    v.C = c;
    if (st) v.st = st + 2 * (size_t)c0;
    return v;
  }
};

// fp16 (hi, lo) split of an activation: two contiguous NHWC planes.
struct SplitView {
  __half* hi = nullptr;
  __half* lo = nullptr;
  int N = 0, H = 0, W = 0, C = 0;   // dims of the planes as the consumer sees them
};

#ifdef __CUDACC__
// see launch_pdl: release the successor grid, then wait for the predecessor grid (no-ops without a programmatic dependency)
__device__ __forceinline__ void pdl_prologue() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
// ---------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier, TMA, wgmma.  Addresses are 32-bit shared-window addresses.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug traps (-> CUDA error) after ~2 s instead of hanging the GPU.  No printf here: a function call
// between wgmma instructions makes ptxas serialise the whole wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// --- wgmma (sm_90a warpgroup MMA) ---
// Shared-memory matrix descriptor of a K-major operand in the 128-byte-swizzled layout TMA writes with
// CU_TENSOR_MAP_SWIZZLE_128B: rows of 64 fp16 (128 B), 8-row atoms of 1024 B.  Start address >> 4 at [0,14),
// leading byte offset (unused for swizzled K-major, canonical 1) at [16,30), stride byte offset 1024 >> 4 at [32,46),
// layout type SWIZZLE_128B (= 1) at [62,64).  Advancing K by 16 fp16 (32 B) adds 2 to the start-address field.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N, fp32 registers of the warpgroup] (+)= A[64 x 16, smem desc] * B[N x 16, smem desc]^T, both K-major fp16
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
// --- clusters (the ping-pong CTA pairs): two CTAs of a cluster of 2 share each weight k-block through TMA multicast ---
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster.  The callers only hand back a stage whose
// wgmma reads have completed (wgmma.wait_group), so the arrive publishes no memory writes: with the default .cta scope it is a
// plain remote arrive, where .release.cluster would put a MEMBAR.ALL.GPU in front of every k-block's release.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// TMA load written to the same shared-memory offset in every CTA of `mask`, each completing bytes on its own barrier at `bar`
__device__ __forceinline__ void tma_load_3d_multicast(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
// warpgroup-wide register reallocation (warp-specialised kernels): every thread of the warpgroup executes the same instruction
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// acc += p, independent of the order of concurrent adds.  p is converted (exactly, unless it has bits below 2^-48) to a signed
// fixed-point integer X with 48 fractional bits, and X = W1 * 2^32 + W0 (W0 = X mod 2^32 >= 0, W1 = floor(X / 2^32)) is added
// as TWO independent integer reductions: acc->lo += W0 (up to 2^32 partial sums cannot wrap it), acc->hi += W1 (range +-2^47).
// No carry crosses between the words, so neither atomic needs its return value: both compile to fire-and-forget RED
// instructions (a carry-propagating 128-bit add needs the old low word back, a round trip to L2 per statistic that the
// epilogue warps of the tensor-core kernels had to wait for).
__device__ __forceinline__ void stat_add(StatAcc* acc, float p) {
  const int bits = __float_as_int(p);
  int ex = (bits >> 23) & 0xff;
  unsigned long long m = (unsigned long long)(bits & 0x7fffff);
  if (ex) m |= 0x800000ull; else ex = 1;          // |p| = m * 2^(ex - 150)
  const int sh = ex - 150 + 48;                   // X = m * 2^sh
  unsigned long long lo = 0, hi = 0;              // |X| as a 128-bit integer
  if (sh >= 64) hi = m << min(sh - 64, 7);         // |p| >= 2^47 cannot occur for activation sums; clamp the shift
  else if (sh > 0) { lo = m << sh; hi = sh > 40 ? m >> (64 - sh) : 0ull; }
  else if (sh > -24) lo = m >> (-sh);
  if (bits < 0) {                                 // two's-complement negate
    lo = ~lo + 1ull;
    hi = ~hi + (lo == 0ull ? 1ull : 0ull);
  }
  const unsigned long long w0 = lo & 0xffffffffull;
  const unsigned long long w1 = (hi << 32) | (lo >> 32);
  if (w0) atomicAdd(&acc->lo, w0);
  if (w1) atomicAdd(reinterpret_cast<unsigned long long*>(&acc->hi), w1);
}
// sum += v with the rounding error of the addition collected in comp (Knuth two-sum): sum + comp is the running total to ~2^-48
__device__ __forceinline__ void two_sum_acc(float& sum, float& comp, float v) {
  const float s = __fadd_rn(sum, v);
  const float bb = __fadd_rn(s, -sum);
  comp = __fadd_rn(comp, __fadd_rn(__fadd_rn(sum, -__fadd_rn(s, -bb)), __fadd_rn(v, -bb)));
  sum = s;
}
__host__ __device__ __forceinline__ double stat_value(const StatAcc& a) {
  return ((double)a.hi * 4294967296.0 + (double)a.lo) * (1.0 / 281474976710656.0);
}

// x * sigmoid(x) on the special-function unit (ex2.approx + fast divide, ~2e-7 relative)
__device__ __forceinline__ float swishf_fast(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  return __fdividef(x, 1.0f + e);
}
// fp32 -> (hi, lo) fp16 pair: hi = rn(x) saturated to the finite fp16 range, lo = rn(x - hi).
// hi + lo carries ~22 significant bits, so hi*hi + hi*lo + lo*hi reproduces an fp32 product to ~2^-21.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  unsigned short h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
  hi = __ushort_as_half(h);
  float r = x - __half2float(hi);
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(r));
  lo = __ushort_as_half(h);
}
// two fp32 values -> packed fp16 hi pair + packed fp16 lo pair (hi = rn(x) saturated to the finite range, lo = rn(x - hi))
__device__ __forceinline__ void split2_f16(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  const __half2 h = *reinterpret_cast<const __half2*>(&hi);
  const float2 f = __half22float2(h);
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - f.y), "f"(x0 - f.x));
}

#endif  // __CUDACC__

}  // namespace ddnm
