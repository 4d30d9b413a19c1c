// The samplers' Gaussian draws as a counter-based generator: the value of one element is a pure function of
// (seed, stream tag, global image row, draw index, element index), so a restored image does not depend on the batch it sat in,
// on padding, on how a schedule was cut into ranges or on how many GPUs shared the work.
//   Philox4x32-10 (Salmon et al., Random123 constants); key = (seed low, seed high); counter = (q, draw, row, tag) with
//   q = element index inside one image (flattened C,H,W) / 4: one call yields the values of elements 4q .. 4q+3.
//   u = ((x >> 9) + 0.5) * 2^-23: 23 bits, so that the sum is exact in fp32 and u lies strictly inside (0,1) (with 24 bits
//   the top inputs would round up to 1.0); Box-Muller on (x0,x1) and (x2,x3):
//   r = sqrtf(-2 logf(u_a)), z = r * cospif(2 u_b), r * sinpif(2 u_b), with the full-precision library functions.
// oracle/noise.py states the same in numpy.
#pragma once
#include <cstdint>
#include <type_traits>

#include <cuda_runtime.h>

#include "../../include/ddnm_b200.h"

namespace ddnm {

// stream tags
enum : unsigned { NZ_LOOP = 0, NZ_XT = 1, NZ_Y = 2, NZ_HQ = 3, NZ_DEQUANT = 4 };

// Where a kernel takes its draws from.  tape != nullptr: a caller's buffer laid out like the images ("row" is then the row
// inside that buffer).  tape == nullptr: generated, row0 = global index of the batch's first image.
struct NoiseSrc {
  const float* tape;
  unsigned long long seed;
  long long row0;
  unsigned tag, draw;
};
inline NoiseSrc noise_tape(const float* tape) { return NoiseSrc{tape, 0ull, 0ll, 0u, 0u}; }
// the generated source of a B-row call of the C ABI (throws on a null seed or rows beyond the 32-bit row counter)
NoiseSrc noise_seeded(const ddnm_noise_seed* seed, unsigned tag, unsigned draw, int B);

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = 0xD2511F53ull * c.x, p1 = 0xCD9E8D57ull * c.z;
    c = make_uint4((unsigned)(p1 >> 32) ^ c.y ^ k.x, (unsigned)p1, (unsigned)(p0 >> 32) ^ c.w ^ k.y, (unsigned)p0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ float noise_uniform(unsigned x) { return ((float)(x >> 9) + 0.5f) * 1.1920928955078125e-7f; }

__device__ __forceinline__ float2 box_muller(unsigned xa, unsigned xb) {
  const float r = sqrtf(-2.0f * logf(noise_uniform(xa)));
  float s, c;
  sincospif(2.0f * noise_uniform(xb), &s, &c);
  return make_float2(r * c, r * s);
}

__device__ __forceinline__ uint4 noise_bits(const NoiseSrc& z, int row, long long q) {
  return philox4x32_10(make_uint4((unsigned)q, z.draw, (unsigned)(z.row0 + row), z.tag),
                       make_uint2((unsigned)z.seed, (unsigned)(z.seed >> 32)));
}
// generated values of elements 4q .. 4q+3 of image `row`
__device__ __forceinline__ float4 noise_quad(const NoiseSrc& z, int row, long long q) {
  const uint4 x = noise_bits(z, row, q);
  const float2 a = box_muller(x.x, x.y), b = box_muller(x.z, x.w);
  return make_float4(a.x, a.y, b.x, b.y);
}
// generated values of elements 2p, 2p+1 (half a quad: one Philox call, one Box-Muller)
__device__ __forceinline__ float2 noise_pair(const NoiseSrc& z, int row, long long p) {
  const uint4 x = noise_bits(z, row, p >> 1);
  return (p & 1) ? box_muller(x.z, x.w) : box_muller(x.x, x.y);
}
__device__ __forceinline__ float noise_at(const NoiseSrc& z, int row, long long elem) {
  const float2 v = noise_pair(z, row, elem >> 1);
  return (elem & 1) ? v.y : v.x;
}
// Every consumer kernel takes GEN as a template parameter, so its tape form is the plain load it always was.  A launch site picks
// the instantiation here: f(std::bool_constant<GEN>{}) with GEN = the draws are generated (no tape).
template <class F>
inline void noise_dispatch(const NoiseSrc& z, F&& f) {
  if (z.tape) f(std::false_type{});
  else f(std::true_type{});
}

// out[b][e] = the generated value of element e of image row0 + b  (ddnm_noise_fill; also fills an operator's one-pair scratch)
void noise_fill(const NoiseSrc& z, float* out, int B, long long per_image, cudaStream_t st);
// out[i] = a*x[i] + b*z[i] over n elements, img per image row: the samplers' time-travel re-noise and hq_demo's _undo.
// out == x is allowed.
void renoise(const float* x, float a, float b, const NoiseSrc& z, float* out, long long n, long long img, cudaStream_t st);

}  // namespace ddnm
