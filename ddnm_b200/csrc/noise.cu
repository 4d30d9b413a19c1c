// Materialised form of the generator of noise.cuh: what a caller uses for x_T and the measurement noise, what the operators
// whose Lambda_noise is a transform (not a map) fill their one-pair scratch with, and what the tests compare the in-register
// consumers against.  Also the one elementwise consumer shared by the loops: the re-noise a*x + b*z.
#include "noise.cuh"

#include "../../include/ddnm_b200.h"
#include "api_util.cuh"

namespace ddnm {

// thread = one quad; the last quad of an image whose length is not a multiple of 4 stores its leading values only
__global__ void noise_fill_kernel(NoiseSrc z, float* __restrict__ out, long long per_image, long long quads, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = (int)(i / quads);
  const long long q = i - (long long)b * quads;
  const float4 v = noise_quad(z, b, q);
  float* o = out + (long long)b * per_image + 4 * q;
  if ((per_image & 3) == 0) {
    *reinterpret_cast<float4*>(o) = v;
  } else {
    const float a[4] = {v.x, v.y, v.z, v.w};
    for (int k = 0; k < 4 && 4 * q + k < per_image; ++k) o[k] = a[k];
  }
}

void noise_fill(const NoiseSrc& z, float* out, int B, long long per_image, cudaStream_t st) {
  const long long quads = (per_image + 3) / 4, total = quads * B;
  noise_fill_kernel<<<(unsigned)cdivll(total, 256), 256, 0, st>>>(z, out, per_image, quads, total);
  CUDA_CHECK(cudaGetLastError());
}

// x and out may alias (the in-place undo), so neither is __restrict__
template <bool GEN>
__global__ void renoise_kernel(const float* x, float a, float b, NoiseSrc z, float* out, long long n, long long img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float zi;
  if (GEN) {
    const long long r = i / img;
    zi = noise_at(z, (int)r, i - r * img);
  } else {
    zi = z.tape[i];
  }
  out[i] = __fadd_rn(__fmul_rn(a, x[i]), __fmul_rn(b, zi));
}

void renoise(const float* x, float a, float b, const NoiseSrc& z, float* out, long long n, long long img, cudaStream_t st) {
  noise_dispatch(z, [&](auto gen) {
    renoise_kernel<decltype(gen)::value><<<(unsigned)cdivll(n, 256), 256, 0, st>>>(x, a, b, z, out, n, img);
  });
  CUDA_CHECK(cudaGetLastError());
}

NoiseSrc noise_seeded(const ddnm_noise_seed* seed, unsigned tag, unsigned draw, int B) {
  DDNM_CHECK(seed != nullptr, "null noise seed");
  DDNM_CHECK(seed->row_offset >= 0 && seed->row_offset + B <= 0xffffffffll, "image rows outside the generator's 32-bit row counter");
  return NoiseSrc{nullptr, seed->seed, seed->row_offset, tag, draw};
}

}  // namespace ddnm

using namespace ddnm;
extern "C" int ddnm_noise_fill(const ddnm_noise_seed* seed, unsigned tag, unsigned draw, float* out, int B, long long per_image,
                               void* stream) {
  DDNM_API_BEGIN
  DDNM_CHECK(out && B >= 1 && per_image >= 1, "bad noise fill arguments");
  const NoiseSrc z = noise_seeded(seed, tag, draw, B);
  DDNM_CHECK(per_image % 4 != 0 || reinterpret_cast<uintptr_t>(out) % 16 == 0, "out must be 16-byte aligned");
  noise_fill(z, out, B, per_image, (cudaStream_t)stream);
  DDNM_API_END
}
