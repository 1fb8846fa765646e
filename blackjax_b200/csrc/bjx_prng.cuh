// Device restatement of the jax.random pieces on the HMC/NUTS path (threefry2x32, partitionable
// mode; jax 0.10.0, the version pinned by the reference's uv.lock:1309-1310).
// Reference call sites: blackjax/mcmc/hmc.py:299, nuts.py:133, trajectory.py:321,645-650,
// proposal.py:123,156,226, util.py:90.  Integer results are bit-exact by construction.
#pragma once
#include <stdint.h>

namespace bjx {

struct Key {
  uint32_t a, b;
};

__host__ __device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) {
#ifdef __CUDA_ARCH__
  return __funnelshift_l(x, x, r);
#else
  return (x << r) | (x >> (32 - r));
#endif
}

// Threefry-2x32, 20 rounds.
__host__ __device__ __forceinline__ void threefry2x32(uint32_t k0, uint32_t k1, uint32_t x0, uint32_t x1,
                                                      uint32_t& o0, uint32_t& o1) {
  const uint32_t k2 = k0 ^ k1 ^ 0x1BD11BDAu;
  x0 += k0;
  x1 += k1;
#define BJX_R4(r0, r1, r2, r3)                \
  x0 += x1; x1 = rotl32(x1, r0); x1 ^= x0;    \
  x0 += x1; x1 = rotl32(x1, r1); x1 ^= x0;    \
  x0 += x1; x1 = rotl32(x1, r2); x1 ^= x0;    \
  x0 += x1; x1 = rotl32(x1, r3); x1 ^= x0;
  BJX_R4(13, 15, 26, 6)   x0 += k1; x1 += k2 + 1u;
  BJX_R4(17, 29, 16, 24)  x0 += k2; x1 += k0 + 2u;
  BJX_R4(13, 15, 26, 6)   x0 += k0; x1 += k1 + 3u;
  BJX_R4(17, 29, 16, 24)  x0 += k1; x1 += k2 + 4u;
  BJX_R4(13, 15, 26, 6)   x0 += k2; x1 += k0 + 5u;
#undef BJX_R4
  o0 = x0;
  o1 = x1;
}

// jax.random.split(key, n)[i] == jax.random.fold_in(key, i) == threefry(key, (0, i))
__host__ __device__ __forceinline__ Key fold_in(Key k, uint32_t data) {
  Key o;
  threefry2x32(k.a, k.b, 0u, data, o.a, o.b);
  return o;
}

// random_bits(key, 32, shape)[i] (row-major linear index i < 2^32)
__host__ __device__ __forceinline__ uint32_t random_bits(Key k, uint32_t i) {
  uint32_t a, b;
  threefry2x32(k.a, k.b, 0u, i, a, b);
  return a ^ b;
}

// jax.random.randint(key, shape, minval, maxval)[i] for int32 (jax/_src/random.py _randint): k1, k2 = split(key);
// higher / lower = random_bits(k1 / k2); span = maxval - minval (1 when maxval <= minval); multiplier =
// ((2^16 % span)^2) % span = 2^32 % span; offset = ((higher % span) * multiplier + lower % span) % span, all in uint32.
__host__ __device__ __forceinline__ int randint_at(Key key, uint32_t i, int minval, int maxval) {
  const uint32_t hi = random_bits(fold_in(key, 0u), i), lo = random_bits(fold_in(key, 1u), i);
  uint32_t span = (uint32_t)maxval - (uint32_t)minval;
  if (maxval <= minval) span = 1u;
  uint32_t mult = (1u << 16) % span;
  mult = (mult * mult) % span;
  const uint32_t off = ((hi % span) * mult + lo % span) % span;
  return (int)((uint32_t)minval + off);
}

__device__ __forceinline__ float bits_to_unit(uint32_t bits) {
  return __fsub_rn(__uint_as_float((bits >> 9) | 0x3F800000u), 1.0f);  // [0,1)
}

// jax.random.uniform(key, ()) in [0,1): max(0, f*1 + 0) == f
__device__ __forceinline__ float uniform01(Key k, uint32_t i = 0u) { return bits_to_unit(random_bits(k, i)); }

// XLA's float32 erf_inv (Giles' polynomial), evaluated unfused like the oracle.
__device__ __forceinline__ float erfinv_f32(float x) {
  float w = -log1pf(-__fmul_rn(x, x));
  const bool lt = w < 5.0f;
  float ww = lt ? __fsub_rn(w, 2.5f) : __fsub_rn(sqrtf(w), 3.0f);
  float p = lt ? 2.81022636e-08f : -0.000200214257f;
#define BJX_H(a, b) p = __fadd_rn(lt ? (a) : (b), __fmul_rn(p, ww));
  BJX_H(3.43273939e-07f, 0.000100950558f)
  BJX_H(-3.5233877e-06f, 0.00134934322f)
  BJX_H(-4.39150654e-06f, -0.00367342844f)
  BJX_H(0.00021858087f, 0.00573950773f)
  BJX_H(-0.00125372503f, -0.0076224613f)
  BJX_H(-0.00417768164f, 0.00943887047f)
  BJX_H(0.246640727f, 1.00167406f)
  BJX_H(1.50140941f, 2.83297682f)
#undef BJX_H
  float r = __fmul_rn(p, x);
  if (fabsf(x) == 1.0f) r = x * __int_as_float(0x7f800000);
  return r;
}

// jax.random.normal(key, (D,))[i] = sqrt(2) * erf_inv(uniform(lo = nextafter(-1, 0), hi = 1))
__device__ __forceinline__ float normal_at(Key k, uint32_t i) {
  const float lo = -0.99999994f;                       // nextafter(-1f, 0f)
  const float span = __fsub_rn(1.0f, lo);              // hi - lo in float32
  float f = bits_to_unit(random_bits(k, i));
  float u = fmaxf(lo, __fadd_rn(__fmul_rn(f, span), lo));
  return __fmul_rn(1.41421356237309515f, erfinv_f32(u));
}

}  // namespace bjx
